"""One context serving single runs and scenario batches in turn.  The single-scenario state and the batch state are separate pools of
the same type: a batch must not change what a single run left, and neither a single run nor an earlier batch may leak into a batch.
Every output is compared with the same call on a fresh context."""
import numpy as np
import pytest

from util import make_case


def _c3_gpu_share():
    # GPU-share slots and per-device memory are part of the state
    return make_case("c3", n_nodes=300, n_workloads=60, replicas=8, n_apps=2, seed_no=21, gpu_pct=25)[1]


def _open_local():
    from simon_b200 import simulator, synth
    from simon_b200.compiler import compile_cluster
    cluster, apps = synth.make_open_local(n_nodes=120, n_workloads=24, replicas=6, seed_no=6)
    pl = simulator.plan(cluster, apps)
    return compile_cluster(pl.nodes, pl.pods, pl.ctx, open_local=True, storage_classes=list(cluster.StorageClasss), local_devices=True)


def _lists(n_nodes):
    rng = np.random.RandomState(5)
    return [np.arange(n_nodes, dtype=np.uint32), np.sort(rng.choice(n_nodes, n_nodes * 2 // 3, replace=False)).astype(np.uint32),
            np.arange(n_nodes - 1, -1, -1, dtype=np.uint32)[:n_nodes // 2].copy()]


def _schedule(eng):
    out_node, score, fail_counts, fail_pod = eng.schedule()
    return dict(out_node=out_node, score=score, fail_counts=fail_counts, fail_pod=fail_pod)


def _state(eng, storage):
    s = dict(results=eng.results(), gpu_slots=eng.gpu_slots(), **eng.state(), **eng.state_ext())
    if storage:
        s["vg_requested"], s["dev_alloc"] = eng.storage_state(), eng.device_state()
    return s


def _batch(eng, storage, lists):
    res, nodes = (eng.run_scenarios_local if storage else eng.run_scenarios)(lists, want_nodes=True)
    for r in res:
        r.pop("elapsed_ms")
    b = dict(res=res, nodes=nodes)
    if storage:
        b["storage"] = [eng.scenario_storage_state(i) for i in range(len(lists))]
    return b


def _same(got, want, path=""):
    if isinstance(want, dict):
        assert sorted(got) == sorted(want), path
        for k in want:
            _same(got[k], want[k], f"{path}.{k}")
    elif isinstance(want, (list, tuple)) and not (want and isinstance(want[0], int)):
        assert len(got) == len(want), path
        for i, (g, w) in enumerate(zip(got, want)):
            _same(g, w, f"{path}[{i}]")
    elif want is None or isinstance(want, (int, float, list)):
        assert got == want, path
    else:
        np.testing.assert_array_equal(got, want, err_msg=path)


@pytest.mark.gpu
@pytest.mark.parametrize("storage", [False, True], ids=["c3_gpu_share", "open_local_devices"])
def test_single_runs_and_batches_on_one_context_match_fresh_contexts(storage):
    from simon_b200.engine import Engine
    c = _open_local() if storage else _c3_gpu_share()
    lists = _lists(c.n_nodes)
    with Engine(c, record_scores=True) as fresh:
        want_run = _schedule(fresh)
        want_state = _state(fresh, storage)
    with Engine(c, record_scores=True) as fresh:
        want_batch = _batch(fresh, storage, lists)
    assert (want_run["out_node"] >= 0).any()
    if storage:
        assert want_state["dev_alloc"].any()
    else:
        assert want_state["gpu_used"].any() and any(want_state["gpu_slots"])
    with Engine(c, record_scores=True) as eng:
        _same(_schedule(eng), want_run, "schedule")
        _same(_batch(eng, storage, lists), want_batch, "batch after schedule")
        _same(_state(eng, storage), want_state, "single state after the batch")
        eng.reset()
        _same(_schedule(eng), want_run, "schedule after reset")
        _same(_state(eng, storage), want_state, "single state after reset + schedule")
        eng.replay(2)
        _same(_state(eng, storage), want_state, "single state after replay")
        _same(_batch(eng, storage, lists), want_batch, "batch after replay")
