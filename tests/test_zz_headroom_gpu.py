"""Headroom probes on the device (simon_probe_run): every probe kernel variant against the CPU checker (tests/checkers.c), with and
without the static-verdict cache, the recompile + simon_schedule_resume equivalence that pins the definition on the workload and the
template path, the context state a probe batch leaves, chunking, the C-entry refusals and the session end to end."""
import copy
import os

import numpy as np
import pytest

from simon_b200 import abi, headroom, scaledown, simulator, synth
from simon_b200.compiler import compile_cluster
from test_headroom import PROBE_LOCAL_VARIANTS, PROBE_VARIANTS, _case
from test_open_local_oracle import make_mixed_local

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
EXAMPLE = os.path.join(HERE, "golden", "reference", "example")
ERR_INVALID, ERR_STATE = -1, -3


def _engine(c, **kw):
    from simon_b200.engine import Engine
    return Engine(c, device=0, **kw)


def _probe_pods(c, rng, n):
    """n pods (with repeats of classes) that reach the scheduler and are not pinned: the probes a user may ask for."""
    guard = scaledown.pod_guard(c)
    ok = [q for q in range(c.pods_dims["n_pods"]) if c.pods["pod_fixed_node"][q] == -1 and guard[q] == -1]
    return [int(q) for q in rng.choice(ok, size=min(n, len(ok)), replace=False)]


def _probes(c, placed, rng, n):
    free = headroom.free_pod_slots(c, placed)
    qs = _probe_pods(c, rng, n)
    return [(q, int(rng.integers(1, 12)) if j % 3 else max(1, free)) for j, q in enumerate(qs)]


def _assert_probe_equal(g, want, what):
    assert (g["n_placed"], g["stop_reason"]) == (want["n_placed"], want["stop_reason"]), what
    for k in ("node", "score", "gpu_slots", "fail_counts"):
        np.testing.assert_array_equal(g[k], want[k], err_msg=f"{what}: {k}")


@pytest.mark.parametrize("kernel", sorted(PROBE_VARIANTS))
def test_probe_variant_matches_checker(kernel):
    import checkers
    from oracle.binding import Oracle
    cs, t, big = PROBE_VARIANTS[kernel]
    rng = np.random.default_rng(23)
    stops = set()
    for seed in (0, 2, 5):
        cluster, apps = synth.make_mix(seed_no=seed, n_nodes=40)
        p = simulator.plan(cluster, apps)
        c = compile_cluster(p.nodes, p.pods, p.ctx)
        o = Oracle(c)
        placed = o.schedule()[0]
        probes = _probes(c, placed, rng, 10)
        for static_cache in (True, False):
            with _engine(c, record_scores=True, cluster_ctas=cs, threads_per_cta=t, force_large=big, static_cache=static_cache) as eng:
                got = eng.probe_run(placed, probes)
                li = eng.last_launch()
                assert li["kernel"] == kernel and li["n_scenarios"] == len(probes) and li["large"] == big, li
            for (q, r), g in zip(probes, got):
                want = checkers.probe(o, placed, q, r)
                _assert_probe_equal(g, want, f"{kernel} seed {seed} pod {q} static_cache {static_cache}")
                st = o.state()
                assert (g["req_mcpu"], g["req_mem"]) == (int(st["req_mcpu"].sum()), int(st["req_mem"].sum()))
                stops.add(g["stop_reason"])
        o.close()
    assert stops == {abi.PROBE_STOP_UNSCHEDULABLE, abi.PROBE_STOP_MAX_REPLICAS}


@pytest.mark.parametrize("kernel", sorted(PROBE_LOCAL_VARIANTS))
def test_probe_local_variant_matches_storage_checker(kernel):
    """The Open-Local family against the checker on the oracle with Open-Local: replicas, VG sums and each probe's VG and device state."""
    import checkers
    from oracle.binding import Oracle
    cs, t, big = PROBE_LOCAL_VARIANTS[kernel]
    seed = 61 + sorted(PROBE_LOCAL_VARIANTS).index(kernel)
    c = make_mixed_local(seed, n_nodes=120, n_workloads=30, max_replicas=8)[1]
    st = c.storage
    o = Oracle(c, open_local=True)
    placed = o.schedule()[0]
    rng = np.random.default_rng(seed)
    qs = _probe_pods(c, rng, 40)
    loc = [q for q in qs if st.class_local[int(c.pods["pod_class"][q])]][:6]
    plain = [q for q in qs if not st.class_local[int(c.pods["pod_class"][q])]][:4]
    assert loc
    probes = [(q, int(rng.integers(1, 30))) for q in loc + plain]
    for static_cache in (True, False):
        with _engine(c, record_scores=True, cluster_ctas=cs, threads_per_cta=t, force_large=big, static_cache=static_cache) as eng:
            got = eng.probe_run(placed, probes)
            li = eng.last_launch()
            assert li["kernel"] == kernel and li["local"] and li["large"] == big, li
            states = [eng.scenario_storage_state(i) for i in range(len(probes))]
        for (q, r), g, (bvg, bdev) in zip(probes, got, states):
            want = checkers.probe(o, placed, q, r)
            _assert_probe_equal(g, want, f"{kernel} pod {q}")
            vg, dev = o.storage_state()
            np.testing.assert_array_equal(bvg, vg, err_msg=f"pod {q}: VG state")
            if dev is not None:
                np.testing.assert_array_equal(bdev, dev, err_msg=f"pod {q}: device state")
            req = sum(int(vg[:int(st.node_n_vg[x]), x].sum()) for x in range(c.n_nodes) if st.node_n_vg[x] >= 0)
            assert g["vg_requested"] == req
    o.close()


def _resume_with_copies(p, c, placed, q, R, open_local=False, scs=None):
    """The equivalence that pins a probe: the pod list with R copies of pod q appended, resumed with `placed` as the prefix.
    -> (out_node of the copies, their GPU slot words, failures (counts, pods), VG state, device state, n_pods before the copies)."""
    pods = list(p.pods) + [copy.copy(p.pods[q]) for _ in range(R)]
    c2 = compile_cluster(p.nodes, pods, p.ctx, open_local=open_local, storage_classes=scs, local_devices=open_local)
    with _engine(c2) as eng:
        out, _s, fc, fp = eng.schedule_resume(placed)
        slots = eng.gpu_slot_words()
        vg = eng.storage_state() if open_local else None
        dev = eng.device_state() if open_local and c2.storage.devices else None
    P = len(p.pods)
    return out[P:], slots[P:], fc, fp, vg, dev, P


def _check_equivalence(p, c, placed, probes, open_local=False, scs=None):
    with _engine(c) as eng:
        got = eng.probe_run(placed, probes)
        states = [eng.scenario_storage_state(i) for i in range(len(probes))] if open_local else None
    for j, ((q, R), g) in enumerate(zip(probes, got)):
        out, slots, fc, fp, vg, dev, P = _resume_with_copies(p, c, placed, q, R, open_local, scs)
        k = g["n_placed"]
        np.testing.assert_array_equal(out[:k], g["node"], err_msg=f"pod {q}")
        np.testing.assert_array_equal(slots[:k], g["gpu_slots"], err_msg=f"pod {q}")
        assert (out[k:] == -1).all(), q                              # the copy after the last placed one and every later copy fail
        if k < R:
            assert fp[0] == P + k, q
            np.testing.assert_array_equal(fc[0], g["fail_counts"], err_msg=f"pod {q}")
        if open_local:
            np.testing.assert_array_equal(states[j][0], vg, err_msg=f"pod {q}: VG state")
            if dev is not None:
                np.testing.assert_array_equal(states[j][1], dev, err_msg=f"pod {q}: device state")
    return got


def test_probes_equal_recompile_and_resume_gpu_share():
    cluster, apps = synth.make_c3(n_nodes=600, n_workloads=80, replicas=20, n_apps=2, gpu_pct=25, seed_no=9)
    p = simulator.plan(cluster, apps)
    c = compile_cluster(p.nodes, p.pods, p.ctx)
    with _engine(c) as eng:
        placed = eng.schedule()[0]
    rng = np.random.default_rng(3)
    from simon_b200.compiler import SCW_GPU_MEM
    off, blob, cls = c.pods["class_off"], c.pods["class_blob"], c.pods["pod_class"]
    qs = _probe_pods(c, rng, 200)
    gpu = [q for q in qs if blob[off[cls[q]] + SCW_GPU_MEM] > 0][:4]
    probes = [(q, 300) for q in gpu] + [(q, int(rng.integers(1, 60))) for q in qs[:4]]
    got = _check_equivalence(p, c, placed, probes)
    assert any((g["gpu_slots"] != 0).any() for g in got)


def test_probes_equal_recompile_and_resume_mix_and_open_local():
    rng = np.random.default_rng(8)
    for seed in (1, 4):
        cluster, apps = synth.make_mix(seed_no=seed, n_nodes=40)
        p = simulator.plan(cluster, apps)
        c = compile_cluster(p.nodes, p.pods, p.ctx)
        with _engine(c) as eng:
            placed = eng.schedule()[0]
        _check_equivalence(p, c, placed, _probes(c, placed, rng, 8))
    p, c, (scs, _devices) = make_mixed_local(12, n_nodes=60, n_workloads=24, max_replicas=6)
    with _engine(c) as eng:
        placed = eng.schedule()[0]
    _check_equivalence(p, c, placed, _probes(c, placed, rng, 8), open_local=True, scs=scs)


def test_first_replica_fails_and_chunks_equal_one_batch():
    cluster, apps, ref, *_ = _case("cpu")
    p = simulator.plan(cluster, apps)
    c = compile_cluster(p.nodes, p.pods, p.ctx)
    with _engine(c, record_scores=True) as eng:
        placed = eng.schedule()[0]
        full = eng.probe_run(placed, [(0, 20)])[0]
        assert full["n_placed"] == 8
        # the live state is full after 8 more: a probe from the state with them has nowhere to go
        fuller = np.concatenate([placed, full["node"]])
    pods = list(p.pods) + [copy.copy(p.pods[0]) for _ in range(8)]
    c2 = compile_cluster(p.nodes, pods, p.ctx)
    with _engine(c2) as eng:
        g = eng.probe_run(fuller, [(3, 5)])[0]
        assert g["n_placed"] == 0 and g["stop_reason"] == abi.PROBE_STOP_UNSCHEDULABLE and len(g["node"]) == 0
        assert int(g["fail_counts"][abi.SFC_CPU]) == 4
    cluster, apps = synth.make_mix(seed_no=6, n_nodes=40)
    p = simulator.plan(cluster, apps)
    c = compile_cluster(p.nodes, p.pods, p.ctx)
    with _engine(c, record_scores=True) as eng:
        placed = eng.schedule()[0]
        probes = _probes(c, placed, np.random.default_rng(2), 11)
        one = eng.probe_run(placed, probes)
        assert eng.last_probe["chunks"] == 1
        parts = eng.probe_run(placed, probes, chunk=3)
        assert eng.last_probe["chunks"] == 4
    for a, b in zip(one, parts):
        _assert_probe_equal(a, b, "chunked")
        assert all(a[k] == b[k] for k in ("req_mcpu", "alloc_mcpu", "req_mem", "alloc_mem"))


def test_context_state_after_a_probe_batch_and_cross_refusals():
    from simon_b200.engine import lib
    cluster, apps = synth.make_mix(seed_no=3, n_nodes=40)
    p = simulator.plan(cluster, apps)
    c = compile_cluster(p.nodes, p.pods, p.ctx)
    L = lib()
    with _engine(c) as eng:
        placed = eng.schedule()[0]
        st, ext, slots = eng.state(), eng.state_ext(), eng.gpu_slot_words()
        probes = _probes(c, placed, np.random.default_rng(1), 4)
        eng.probe_run(placed, probes)
        for k, v in eng.state().items():                            # the single-scenario state describes `placed`
            assert np.array_equal(v, st[k]), k
        for k, v in eng.state_ext().items():
            assert np.array_equal(v, ext[k]), k
        assert np.array_equal(eng.gpu_slot_words(), slots)
        node = np.zeros(64, np.int32)
        assert L.simon_probe_download(eng.h, 0, node.ctypes.data, None, None, None) == 0
        assert L.simon_drain_download(eng.h, 0, *([None] * 7)) == ERR_STATE
        order = scaledown.NodeOrder(c)
        eng.drain_run(placed, [order.remaining([0])])
        assert L.simon_probe_download(eng.h, 0, node.ctypes.data, None, None, None) == ERR_STATE
        assert L.simon_drain_download(eng.h, 0, *([None] * 7)) == 0
        eng.probe_run(placed, probes)
        assert L.simon_drain_download(eng.h, 0, *([None] * 7)) == ERR_STATE
        assert L.simon_scenarios_storage_download(eng.h, 0, None, None) == ERR_STATE       # no storage uploaded
        eng.reset()                                                  # a single run from the empty state places as before
        assert np.array_equal(eng.schedule()[0], placed)
        assert eng.last_launch()["kernel"].startswith("simon_place_kernel_")


def test_c_entry_refusals():
    from simon_b200.engine import lib
    cluster, apps = synth.make_mix(seed_no=0, n_nodes=30)
    p = simulator.plan(cluster, apps)
    c = compile_cluster(p.nodes, p.pods, p.ctx)
    L = lib()
    guard = scaledown.pod_guard(c)
    fixed = c.pods["pod_fixed_node"]
    P = c.pods_dims["n_pods"]
    pinned = int(np.nonzero(guard >= 0)[0][0])
    bound = int(np.nonzero(fixed >= 0)[0][0])
    ok = _probe_pods(c, np.random.default_rng(0), 1)[0]
    with _engine(c) as eng:
        placed = eng.schedule()[0]
        res = (abi.SimonProbeResult * 1)()
        loc = (abi.SimonScenarioLocalResult * 1)()

        def run(q, r, pl=placed, out_local=None):
            arr = (abi.SimonProbe * 1)(abi.SimonProbe(q, r))
            rc = L.simon_probe_run(eng.h, np.ascontiguousarray(pl, np.int32).ctypes.data, arr, 1, res, out_local)
            return rc, (L.simon_last_error(eng.h) or b"").decode()
        for q, r, msg in ((P, 1, "out of range"), (pinned, 1, "pinned class"), (bound, 1, "spec.nodeName"), (ok, 0, "max_replicas is 0")):
            rc, m = run(q, r)
            assert rc == ERR_INVALID and msg in m, (q, r, m)
        bad = placed.copy()
        bad[ok] = c.n_nodes + 3
        rc, m = run(ok, 1, pl=bad)
        assert rc == ERR_INVALID and "out of range" in m
        rc, m = run(ok, 1, out_local=loc)
        assert rc == ERR_STATE and "out_local" in m
        assert eng.last_launch()["kernel"].startswith("simon_place_kernel_")        # nothing was launched by a refused call
        assert run(ok, 2)[0] == 0 and eng.last_launch()["kernel"].startswith("simon_probe_kernel_")
        c.class_pod_limit = [P] * len(c.class_pod_limit)                            # Engine.probe_run's refusal, on the host
        with pytest.raises(RuntimeError, match="int32 bounds"):
            eng.probe_run(placed, [(ok, 1)])


def test_session_headroom_on_the_reference_example():
    from simon_b200.objects import AppResource, create_cluster_resource_from_cluster_config, get_object_from_yaml_content, \
        get_yaml_content_from_directory
    cluster = create_cluster_resource_from_cluster_config(os.path.join(EXAMPLE, "cluster", "demo_1"))
    app = AppResource("simple", get_object_from_yaml_content(get_yaml_content_from_directory(os.path.join(EXAMPLE, "application", "simple"))))
    with simulator.NewSimulator() as sim:
        sim.RunCluster(simulator.PrepareCluster(cluster))
        sim.ScheduleApp(app)
        before = (sim.placements.copy(), sim.engine, sim.compiled)
        kinds = {(r.tmpl.workload_kind, r.tmpl.workload_namespace, r.workload_name) for r in sim.compiled.pod_recs
                 if r.tmpl.workload_kind not in ("DaemonSet", "Pod")}
        refs = sorted(f"{k}/{ns}/{n}" for k, ns, n in kinds)[:4]
        tmpl = {"apiVersion": "v1", "kind": "Pod", "metadata": {"name": "probe", "namespace": "default", "labels": {"app": "probe"}},
                "spec": {"containers": [{"name": "c", "image": "x", "resources": {"requests": {"cpu": "500m", "memory": "512Mi"}}}]}}
        res = sim.Headroom(refs + [tmpl])
        assert [r.Probe for r in res] == refs + ["Pod/default/probe"]
        free = headroom.free_pod_slots(sim.compiled, sim.placements)
        for r in res:
            assert r.Stopped in ("Unschedulable", "MaxReplicas") and len(r.Nodes) == r.Replicas <= free
            assert (r.Reason is not None) == (r.Stopped == "Unschedulable")
            if r.Reason:
                assert "nodes are available" in r.Reason
        capped = sim.Headroom(refs[:1], max_replicas=1)[0]
        assert capped.Replicas <= 1
        assert np.array_equal(sim.placements, before[0]) and sim.engine is before[1] and sim.compiled is before[2]
        with pytest.raises(ValueError, match="no workload"):
            sim.Headroom(["Deployment/default/none"])
        with pytest.raises(ValueError, match="at least 1"):
            sim.Headroom(refs[:1], max_replicas=0)
        with pytest.raises(ValueError, match="spec.nodeName"):
            sim.Headroom([dict(tmpl, spec=dict(tmpl["spec"], nodeName="x"))])
        drained = sim.DrainNodes([[sim.compiled.node_names[0]]])
        assert len(drained) == 1
    res2 = headroom.estimate(cluster, [app], refs[:2])
    assert [(r.Replicas, r.Nodes) for r in res2] == [(r.Replicas, r.Nodes) for r in res[:2]]
