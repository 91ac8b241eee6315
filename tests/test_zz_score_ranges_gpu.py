"""The device on the score-range cases of test_score_ranges.py, against the C oracle.

Per case: the per-node totals and filter verdicts of the first pods of the scored workload (Engine.dump_pod); full runs on three
placement-kernel variants, each at an explicit geometry and asserted with last_launch() (unrolled node slots, a run-time slot
count, the large-cluster variant), compared in placements, recorded winning scores, failure records and state(); and every
NodeAffinity and spread case once more as a scenario batch and as drains, which instantiate the same body separately.
Move scoring (LeastAllocated / BalancedAllocation of the source and target nodes) on the adversarial BalancedAllocation and
LeastAllocated shapes of test_gpu_detail.py: every pod onto every node, gain and code per move against the move checker.
"""
import functools

import numpy as np
import pytest

from test_gpu_detail import _ba_adversarial_caps, _check_pod
from test_score_ranges import CASES, NA_CASES, PTS_CASES, build, pods_of

pytestmark = pytest.mark.gpu

# (CTAs per scenario, threads per CTA, force_large) -> the kernel it launches on the 160-node cases
GEOMS = {"unrolled": ((2, 96, False), "simon_place_kernel_256_1"),
         "runtime_slots": ((1, 32, False), "simon_place_kernel_256_0"),
         "large": ((2, 64, True), "simon_place_kernel_big")}


@functools.lru_cache(maxsize=None)
def case(name):
    return build(name)


@functools.lru_cache(maxsize=None)
def oracle_full(name):
    from oracle.binding import Oracle
    _p, c = case(name)
    o = Oracle(c)
    res = o.schedule() + (o.state(),)
    o.close()
    return res


@pytest.mark.parametrize("name", sorted(CASES))
def test_per_node_totals_match_oracle(name):
    _p, c = case(name)
    for pod in pods_of(c, "a")[:4]:
        _check_pod(c, pod)


@pytest.mark.parametrize("geom", sorted(GEOMS))
@pytest.mark.parametrize("name", sorted(CASES))
def test_full_run_matches_oracle(name, geom):
    from simon_b200.engine import Engine
    _p, c = case(name)
    (cs, t, big), kernel = GEOMS[geom]
    ref, rscore, rfc, rfp, rst = oracle_full(name)
    with Engine(c, device=0, record_scores=True, cluster_ctas=cs, threads_per_cta=t, force_large=big) as eng:
        out, score, fc, fp = eng.schedule()
        li = eng.last_launch()
        assert li["kernel"] == kernel and (li["cluster_ctas"], li["threads_per_cta"]) == (cs, t), li
        st = eng.state()
    bad = np.nonzero(out != ref)[0]
    assert len(bad) == 0, f"{name} {geom}: {len(bad)} mismatches, first at pods {bad[:5]}: gpu {out[bad[:5]]} oracle {ref[bad[:5]]}"
    sched = ref >= 0
    np.testing.assert_array_equal(score[sched], rscore[sched], err_msg=f"{name} {geom}: winning scores")
    np.testing.assert_array_equal(fp, rfp, err_msg=name)
    np.testing.assert_array_equal(fc, rfc, err_msg=name)
    for k in rst:
        np.testing.assert_array_equal(st[k], rst[k], err_msg=f"{name} {geom}: {k}")


@pytest.mark.parametrize("name", NA_CASES + PTS_CASES)
def test_scenario_batch_matches_oracle(name):
    from oracle.binding import Oracle
    from simon_b200.engine import Engine
    _p, c = case(name)
    n = c.n_nodes
    lists = [np.arange(n), np.arange(0, n, 2), np.arange(n)[::-1][: (2 * n) // 3].copy(),
             np.random.default_rng(5).permutation(n)[: (4 * n) // 5]]
    with Engine(c, device=0) as eng:
        res, nodes = eng.run_scenarios(lists, want_nodes=True)
        assert eng.last_launch()["n_scenarios"] == len(lists)
    o = Oracle(c)
    for i, act in enumerate(lists):
        o.set_active(act)
        o.reset()
        ref = o.schedule()[0]
        np.testing.assert_array_equal(nodes[i], ref, err_msg=f"{name} scenario {i}")
        assert res[i]["n_unscheduled"] == int((ref == -1).sum()), i
    o.close()


@pytest.mark.parametrize("name", NA_CASES + PTS_CASES)
def test_drains_match_checker(name):
    import checkers
    from oracle.binding import Oracle
    from simon_b200 import scaledown
    from simon_b200.engine import Engine
    from test_drain import _assert_drain_equal
    _p, c = case(name)
    o = Oracle(c)
    placed = o.schedule()[0]
    order = scaledown.NodeOrder(c)
    used = sorted({int(g) for g in placed if g >= 0})
    drains = [[used[0]], [used[-1]], used[: len(used) // 2], used]
    remain = [order.remaining(d) for d in drains]
    with Engine(c, device=0, record_scores=True) as eng:
        got = eng.drain_run(placed, remain)
    for d, rl, g in zip(drains, remain, got):
        want = checkers.drain(o, placed, rl)
        _assert_drain_equal(g, want, f"{name} drain {d}")
        pos = g["node"] >= 0
        assert pos.any() and np.array_equal(g["score"][pos], want["score"][pos]), d
    o.close()


def _cluster(caps, pods):
    """Nodes of (mCPU, bytes) capacities and plain pods of (mCPU, bytes) requests, compiled."""
    from simon_b200 import simulator
    from simon_b200.compiler import compile_cluster
    from simon_b200.objects import AppResource, ResourceTypes
    cluster = ResourceTypes()
    for i, (capc, capm) in enumerate(caps):
        cluster.Nodes.append({"kind": "Node", "metadata": {"name": f"n{i:04d}", "labels": {"kubernetes.io/hostname": f"n{i:04d}"}},
                              "spec": {}, "status": {"allocatable": {"cpu": f"{capc}m", "memory": str(capm), "pods": "110"}}})
    app = AppResource("a", ResourceTypes())
    for j, (rc, rm) in enumerate(pods):
        app.Resource.Pods.append({"kind": "Pod", "metadata": {"name": f"p{j}", "namespace": "default"},
                                  "spec": {"containers": [{"name": "c", "image": "x", "resources": {"requests": {"cpu": f"{rc}m", "memory": str(rm)}}}]}})
    p = simulator.plan(cluster, [app])
    return compile_cluster(p.nodes, p.pods, p.ctx)


def _ba_moves_cluster(req_c, req_mi):
    req_m = req_mi * 1024 * 1024
    caps = _ba_adversarial_caps(req_c, req_m, 200)
    assert len(caps) >= 50
    return _cluster(caps, [(req_c, req_m)] * 3)


def _la_moves_cluster():
    rng = np.random.RandomState(5)
    caps = [(int(rng.randint(1000, 2000000)), int(rng.randint(1, 1 << 30)) * (1 << 25) + int(rng.randint(0, 1 << 20))) for _ in range(256)]
    return _cluster(caps, [(500, (1 << 40) + 12345), (999, (1 << 52) + 1), (100, 3)])


MOVE_SHAPES = {"ba_300_768": lambda: _ba_moves_cluster(300, 768), "ba_700_1536": lambda: _ba_moves_cluster(700, 1536),
               "ba_1000_1000": lambda: _ba_moves_cluster(1000, 1000), "la_beyond_2_pow_52": _la_moves_cluster}


@pytest.mark.parametrize("shape", sorted(MOVE_SHAPES))
def test_move_scoring_on_adversarial_shapes(shape):
    """Every placed pod onto every node: the move kernel's gain (LeastAllocated + BalancedAllocation of both nodes, smv_la /
    smv_own) and code against simon_oracle_moves_score, on nodes whose BalancedAllocation sits on / next to an integer or
    whose (capacity - requested) x 100 is far above 2^52."""
    from oracle.binding import Oracle
    from test_moves_scope import _engine_vs_checker
    c = MOVE_SHAPES[shape]()
    o = Oracle(c)
    out = o.schedule()[0]
    assert (out >= 0).all()
    mv = np.array([(q, g) for q in range(len(out)) for g in range(c.n_nodes)], np.uint32)
    code = _engine_vs_checker(c, o, out, mv, 0)
    o.close()
    assert (code == 0).sum() > c.n_nodes
