"""GPU parity: the CUDA engine (through the C ABI) must reproduce the oracle bit for bit."""
import numpy as np
import pytest

from util import assert_ext_equal, make_case, run_oracle, run_oracle_ext

pytestmark = pytest.mark.gpu


def _engine(c, **kw):
    from simon_b200.engine import Engine
    return Engine(c, device=0, record_scores=True, **kw)


CASES = [
    ("c2", dict(n_nodes=100, n_workloads=20, replicas=10, seed_no=2)),
    ("c2", dict(n_nodes=1000, n_workloads=100, replicas=100, seed_no=2)),
    ("c3", dict(n_nodes=60, n_workloads=40, replicas=8, n_apps=2, seed_no=3)),
    ("c3", dict(n_nodes=300, n_workloads=100, replicas=10, n_apps=2, seed_no=21)),
    ("c3", dict(n_nodes=1500, n_workloads=200, replicas=20, n_apps=4, seed_no=5)),
    ("c3", dict(n_nodes=3000, n_workloads=300, replicas=30, n_apps=3, seed_no=9)),
]


@pytest.mark.parametrize("kind,kw", CASES)
def test_parity_with_oracle(kind, kw):
    p, c = make_case(kind, **kw)
    (ref, rscore, rfc, rfp), rstate = run_oracle(c)
    with _engine(c) as eng:
        out, score, fc, fp = eng.schedule()
        st = eng.state()
    bad = np.nonzero(out != ref)[0]
    assert len(bad) == 0, f"first mismatches at pods {bad[:5]}: gpu {out[bad[:5]]} oracle {ref[bad[:5]]}"
    sched = ref >= 0
    np.testing.assert_array_equal(score[sched & (rscore > 0)], rscore[sched & (rscore > 0)])
    np.testing.assert_array_equal(fp, rfp)
    np.testing.assert_array_equal(fc, rfc)
    for k in rstate:
        np.testing.assert_array_equal(st[k], rstate[k], err_msg=k)


@pytest.mark.parametrize("seed", [100, 101, 102, 103, 206, 209, 212, 215, 219, 223, 228, 238])
def test_parity_mixed_features(seed):
    """synth.make_mix: every predicate / score input in random combination (see tests/test_oracle_cpu.py), incl. GPU share,
    host ports, extended resources, hard spread constraints, required pod affinity, DaemonSets and pre-bound pods."""
    p, c = make_case("mix", seed_no=seed, n_nodes=20 + (seed % 5) * 25, n_workloads=20 + (seed % 7) * 10, max_replicas=4 + seed % 6)
    (ref, rscore, rfc, rfp), rstate, rext, rslots = run_oracle_ext(c)
    with _engine(c) as eng:
        out, score, fc, fp = eng.schedule()
        st = eng.state()
        assert_ext_equal(eng, rext, rslots)
    np.testing.assert_array_equal(out, ref)
    sched = ref >= 0
    np.testing.assert_array_equal(score[sched & (rscore > 0)], rscore[sched & (rscore > 0)])
    np.testing.assert_array_equal(fp, rfp)
    np.testing.assert_array_equal(fc, rfc)
    for k in rstate:
        np.testing.assert_array_equal(st[k], rstate[k], err_msg=k)


@pytest.mark.parametrize("cs,tpb", [(1, 256), (2, 128), (4, 64), (8, 128), (16, 64), (16, 320), (4, 320), (9, 96), (5, 160), (3, 320)])
def test_parity_cluster_geometries(cs, tpb):
    p, c = make_case("c3", n_nodes=700, n_workloads=80, replicas=12, n_apps=2, seed_no=13)
    (ref, _, rfc, _), _ = run_oracle(c)
    with _engine(c, cluster_ctas=cs, threads_per_cta=tpb) as eng:
        out, _, fc, _ = eng.schedule()
    np.testing.assert_array_equal(out, ref)
    np.testing.assert_array_equal(fc, rfc)


def test_incremental_calls_match_single_call():
    p, c = make_case("c3", n_nodes=400, n_workloads=60, replicas=10, n_apps=2, seed_no=17)
    (ref, _, _, _), _ = run_oracle(c)
    P = len(ref)
    with _engine(c) as eng:
        a, _, _, _ = eng.schedule(0, P // 3)
        b, _, _, _ = eng.schedule(P // 3, P - P // 3)
    np.testing.assert_array_equal(np.concatenate([a, b]), ref)


def test_full_size_c3_properties():
    """BASELINE.json's 10k-node x 100k-pod configuration: size-independent properties + EVERY decision against the oracle."""
    from oracle.binding import Oracle
    p, c = make_case("c3", n_nodes=10000, n_workloads=1000, replicas=100, n_apps=10, seed_no=3)
    with _engine(c) as eng:
        out, score, fc, fp = eng.schedule()
        st = eng.state()
        eng.reset()
        out2, _, fc2, fp2 = eng.schedule()
    # idempotence: a second pass from the empty state reproduces every placement and every failure histogram
    np.testing.assert_array_equal(out, out2)
    np.testing.assert_array_equal(fc, fc2)
    # accounting: NodeInfo aggregates equal the sum over placed pods, and no node is over-committed
    cls = c.pods["pod_class"]
    blob, off = c.pods["class_blob"], c.pods["class_off"]
    req = np.array([[blob[int(off[k]) + w] for w in (0, 1, 2)] for k in range(c.pods_dims["n_classes"])], dtype=np.int64)
    placed = out >= 0
    for col, name in enumerate(["req_mcpu", "req_mem", "req_eph"]):
        agg = np.zeros(c.n_nodes, np.int64)
        np.add.at(agg, out[placed], req[cls[placed], col])
        np.testing.assert_array_equal(agg, st[name], err_msg=name)
    assert (st["req_mcpu"] <= c.snap["alloc_mcpu"]).all() and (st["req_mem"] <= c.snap["alloc_mem"]).all()
    assert (st["num_pods"] <= c.snap["alloc_pods"]).all()
    assert int(st["num_pods"].sum()) == int(placed.sum())
    # every unschedulable pod has a complete reason histogram (one or more reasons per node)
    assert len(fp) == int((out == -1).sum())
    assert (fc.sum(axis=1) >= c.n_nodes).all()
    # EVERY decision of the headline configuration against the oracle (16 host threads: placements do not depend on the
    # thread count, tests/test_oracle_cpu.py), including the late, crowded-cluster regime where feasibility flips, the
    # single-node fast path and the summary restores fire most
    import os
    o = Oracle(c, threads=min(16, len(os.sched_getaffinity(0))))
    ref, rscore, rfc, rfp = o.schedule()
    bad = np.nonzero(out != ref)[0]
    assert len(bad) == 0, f"{len(bad)} mismatches, first at pods {bad[:5]}: gpu {out[bad[:5]]} oracle {ref[bad[:5]]}"
    sched = ref >= 0
    np.testing.assert_array_equal(score[sched & (rscore > 0)], rscore[sched & (rscore > 0)])
    np.testing.assert_array_equal(fp, rfp)
    np.testing.assert_array_equal(fc, rfc)
    rst = o.state()
    for k in rst:
        np.testing.assert_array_equal(st[k], rst[k], err_msg=k)


def _cmp(c):
    """Placements, every scheduled pod's score (zeros included: a pod with one feasible node is not scored), failure records
    and state() against the oracle."""
    (ref, rscore, rfc, rfp), rstate = run_oracle(c)
    with _engine(c) as eng:
        out, score, fc, fp = eng.schedule()
        st = eng.state()
        li = eng.last_launch()
    np.testing.assert_array_equal(out, ref)
    np.testing.assert_array_equal(score[ref >= 0], rscore[ref >= 0])
    np.testing.assert_array_equal(fp, rfp)
    np.testing.assert_array_equal(fc, rfc)
    for k in rstate:
        np.testing.assert_array_equal(st[k], rstate[k], err_msg=k)
    return out, li


def test_edge_empty_pod_list():
    from simon_b200 import simulator, synth
    from simon_b200.compiler import compile_cluster
    cluster, apps = synth.make_c2(n_nodes=5, n_workloads=0, replicas=1)
    p = simulator.plan(cluster, apps)
    c = compile_cluster(p.nodes, p.pods, p.ctx)
    assert len(_cmp(c)[0]) == 0


def test_edge_single_node_fills_up():
    p, c = make_case("c2", n_nodes=1, n_workloads=3, replicas=50, seed_no=2)
    out = _cmp(c)[0]
    assert (out == 0).sum() > 0 and (out == -1).sum() > 0        # F == 1 short-circuit, then "Insufficient ..." for the rest


def test_edge_no_nodes():
    p, c = make_case("c2", n_nodes=0, n_workloads=2, replicas=2, seed_no=2)
    out = _cmp(c)[0]
    assert (out == -1).all()


def test_edge_zero_count_and_tail_calls():
    p, c = make_case("c3", n_nodes=40, n_workloads=10, replicas=4, n_apps=1, seed_no=4)
    (ref, _, _, _), _ = run_oracle(c)
    P = c.pods_dims["n_pods"]
    with _engine(c) as eng:
        o0 = eng.schedule(0, 0)[0]
        a = eng.schedule(0, P - 1)[0]
        b = eng.schedule(P - 1, 1)[0]
    assert len(o0) == 0
    np.testing.assert_array_equal(np.concatenate([a, b]), ref)


def test_large_cluster_variant_40k_nodes():
    """A scenario that does not fit the cluster's shared memory (40,000 nodes; round 1 refused it) runs on the large-cluster
    variant - the same kernel with its per-node arrays in global memory - and reproduces the oracle bit for bit, scores included."""
    p, c = make_case("c3", n_nodes=40000, n_workloads=60, replicas=20, n_apps=2, seed_no=7)
    out, li = _cmp(c)
    assert (out >= 0).sum() > 1000
    assert li["large"] and li["node_slots"] == 8, li


def test_limit_too_many_nodes_is_an_error_not_a_fallback():
    """Beyond 16 CTAs x 320 threads x 64 node slots the engine refuses with a message (there is no CPU path)."""
    from simon_b200 import simulator, synth
    from simon_b200.compiler import compile_cluster
    cluster, apps = synth.make_c2(n_nodes=330000, n_workloads=1, replicas=1, seed_no=2)
    p = simulator.plan(cluster, apps)
    c = compile_cluster(p.nodes, p.pods, p.ctx)
    with _engine(c) as eng:
        with pytest.raises(RuntimeError, match="engine limit|exceeds"):
            eng.schedule()
