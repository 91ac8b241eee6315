"""Explained decisions (simon_explain_kernel_*) and headroom probes (simon_probe_kernel_*) at the engine limits, the score-range edges
and past 65,536 nodes, against the CPU checkers (explain_oracle.expected, checkers.probe), exactly.

A. Every builder of test_engine_limits.py, every pod explained at top_k 16 (15 extra max-reductions per decision) on the geometries
   of test_explain_probe_edges.limit_geoms, and without the static-verdict cache on three of them; one run at top_k 1.
B. Every case of test_score_ranges.py the same way on test_zz_score_ranges_gpu's geometries; the adversarial BalancedAllocation and
   LeastAllocated shapes (words 0 and 1 of own_core's parts); extra_max with a total past 2^31 - 1.
C. zone_case(65537, 20, 3) with hand-derived records (counts past 16 bits), and the 70,000-node C3 in the engine's own geometry.
D. Simulator.Explain on an Open-Local session (simon_explain_local_kernel_*, word 9).
E. Probes of the workloads that carry each builder's limit and of each score-range case's scored workload, and a probe that runs
   a class's InterPodAffinity score up to its int32 guard (class_pod_limit), with the recompile-and-resume equivalence.

Each run equals the same run without the explained set (placements, scores, failure records, state(), state_ext(), GPU slots), an
unschedulable pod's histogram is its failure record, explain.build accepts every record with more than one listed node, and every
launch is asserted with last_launch(): kernel, geometry and node slots per thread."""
import copy

import numpy as np
import pytest

from explain_oracle import assert_records_equal, expected
from simon_b200 import abi, explain, headroom, scaledown
from simon_b200.compiler import CompileError, compile_cluster
from test_explain_probe_edges import (BOUND_W, EXPLAIN_BUILDERS, EXPLAIN_CASES, LIMIT_PROBES, NO_STATIC_CACHE, PROBE_CASES,
                                      PROBE_REFUSED, RANGE_GEOMS, assert_wrap_records, bound_case, bound_limit, limit_geoms, wrap_case)
from test_score_ranges import CASES, pods_of
from test_zz_engine_limits_gpu import case as limit_case
from test_zz_explain_gpu import _assert_rejected_is_fail_record, _assert_same_run, _run
from test_zz_headroom_gpu import _assert_probe_equal, _probe_pods, _resume_with_copies
from test_zz_kernel_variants_gpu import _engine
from test_zz_large_cluster_gpu import THREADS, family_case
from test_zz_score_ranges_gpu import MOVE_SHAPES, case as range_case

pytestmark = pytest.mark.gpu
TOP = abi.EXPLAIN_MAX_TOP
I32_MAX = (1 << 31) - 1


def _geom(g):
    return (0, 0, False) if g is None else g


def _assert_launch(li, family, suffix, geom, n_nodes, what=""):
    """The launch ran simon_<family>_kernel_<suffix> at the forced geometry (if any), with ceil(nodes / threads) node slots."""
    assert li["kernel"] == f"simon_{family}_kernel_{suffix}", (what, li)
    assert li["n_nodes"] == n_nodes, (what, li)
    if geom is not None:
        assert (li["cluster_ctas"], li["threads_per_cta"], li["large"]) == geom, (what, li)
    assert li["node_slots"] == -(-n_nodes // (li["cluster_ctas"] * li["threads_per_cta"])), (what, li)


def _rows(rec, nodes, i):
    return [(int(x["node"]), [int(v) for v in x["words"]]) for x in nodes[i][:int(rec[i]["n_top"])]]


def _explain_run(c, geom, want, pods, what, plugins=None, **kw):
    """Every pod of `pods` explained at top_k 16 against `want`, and the run equal to the same run without the set.
    -> (last launch, records, nodes)."""
    with _engine(c, *_geom(geom), record_scores=True, **kw) as eng:
        plain = _run(eng)
        eng.reset()
        got = _run(eng, explain=pods, top_k=TOP)
        li = eng.last_launch()
        rec, nodes = eng.explanations()
    _assert_same_run(got, plain, what)
    assert_records_equal(rec, nodes, want, pods, what)
    _assert_rejected_is_fail_record(rec, pods, got[2], got[3])
    built = 0
    for i in np.nonzero(rec["n_top"] > 1)[0]:
        explain.build(c, int(pods[i]), rec[i], nodes[i], plugins)
        built += 1
    assert built > 0, what
    return li, rec, nodes


# ---- A: explain at the engine limits --------------------------------------------------------------------------------------------

_WANT = {}


def _want_limit(name):
    if name not in _WANT:
        _p, c = limit_case(name)
        _WANT[name] = expected(c, np.arange(c.pods_dims["n_pods"], dtype=np.uint32), TOP, threads=THREADS)
    return _WANT[name]


@pytest.mark.parametrize("name", EXPLAIN_BUILDERS)
def test_explain_at_the_engine_limit(name):
    _p, c = limit_case(name)
    n = c.n_nodes
    pods = np.arange(c.pods_dims["n_pods"], dtype=np.uint32)
    want = _want_limit(name)
    runs = [(g, geom, suffix, {}) for g, (geom, suffix) in limit_geoms(name, n).items()]
    if name in NO_STATIC_CACHE:
        runs.append(("no static cache", None, "256", dict(static_cache=False)))
    for g, geom, suffix, kw in runs:
        what = f"{name} {g}"
        li, rec, _nodes = _explain_run(c, geom, want, pods, what, **kw)
        _assert_launch(li, "explain", suffix, geom, n, what)
        if g == "one_cta" and n > 32:
            assert li["node_slots"] >= 2, li
    F, k = rec["feasible"], rec["n_top"]
    assert (k == TOP).any() and ((F > 1) & (F < TOP)).any() and ((rec["node"] == -1) & (F == 0)).any(), name


def test_explain_top_1_runs_no_extra_round():
    """top_k 1: the arg-max alone, no extra max-reduction; the records are the top-16 checker's cut to one node."""
    name = "atoms1024"
    _p, c = limit_case(name)
    pods = np.arange(c.pods_dims["n_pods"], dtype=np.uint32)
    want = [dict(w, top=w["top"][:1]) for w in _want_limit(name)]
    with _engine(c, 0, 0, False, record_scores=True) as eng:
        plain = _run(eng)
        eng.reset()
        got = _run(eng, explain=pods, top_k=1)
        li = eng.last_launch()
        rec, nodes = eng.explanations()
    _assert_launch(li, "explain", "256", None, c.n_nodes)
    _assert_same_run(got, plain, "top_k 1")
    assert_records_equal(rec, nodes, want, pods, "top_k 1")
    assert (rec["feasible"] > 1).sum() > 100 and (rec["n_top"] <= 1).all()


# ---- B: explain at the score-range edges ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", EXPLAIN_CASES)
def test_explain_at_the_score_range_edge(name):
    _p, c = range_case(name)
    plugins = CASES[name][1]() if CASES[name][1] else None
    pods = np.arange(c.pods_dims["n_pods"], dtype=np.uint32)
    want = expected(c, pods, TOP, threads=THREADS)
    for g, (geom, suffix) in RANGE_GEOMS.items():
        li, rec, nodes = _explain_run(c, geom, want, pods, f"{name} {g}", plugins)
        _assert_launch(li, "explain", suffix, geom, c.n_nodes, f"{name} {g}")
    if name == "extra_max":
        totals = [w[8] for i in range(len(pods)) for _g, w in _rows(rec, nodes, i)]
        assert max(totals) > I32_MAX, max(totals)


@pytest.mark.parametrize("shape", sorted(MOVE_SHAPES))
def test_explain_on_the_adversarial_score_shapes(shape):
    """BalancedAllocation on / next to an integer, LeastAllocated with (capacity - requested) x 100 far above 2^52: words 0 and 1
    of every listed node (own_core's parts) equal the checker's.  On the BalancedAllocation shapes the first pod's listed nodes
    include one whose BalancedAllocation input lies within 1e-7 of an integer (own_core's exact fallback)."""
    c = MOVE_SHAPES[shape]()
    pods = np.arange(c.pods_dims["n_pods"], dtype=np.uint32)
    want = expected(c, pods, TOP, threads=THREADS)
    li, rec, nodes = _explain_run(c, None, want, pods, shape)
    _assert_launch(li, "explain", "256", None, c.n_nodes, shape)
    assert (rec["n_top"] == TOP).all()
    if shape.startswith("ba_"):
        req_c, req_mi = (int(x) for x in shape.split("_")[1:])
        x = [(1.0 - abs(req_c / int(c.snap["alloc_mcpu"][g]) - req_mi * 1024 * 1024 / int(c.snap["alloc_mem"][g]))) * 100.0
             for g, _w in _rows(rec, nodes, 0)]
        assert min(abs(v - round(v)) for v in x) < 1e-7, x


# ---- C: explain past 65,536 nodes -----------------------------------------------------------------------------------------------

def _assert_large(li, n_nodes):
    assert li["kernel"] == "simon_explain_kernel_big" and li["large"], li
    assert (li["cluster_ctas"], li["threads_per_cta"], li["node_slots"]) == (16, 320, -(-n_nodes // (16 * 320))), li


def test_explain_wrap_case_known_answers():
    c = wrap_case()
    pods = np.arange(3, dtype=np.uint32)
    with _engine(c, 0, 0, False, record_scores=True) as eng:
        plain = _run(eng)
        eng.reset()
        got = _run(eng, explain=pods, top_k=TOP)
        li = eng.last_launch()
        rec, nodes = eng.explanations()
    _assert_large(li, c.n_nodes)
    _assert_same_run(got, plain, "wrap")
    assert_wrap_records(c, rec, [_rows(rec, nodes, i) for i in range(3)])
    assert _assert_rejected_is_fail_record(rec, pods, got[2], got[3]) == 1
    assert_records_equal(rec, nodes, expected(c, pods, TOP, threads=THREADS), pods, "wrap")


def test_explain_c3_70000_every_pod():
    c = family_case("70k")
    P = c.pods_dims["n_pods"]
    with _engine(c, 0, 0, False, record_scores=True) as eng:
        plain = _run(eng)
        eng.reset()
        got = _run(eng, explain=np.arange(P, dtype=np.uint32), top_k=TOP)
        li = eng.last_launch()
        rec, nodes = eng.explanations()
    _assert_large(li, c.n_nodes)
    _assert_same_run(got, plain, "c3 70000")
    reached = np.nonzero(c.pods["pod_fixed_node"] == -1)[0]
    sample = np.sort(np.random.default_rng(5).choice(reached, 200, replace=False)).astype(np.uint32)
    assert_records_equal(rec[sample], nodes[sample], expected(c, sample, TOP, threads=THREADS), sample, "c3 70000")
    assert (rec["n_top"][sample] == TOP).sum() > 100


# ---- D: Simulator.Explain on an Open-Local session ------------------------------------------------------------------------------

def test_simulator_explain_open_local_session():
    from simon_b200.simulator import NewSimulator, PrepareCluster, WithOpenLocal
    from simon_b200.workloads import make_valid_pod_by_pod
    from test_zz_grow_gpu import _mixed_local
    cluster, apps = _mixed_local(11, 60)
    sim = NewSimulator(WithOpenLocal(devices=True))
    sim.RunCluster(PrepareCluster(cluster))
    sim.ScheduleApp(apps[0])
    c = sim.compiled
    before = (sim.placements.copy(), sim.gpu_slots.copy(), sim.scores.copy())
    cls = c.pods["pod_class"]
    # pods the scheduler places (no DaemonSet pods); those with volumes among the ones the session placed, so that most are scored
    reached = np.nonzero((c.pods["pod_fixed_node"] == -1) & (scaledown.pod_guard(c) == -1))[0]
    local = [int(q) for q in reached if c.storage.class_local[int(cls[q])] and sim.placements[q] >= 0]
    plain = [int(q) for q in reached if not c.storage.class_local[int(cls[q])]]
    rng = np.random.default_rng(4)
    qs = sorted(rng.choice(local, 7, replace=False).tolist() + rng.choice(plain, 5, replace=False).tolist())
    names = [f"{c.pod_recs[q].tmpl.namespace}/{c.pod_recs[q].name}" for q in qs]
    tq = next(q for q in reversed(qs) if c.storage.class_local[int(cls[q])] and c.pod_recs[q].tmpl.workload_kind == "ReplicaSet")
    tmpl = copy.deepcopy(c.pod_recs[tq].tmpl.pod)
    tmpl["metadata"] = dict(tmpl.get("metadata") or {}, name="probe-template", namespace="default")
    tmpl.get("spec", {}).pop("nodeName", None)
    res = sim.Explain(names + [tmpl], top=TOP)
    li = sim.engine.last_launch()
    assert li["kernel"].startswith("simon_explain_local_kernel_") and li["local"], li
    for a, b in zip(before, (sim.placements, sim.gpu_slots, sim.scores)):
        np.testing.assert_array_equal(a, b)

    def same(ex, w, cc):
        assert ex.Feasible == w["feasible"] and ex.Node == (cc.node_names[w["node"]] if w["node"] >= 0 else "")
        assert [(n.Name, n.Total) for n in ex.Nodes] == [(cc.node_names[g], wd[8]) for g, wd in w["top"]]
        if w["feasible"] > 1:
            for n, (_g, wd) in zip(ex.Nodes, w["top"]):
                assert {p: n.Scores[p] for p, _i, _wt in explain.PLUGINS} == {p: wt * wd[i] for p, i, wt in explain.PLUGINS}
        return sum(wd[9] != 0 for _g, wd in w["top"])

    want = expected(c, qs, TOP, open_local=True, threads=THREADS)
    n_ol = sum(same(ex, w, c) for ex, w in zip(res, want))
    assert n_ol > 0, "no listed node carries an Open-Local score"
    # the template: the session's pods, then the template as one more pending pod
    p = sim._plan()
    scs = list(sim.cluster.StorageClasss) + [sc for a in sim.apps for sc in a.Resource.StorageClasss]
    c2 = compile_cluster(p.nodes, p.pods + [make_valid_pod_by_pod(tmpl)], p.ctx, open_local=True, storage_classes=scs,
                         local_devices=True)
    same(res[-1], expected(c2, [len(p.pods)], TOP, open_local=True, threads=THREADS)[0], c2)
    sim.Close()


# ---- E: probes at the limits and edges ------------------------------------------------------------------------------------------

def _want_probes(c, placed, probes, open_local=False):
    """The checker's probes, with the occupancy sums the engine reports."""
    import checkers
    from oracle.binding import Oracle
    o = Oracle(c, threads=THREADS, open_local=open_local)
    out = []
    for q, r in probes:
        w = checkers.probe(o, placed, q, r)
        st = o.state()
        w["sums"] = (int(st["req_mcpu"].sum()), int(c.snap["alloc_mcpu"].sum()), int(st["req_mem"].sum()), int(c.snap["alloc_mem"].sum()))
        out.append(w)
    o.close()
    return out


def _run_probes(c, placed, probes, want, geom, suffix, what, **kw):
    with _engine(c, *_geom(geom), record_scores=True, **kw) as eng:
        got = eng.probe_run(placed, probes)
        for li in eng.last_probe["launches"]:
            _assert_launch(li, "probe", suffix, geom, c.n_nodes, what)
    for (q, r), g, w in zip(probes, got, want):
        _assert_probe_equal(g, w, f"{what}: pod {q} x {r}")
        assert (g["req_mcpu"], g["alloc_mcpu"], g["req_mem"], g["alloc_mem"]) == w["sums"], (what, q, r)
    return got


def _oracle_placed(c):
    from oracle.binding import Oracle
    o = Oracle(c, threads=THREADS)
    placed = o.schedule()[0]
    o.close()
    return placed


@pytest.mark.parametrize("name", EXPLAIN_BUILDERS)
def test_probes_at_the_engine_limit(name):
    """The first probe-able pod of each workload that carries the limit, then up to 5 more: R = the free pod slots (within the
    class's int32 bound) for every other probe, a small R for the rest."""
    _p, c = limit_case(name)
    placed = _oracle_placed(c)
    rng = np.random.default_rng(31)
    P, cls = c.pods_dims["n_pods"], c.pods["pod_class"]
    ok = (c.pods["pod_fixed_node"] == -1) & (scaledown.pod_guard(c) == -1)
    qs = [next(q for q in pods_of(c, wl) if ok[q]) for wl in LIMIT_PROBES[name]]
    qs += [q for q in _probe_pods(c, rng, 5 + len(qs)) if q not in qs][:5]
    free = headroom.free_pod_slots(c, placed)
    probes = []
    for j, q in enumerate(qs):
        room = c.class_pod_limit[int(cls[q])] - P
        probes.append((q, min(free, room) if j % 2 == 0 else min(int(rng.integers(1, 8)), room)))
    assert all(r >= 1 for _q, r in probes), probes
    want = _want_probes(c, placed, probes)
    runs = [(g, geom, suffix, {}) for g, (geom, suffix) in limit_geoms(name, c.n_nodes).items()]
    runs.append(("no static cache", None, "256", dict(static_cache=False)))
    for g, geom, suffix, kw in runs:
        _run_probes(c, placed, probes, want, geom, suffix, f"{name} {g}", **kw)
    stops = {w["stop_reason"] for w in want}
    assert sum(w["n_placed"] for w in want) > 0 and abi.PROBE_STOP_UNSCHEDULABLE in stops, (name, stops)


@pytest.mark.parametrize("name", PROBE_CASES)
def test_probe_at_the_score_range_edge(name):
    """The scored workload's first pod with R = the free pod slots; ipa_near_bound's class is at its bound: refused on the host."""
    _p, c = range_case(name)
    placed = _oracle_placed(c)
    q = pods_of(c, "a")[0]
    P = c.pods_dims["n_pods"]
    room = c.class_pod_limit[int(c.pods["pod_class"][q])] - P
    if name in PROBE_REFUSED:
        with _engine(c, 0, 0, False) as eng:
            eng.schedule()
            li = eng.last_launch()
            with pytest.raises(RuntimeError, match="exceed its class's int32 bounds"):
                eng.probe_run(placed, [(q, 1)])
            assert eng.last_launch() == li
        return
    probes = [(q, min(headroom.free_pod_slots(c, placed), room))]
    want = _want_probes(c, placed, probes)
    runs = [("engine", None, "256", {}), ("no static cache", None, "256", dict(static_cache=False))]
    runs += [(g, geom, suffix, {}) for g, (geom, suffix) in RANGE_GEOMS.items()]
    for g, geom, suffix, kw in runs:
        _run_probes(c, placed, probes, want, geom, suffix, f"{name} {g}", **kw)


def test_probe_at_the_affinity_bound():
    """R = class_pod_limit - n_pods replicas of a pod whose class's raw InterPodAffinity score grows by 2 w per replica: the probe
    stops at MAX_REPLICAS with the raw score within 2 w of 2^31 - 1, equal to the checker and to the recompile-and-resume
    equivalence; one more replica is refused by Engine.probe_run and by compile_cluster; and the list with the R copies explained at
    top_k 16 equals the checker (word 2 at the largest raw score)."""
    p, c = bound_case()
    placed = _oracle_placed(c)
    P, lim = c.pods_dims["n_pods"], bound_limit(c)
    R = lim - P
    probes = [(0, R)]
    want = _want_probes(c, placed, probes)
    assert want[0]["stop_reason"] == abi.PROBE_STOP_MAX_REPLICAS and want[0]["n_placed"] == R
    for g, geom, suffix in (("engine", None, "256"), ("large", (2, 32, True), "big")):
        got = _run_probes(c, placed, probes, want, geom, suffix, f"bound {g}")[0]
    with _engine(c, 0, 0, False) as eng:
        eng.schedule()
        li = eng.last_launch()
        with pytest.raises(RuntimeError, match="exceed its class's int32 bounds"):
            eng.probe_run(placed, [(0, R + 1)])
        assert eng.last_launch() == li
    out, slots, _fc, _fp, _vg, _dev, _P = _resume_with_copies(p, c, placed, 0, R)
    np.testing.assert_array_equal(out, got["node"])
    np.testing.assert_array_equal(slots, got["gpu_slots"])
    # every pod in z0: the last replica sees 2 w per pod before it in the zone
    allp = np.concatenate([placed, got["node"]])
    assert all(c.node_names[g].startswith("n") for g in allp)
    raw_last = 2 * BOUND_W * (len(allp) - 1)
    assert 0 <= I32_MAX - raw_last < 2 * 2 * BOUND_W, raw_last
    with pytest.raises(CompileError, match="inter-pod affinity"):
        compile_cluster(p.nodes, list(p.pods) + [copy.copy(p.pods[0]) for _ in range(R + 1)], p.ctx)
    c2 = compile_cluster(p.nodes, list(p.pods) + [copy.copy(p.pods[0]) for _ in range(R)], p.ctx)
    assert c2.pods_dims["n_pods"] == lim
    pods = np.arange(lim, dtype=np.uint32)
    li, rec, nodes = _explain_run(c2, None, expected(c2, pods, TOP, threads=THREADS), pods, "bound explain")
    _assert_launch(li, "explain", "256", None, c2.n_nodes)
    last = _rows(rec, nodes, lim - 1)
    assert len(last) == c2.n_nodes and {w[2] for _g, w in last} == {0, 100}
