"""Explained decisions and headroom probes at the engine limits, the score-range edges and past 65,536 nodes: the case builders and
tables that tests/test_zz_explain_probe_edges_gpu.py runs, checked on the CPU.

The GPU file runs the explain kernels (simon_explain_kernel_*) and the probe kernels (simon_probe_kernel_*) on every builder of
test_engine_limits.py and every case of test_score_ranges.py, at the geometries of GEOMS, and compares them exactly with
explain_oracle.expected and checkers.probe.  Two cases are new here:
  * wrap_case: zone_case(65537, 20, 3) of test_zz_large_cluster_gpu, whose explained records have known answers (rejected counts and
    feasible counts past 16 bits);
  * bound_case: a Deployment with a preferred podAffinity term to its own label on the zone key, of weight BOUND_W, so that its
    class_pod_limit is 240 pods and a probe up to that limit drives the raw InterPodAffinity score to within 2 x BOUND_W of 2^31 - 1.

CPU: the new cases reach their edges, the known answers hold on the CPU checker, and the tables cover every explain / probe kernel
(the Open-Local variants are covered by test_zz_explain_gpu and test_zz_headroom_gpu: no builder or score-range case has Open-Local)
and every builder and score-range case."""
import numpy as np
import pytest

from simon_b200 import abi, objects as O, simulator
from simon_b200.compiler import CompileError, compile_cluster
from test_engine_limits import BUILDERS, ZONE, _dep, _node, _term
from test_score_ranges import CASES
from util import compiled_kernels

P = "preferredDuringSchedulingIgnoredDuringExecution"

# ---- geometries ---------------------------------------------------------------------------------------------------------------
# Each builder runs its explained decisions and probes at four geometries: the engine's own ("engine": the 256-thread variant at
# these sizes), one CTA at the fewest whole warps that give every thread at least 2 node slots ("one_cta"; the warp-wide reductions
# of the body need whole warps, so a builder of at most 32 nodes gets 1 CTA x 32 threads and 1 slot), one CTA wider than 256
# threads ("wide": the 320- and 384-thread variants, alternating over the builders) and the large-cluster variant at 2 x 32
# threads ("large").  The score-range cases (160 nodes) run test_zz_score_ranges_gpu.GEOMS.


def one_cta_threads(n_nodes):
    return max(32, 32 * (n_nodes // 64))


def limit_geoms(name, n_nodes):
    """-> {geometry: ((CTAs, threads, force_large) or None for the engine's own, the kernel suffix it launches)}."""
    wide = 288 if sorted(BUILDERS).index(name) % 2 == 0 else 352
    return {"engine": (None, "256"), "one_cta": ((1, one_cta_threads(n_nodes), False), "256"),
            "wide": ((1, wide, False), "320" if wide == 288 else "384"), "large": ((2, 32, True), "big")}


RANGE_GEOMS = {"unrolled": ((2, 96, False), "256"), "runtime_slots": ((1, 32, False), "256"), "large": ((2, 64, True), "big")}

# workloads that carry each builder's limit (test_engine_limits.check_at_limit): their first probe-able pod is probed
LIMIT_PROBES = {"scalars8": ["s7", "mix7"], "atoms1024": ["sel15", "pref15"], "taints256": ["tol255", "all"],
                "soft_taints256": ["none", "spread"], "topo8": ["hard7", "anti7", "pref7"], "entries32": ["a", "e", "m"],
                "commit_list_long": ["t"], "big_record": ["big"], "gpu8": ["g64", "g20"]}
# builders that also run explained once without the static-verdict cache
NO_STATIC_CACHE = ["atoms1024", "taints256", "big_record"]
# score-range cases whose probe is refused on the host (class_pod_limit == n_pods)
PROBE_REFUSED = ["ipa_near_bound"]
EXPLAIN_BUILDERS = sorted(LIMIT_PROBES)
EXPLAIN_CASES = sorted(CASES)
PROBE_CASES = sorted(CASES)
NODES = {"scalars8": 24, "atoms1024": 128, "taints256": 41, "soft_taints256": 48, "topo8": 60, "entries32": 20,
         "commit_list_long": 30, "big_record": 80, "gpu8": 16}


# ---- new cases ----------------------------------------------------------------------------------------------------------------

def wrap_case():
    """65,537 nodes in zone a, 20 in zone b, 3 replicas with required anti-affinity to themselves on the zone key."""
    from test_zz_large_cluster_gpu import zone_case
    return zone_case(65537, 20, 3)


def wrap_known(c):
    """The hand-derived records of the three replicas at top_k 16: (node name, F, rejected[SFC_IPA_ANTI], listed node names)."""
    a = [f"a{i:06d}" for i in range(8)]
    first = [x for i in range(8) for x in (a[i], f"b{i}")]
    return [("a000000", 65557, 0, first), ("b0", 20, 65537, [f"b{i}" for i in range(16)]), ("", 0, 65557, [])]


def assert_wrap_records(c, rec, nodes):
    """Records (dicts of explain_oracle.record, or Engine.explanations rows) of the three replicas equal wrap_known."""
    for i, (node, F, anti, listed) in enumerate(wrap_known(c)):
        r = rec[i]
        got_node = c.node_names[int(r["node"])] if int(r["node"]) >= 0 else ""
        assert (got_node, int(r["feasible"]), int(r["rejected"][abi.SFC_IPA_ANTI])) == (node, F, anti), (i, got_node, r["feasible"])
        assert int(np.asarray(r["rejected"]).sum()) == anti, i        # the anti-affinity is the only reason
        rows = nodes[i]
        assert [c.node_names[g] for g, _w in rows] == listed, i
        assert len({w[8] for _g, w in rows}) <= 1, i                   # one total on every listed node


BOUND_W = ((1 << 31) - 1) // (2 * 240)         # 4,473,924: class_pod_limit 240
BOUND_PODS = 10                                  # replicas in the pod list; a probe adds up to 230 more


def bound_case(replicas=BOUND_PODS, n_z0=12):
    """n_z0 identical nodes in zone z0 and one in z1 (110 pod slots each), and `replicas` pods of a Deployment with a preferred
    podAffinity term of weight BOUND_W to its own label on the zone key.  The class scores its own term and the same term of its
    placed pods, 2 w per matching pod in the zone: class_pod_limit = (2^31 - 1) // (2 w) = 240.  The first replica lands on the first
    z0 node and the others follow it into z0, so z0's raw score climbs by 2 w per pod while z1's stays 0.  -> (plan, compiled)."""
    nodes = [_node(f"n{i:02d}", 16, zone="z0") for i in range(n_z0)] + [_node("m00", 16, zone="z1")]
    aff = {"podAffinity": {P: [{"weight": BOUND_W, "podAffinityTerm": _term(ZONE, app="bound")}]}}
    dep = _dep("bound", replicas, cpu="10m", affinity=aff)
    p = simulator.plan(O.ResourceTypes(Nodes=nodes), [O.AppResource("bound", O.ResourceTypes(Deployments=[dep]))])
    return p, compile_cluster(p.nodes, p.pods, p.ctx)


def bound_limit(c):
    return c.class_pod_limit[int(c.pods["pod_class"][0])]


# ---- CPU tests ----------------------------------------------------------------------------------------------------------------

def test_tables_cover_every_explain_and_probe_kernel():
    kernels = set()
    for name in EXPLAIN_BUILDERS:
        kernels |= {s for _g, s in limit_geoms(name, NODES[name]).values()}
    kernels |= {s for _g, s in RANGE_GEOMS.values()}
    assert {f"simon_explain_kernel_{s}" for s in kernels} == compiled_kernels("simon_explain_kernel_")
    assert {f"simon_probe_kernel_{s}" for s in kernels} == compiled_kernels("simon_probe_kernel_")


def test_tables_cover_every_builder_and_case():
    from test_zz_score_ranges_gpu import GEOMS
    assert {g: v[0] for g, v in RANGE_GEOMS.items()} == {g: v[0] for g, v in GEOMS.items()}
    assert set(EXPLAIN_BUILDERS) == set(BUILDERS) == set(NODES)
    assert set(NO_STATIC_CACHE) <= set(BUILDERS)
    assert set(EXPLAIN_CASES) == set(CASES) == set(PROBE_CASES) and set(PROBE_REFUSED) <= set(CASES)


@pytest.mark.parametrize("name", sorted(BUILDERS))
def test_builder_geometries(name):
    """The node counts the geometry table assumes, the one-CTA geometry's slots, and the probed workloads exist."""
    from test_engine_limits import compiled
    _p, c = compiled(*BUILDERS[name]())
    assert c.n_nodes == NODES[name]
    t = one_cta_threads(c.n_nodes)
    assert t % 32 == 0 and (-(-c.n_nodes // t) >= 2) == (c.n_nodes > 32)
    names = {r.tmpl.workload_name for r in c.pod_recs}
    assert set(LIMIT_PROBES[name]) <= names


def test_probe_refused_cases_are_at_their_limit():
    from test_score_ranges import build, pods_of
    for name in PROBE_CASES:
        _p, c = build(name)
        q = pods_of(c, "a")[0]
        lim = c.class_pod_limit[int(c.pods["pod_class"][q])]
        assert (lim <= c.pods_dims["n_pods"]) == (name in PROBE_REFUSED), (name, lim)


def test_bound_case_reaches_the_affinity_guard():
    p, c = bound_case()
    lim = bound_limit(c)
    assert lim == ((1 << 31) - 1) // (2 * BOUND_W) == 240
    assert sum(int(x) for x in c.snap["alloc_pods"]) >= lim
    with pytest.raises(CompileError, match="inter-pod affinity"):
        bound_case(lim + 1)
    p2, c2 = bound_case(lim)
    assert bound_limit(c2) == lim


def test_bound_case_probe_on_the_checker():
    """On the CPU checker: the probe of lim - n_pods replicas places them all, every pod in z0, and the last replica sees a raw
    InterPodAffinity score within 2 w of 2^31 - 1."""
    import checkers
    from oracle.binding import Oracle
    p, c = bound_case()
    o = Oracle(c)
    placed = o.schedule()[0]
    R = bound_limit(c) - c.pods_dims["n_pods"]
    want = checkers.probe(o, placed, 0, R)
    o.close()
    assert want["n_placed"] == R and want["stop_reason"] == abi.PROBE_STOP_MAX_REPLICAS
    zones = np.array([c.node_names[g].startswith("n") for g in np.concatenate([placed, want["node"]])])
    assert zones.all()
    raw_last = 2 * BOUND_W * (len(zones) - 1)
    assert 0 <= (1 << 31) - 1 - raw_last < 2 * 2 * BOUND_W


def test_wrap_case_known_answers_on_the_checker():
    import explain_oracle
    c = wrap_case()
    names = c.node_names
    assert names[:4] == ["a000000", "b0", "a000001", "b1"]
    want = explain_oracle.expected(c, [0, 1, 2], 16, threads=8)
    assert_wrap_records(c, want, [w["top"] for w in want])
