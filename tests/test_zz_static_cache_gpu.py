"""The placement and move kernels with the static verdict cache off, against the CPU oracle and the checkers.

The pod upload keeps a per-(static signature, node) verdict cache (the node-static filter verdict, NodeAffinity raw score, soft
taint count and the selection / hard-key / ignored-node flags) while it fits 2 GiB.  Past that, the placement kernel works out every
static verdict at every class switch, the move kernel and simon_moves_hard_prep evaluate selection, node name, taints and hard
topology keys inline, and simon_static_fill does not run.  Real clusters reach that regime (hundreds of thousands of nodes, or
tens of thousands of distinct node selectors), so the same inline code is checked here on the suite's own clusters with the cache
switched off (Engine(static_cache=False), SIMON_OPT_NO_STATIC_CACHE), and once on a cluster above the real cap.

Each placement test also shows that the uncached path ran: the leader thread's static evaluations (stats()["static_evals"]) are
at least its class switches, and more than in the same run with the cache on.  The file sorts after the rest of the suite.
"""
import copy
import os

import numpy as np
import pytest

import test_drain as TD
import test_zz_engine_limits_gpu as LIM
import test_zz_kernel_variants_gpu as KV
from test_engine_limits import BUILDERS

pytestmark = pytest.mark.gpu
GPU, HARD = 1, 2


def _engine(c, cs=0, t=0, big=False, **kw):
    from simon_b200.engine import Engine
    return Engine(c, device=0, cluster_ctas=cs, threads_per_cta=t, force_large=big, **kw)


def _stats_of(c, cs, t, big, pin_fast=True):
    """stats() of a full run with the cache on, at the same geometry."""
    with _engine(c, cs, t, big, pin_fast=pin_fast) as eng:
        eng.schedule(download=False)
        return eng.stats()


def _revisits_a_signature(c):
    """Whether the pods the scheduler places switch between classes more often than they have static signatures, so that a run
    with the cache finds some of its verdicts cached."""
    from simon_b200.compiler import SCW_STATIC_SIG
    off, blob = c.pods["class_off"], c.pods["class_blob"]
    seq = c.pods["pod_class"][c.pods["pod_fixed_node"] == -1]
    sig = np.array([int(blob[int(off[k]) + SCW_STATIC_SIG]) for k in range(len(off) - 1)])
    return len(seq) > 0 and 1 + int((np.diff(seq) != 0).sum()) > len(np.unique(sig[seq]))


def _assert_uncached(c, st, cached, what):
    """Every class switch evaluated the leader thread's static verdicts; with the cache on, revisited signatures were not."""
    assert st["class_switches"] > 0 and st["static_evals"] >= st["class_switches"], (what, st["static_evals"], st["class_switches"])
    if _revisits_a_signature(c):
        assert st["static_evals"] > cached["static_evals"], (what, st["static_evals"], cached["static_evals"])
    else:
        assert st["static_evals"] >= cached["static_evals"], (what, st["static_evals"], cached["static_evals"])


# ---- placement -------------------------------------------------------------------------------------------------------------

PLACE = [e for e in KV.ENTRIES if not e[1].startswith("local")]
LOCAL = [e for e in KV.ENTRIES if e[1].startswith("local")]


@pytest.mark.parametrize("kernel,fam,cs,t,big", PLACE, ids=[f"{k[6:]}-{cs}x{t}" for k, fam, cs, t, big in PLACE])
def test_variant_matches_oracle_uncached(kernel, fam, cs, t, big):
    """Every placement variant at the geometry of test_zz_kernel_variants_gpu.VARIANTS, both pinned-class paths: node, winning
    score, failure records, state(), state_ext() and GPU slot words against the oracle."""
    c = KV.family(fam)
    for pin_fast in (True, False):
        with _engine(c, cs, t, big, record_scores=True, pin_fast=pin_fast, static_cache=False) as eng:
            out, score, fc, fp = eng.schedule()
            li = eng.last_launch()
            assert li["kernel"] == kernel and (li["cluster_ctas"], li["threads_per_cta"], li["large"]) == (cs, t, big), li
            what = f"{kernel} {cs}x{t} pin_fast={pin_fast} uncached"
            KV.assert_matches_oracle(fam, out, score, fc, fp, eng, what)
            _assert_uncached(c, eng.stats(), _stats_of(c, cs, t, big, pin_fast), what)


@pytest.mark.parametrize("kernel,fam,cs,t,big", LOCAL, ids=[f"{k[6:]}-{cs}x{t}" for k, fam, cs, t, big in LOCAL])
def test_open_local_variant_matches_restated_composition_uncached(kernel, fam, cs, t, big):
    from test_open_local import check_restated_open_local
    c = KV.family(fam)
    with _engine(c, cs, t, big, record_scores=True, static_cache=False) as eng:
        out, score, _fc, _fp = eng.schedule()
        final = eng.storage_state()
        li = eng.last_launch()
        st = eng.stats()
    assert li["kernel"] == kernel and li["local"] and li["large"] == big, li
    assert check_restated_open_local(c, out, score, final) > 0
    assert (out >= 0).sum() > len(out) // 2
    _assert_uncached(c, st, _stats_of(c, cs, t, big), kernel)


@pytest.mark.parametrize("name", sorted(BUILDERS))
def test_engine_limit_full_run_matches_oracle_uncached(name):
    """Every builder of test_engine_limits.py, at the engine's own geometry and with the large-cluster variant."""
    _p, c = LIM.case(name)
    for big in (False, True):
        with _engine(c, big=big, record_scores=True, static_cache=False) as eng:
            out, score, fc, fp = eng.schedule()
            li = eng.last_launch()
            assert (li["kernel"] == "simon_place_kernel_big") == big and li["large"] == big, li
            LIM._assert_run(name, eng, out, score, fc, fp, f"{name} large={big} uncached")
            _assert_uncached(c, eng.stats(), _stats_of(c, 0, 0, big), f"{name} large={big}")


# ---- batches, drains, resume -----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kernel,cs,t,big", [("simon_place_kernel_384_2", 2, 352, False), ("simon_place_kernel_big", 2, 160, True)])
def test_scenario_batch_matches_oracle_uncached(kernel, cs, t, big):
    """All nodes, every other node, a reversed subset and a random subset of the dense mix in one batch, each against the oracle
    restricted to the same node list."""
    from oracle.binding import Oracle
    c = KV.family("dense")
    lists = KV._node_lists(c.n_nodes, 7)
    with _engine(c, cs, t, big, static_cache=False) as eng:
        res, nodes = eng.run_scenarios(lists, want_nodes=True)
        li = eng.last_launch()
    assert (li["kernel"], li["n_scenarios"], li["large"]) == (kernel, len(lists), big), li
    o = Oracle(c, threads=min(16, len(os.sched_getaffinity(0))))
    for i, act in enumerate(lists):
        o.set_active(act)
        o.reset()
        ref = o.schedule()[0]
        st = o.state()
        np.testing.assert_array_equal(nodes[i], ref, err_msg=f"scenario {i}")
        assert res[i]["n_unscheduled"] == int((ref == -1).sum()), i
        assert (res[i]["req_mcpu"], res[i]["req_mem"]) == (int(st["req_mcpu"][act].sum()), int(st["req_mem"][act].sum())), i
    o.close()


@pytest.mark.parametrize("kernel", sorted(TD.DRAIN_VARIANTS))
def test_drain_variant_matches_checker_uncached(kernel):
    import checkers
    from simon_b200 import scaledown, synth
    cs, t, big = TD.DRAIN_VARIANTS[kernel]
    rng = np.random.default_rng(11)
    for seed in (0, 5):
        c = TD._compiled(*synth.make_mix(seed_no=seed, n_nodes=40))
        o, placed = TD._live(c)
        order = scaledown.NodeOrder(c)
        drains = TD._drains(c, rng, n_single=12)
        remain = [order.remaining(d) for d in drains]
        with _engine(c, cs, t, big, record_scores=True, static_cache=False) as eng:
            got = eng.drain_run(placed, remain)
            assert eng.last_launch()["kernel"] == kernel
        for d, rl, g in zip(drains, remain, got):
            want = checkers.drain(o, placed, rl)
            TD._assert_drain_equal(g, want, f"{kernel} seed {seed} drain {d} uncached")
            pos = g["node"] >= 0
            assert np.array_equal(g["score"][pos], want["score"][pos]), d
        o.close()


@pytest.mark.parametrize("kernel,cs,t,big", [("simon_place_kernel_384_2", 2, 352, False), ("simon_place_kernel_big", 2, 160, True)])
def test_resume_from_half_matches_oracle_uncached(kernel, cs, t, big):
    ref, _s, _fc, _fp, rst, rext, rslots = KV.oracle_run("dense")
    c = KV.family("dense")
    P = len(ref)
    with _engine(c, cs, t, big, static_cache=False) as eng:
        out = eng.schedule_resume(ref[: P // 2])[0]
        assert eng.last_launch()["kernel"] == kernel
        np.testing.assert_array_equal(out, ref)
        st, ext = eng.state(), eng.state_ext()
        for k in rst:
            np.testing.assert_array_equal(st[k], rst[k], err_msg=k)
        for k in rext:
            np.testing.assert_array_equal(ext[k], rext[k], err_msg=k)
        np.testing.assert_array_equal(eng.gpu_slot_words()[P // 2:], rslots[P // 2:])


# ---- per-node detail -------------------------------------------------------------------------------------------------------

def _with_node_name(c, cls, node):
    """c with class `cls` restricted to node `node` by spec.nodeName (SCW_NODE_NAME >= 0), under a static signature of its own,
    and its pods left to the scheduler."""
    from simon_b200.compiler import SCW_NODE_NAME, SCW_STATIC_SIG
    c2 = copy.copy(c)
    c2.pods = dict(c.pods)
    c2.pods_dims = dict(c.pods_dims)
    blob = np.array(c.pods["class_blob"], copy=True)
    at = int(c.pods["class_off"][cls])
    assert blob[at + SCW_NODE_NAME] == -1
    blob[at + SCW_NODE_NAME] = node
    blob[at + SCW_STATIC_SIG] = c.pods_dims["n_static_sigs"]
    c2.pods["class_blob"] = blob
    c2.pods_dims["n_static_sigs"] = c.pods_dims["n_static_sigs"] + 1
    return c2


def _dump_vs_oracle(c, pod):
    """The engine's per-node filter verdicts (a mask of simon_fail_code bits) and totals of `pod` against the oracle's per-node
    stage numbers and totals: the same stage on every node, any of the four static stages for a static failure.  -> the oracle's
    stages."""
    from oracle.binding import Oracle
    from test_moves_scope import _stage_of
    o = Oracle(c)
    o.enable_dump()
    ref_out = o.schedule(0, pod + 1)[0]
    ref_code, sc = o.last_detail()
    o.close()
    ref_code = np.array(ref_code, np.int32)
    ref_total = np.array([int(x[8]) for x in sc], np.int64)
    with _engine(c, static_cache=False) as eng:
        out, tot, code = eng.dump_pod(pod)
    np.testing.assert_array_equal(out, ref_out)
    stage = np.array([_stage_of(int(x)) for x in code])
    bad = np.nonzero(np.where(stage < 0, (ref_code < 1) | (ref_code > 4), stage != ref_code))[0]
    assert len(bad) == 0, f"pod {pod}: verdicts differ on nodes {bad[:8]}: gpu {code[bad[:8]]} oracle stages {ref_code[bad[:8]]}"
    feas = ref_code == 0
    if feas.sum() > 1:
        bad = np.nonzero(feas & (tot != ref_total))[0]
        assert len(bad) == 0, f"pod {pod}: totals differ on nodes {bad[:8]}: gpu {tot[bad[:8]]} oracle {ref_total[bad[:8]]}"
    return ref_code


def test_per_node_detail_matches_oracle_uncached():
    """Engine.dump_pod of ordinary pods of the dense mix, of a pinned (DaemonSet) pod, and of a pod whose class names a node
    (spec.nodeName): totals and per-node verdict codes against the oracle's detail."""
    from simon_b200.compiler import CLS_PINNED, SCW_FLAGS
    c = KV.family("dense")
    ref = KV.oracle_run("dense")[0]
    cls, fixed, pin = c.pods["pod_class"], c.pods["pod_fixed_node"], c.pods["pod_pin_node"]
    flags = np.array([int(c.pods["class_blob"][int(c.pods["class_off"][k]) + SCW_FLAGS]) for k in range(len(c.pods["class_off"]) - 1)])
    free = np.nonzero((fixed == -1) & (pin < 0) & ((flags[cls] & CLS_PINNED) == 0))[0]
    pinned = np.nonzero((fixed == -1) & (pin >= 0))[0]
    assert len(free) > 400 and len(pinned) > 0
    codes = set()
    for pod in (int(free[10]), int(free[len(free) // 2]), int(free[-1]), int(pinned[len(pinned) // 2])):
        codes |= set(_dump_vs_oracle(c, pod).tolist())
    assert 0 in codes and len(codes) > 2
    # a placed pod's class narrowed to the node the oracle gave it, and its first pod dumped: NodeName fails everywhere else
    q = int(free[np.nonzero(ref[free] >= 0)[0][len(free) // 3]])
    c2 = _with_node_name(c, int(cls[q]), int(ref[q]))
    first = int(np.nonzero(c2.pods["pod_class"] == cls[q])[0][0])
    code = _dump_vs_oracle(c2, first)
    others = np.arange(c.n_nodes) != ref[q]
    assert (code[others] != 0).all() and (code[others] == 2).sum() > c.n_nodes // 2
    # and the whole pod list of the narrowed cluster
    from oracle.binding import Oracle
    o = Oracle(c2, threads=min(16, len(os.sched_getaffinity(0))))
    want = o.schedule()
    o.close()
    with _engine(c2, record_scores=True, static_cache=False) as eng:
        got = eng.schedule()
    np.testing.assert_array_equal(got[0], want[0])
    np.testing.assert_array_equal(got[2], want[2])
    np.testing.assert_array_equal(got[3], want[3])


# ---- moves -----------------------------------------------------------------------------------------------------------------

def _inline_reasons_cluster():
    """Every reason the move kernel's inline static verdict knows, and hard-spread domains that must stay unregistered.

    Zones A (a1 with 64 cores, a2, u1 unschedulable), B (b1, t1 with a NoSchedule taint), C (c1), D (only x1, outside the
    selection pool=main) and E (only e1, without the rack label).  Pods labelled app=s are pre-bound by spec.nodeName on a2, b1
    and c1.  p (app=s, pool=main, DoNotSchedule spread over zone and rack, maxSkew 1) is placed on a1: A, B and C count 1, so every
    registered zone allows it.  m (pool=main, no spread) is placed too.  Moving p from a1 to b1 is feasible only while D and E stay
    unregistered: registered, either would bring the zone minimum to 0."""
    from test_moves_scope import _compile, _node, _pod
    main, s = {"pool": "main"}, {"app": "s"}
    nodes = [_node("a1", 64, "A", {**main, "rack": "r1"}), _node("a2", 4, "A", {**main, "rack": "r2"}),
             _node("u1", 4, "A", {**main, "rack": "r1"}), _node("b1", 4, "B", {**main, "rack": "r1"}),
             _node("t1", 4, "B", {**main, "rack": "r2"}, taints=[{"key": "ded", "value": "1", "effect": "NoSchedule"}]),
             _node("c1", 4, "C", {**main, "rack": "r2"}), _node("x1", 4, "D", {"pool": "other", "rack": "r1"}),
             _node("e1", 4, "E", main)]
    nodes[2]["spec"]["unschedulable"] = True
    tsc = {"topologySpreadConstraints": [{"maxSkew": 1, "topologyKey": k, "whenUnsatisfiable": "DoNotSchedule",
                                          "labelSelector": {"matchLabels": s}} for k in ("topology.kubernetes.io/zone", "rack")],
           "nodeSelector": main}
    pods = [_pod("r-a2", s, "a2"), _pod("r-b1", s, "b1"), _pod("r-c1", s, "c1"), _pod("p", s, spec_extra=tsc),
            _pod("m", spec_extra={"nodeSelector": main})]
    return _compile(nodes, pods)


def test_moves_hit_every_inline_reason_uncached():
    """Hand-picked moves onto an unschedulable node, onto a tainted node, outside the node selection, of a pod bound by
    spec.nodeName onto other nodes, and a hard-spread move whose verdict depends on the domains that only unselected or keyless
    nodes carry, at scope 0 and GPU|HARD, against the scoped checker."""
    from oracle.binding import Oracle
    from simon_b200.abi import SFC_STATIC
    from test_moves_scope import _engine_vs_checker
    c, names = _inline_reasons_cluster()
    o = Oracle(c)
    out = o.schedule()[0]
    n = {x: c.node_names.index(x) for x in ("a1", "a2", "u1", "b1", "t1", "c1", "x1", "e1")}
    q = {x: names.index(x) for x in names}
    assert out[q["p"]] == n["a1"] and out[q["m"]] == n["a1"]
    mv = [(q["m"], n["u1"]), (q["m"], n["t1"]), (q["m"], n["x1"]),(q["r-b1"], n["a1"]), (q["r-b1"], n["c1"]), (q["p"], n["b1"]), (q["p"], n["x1"]), (q["p"], n["e1"])]
    mv = np.array(mv, np.uint32)
    for scope in (0, GPU | HARD):
        code = _engine_vs_checker(c, o, out, mv, scope, static_cache=False)
        static = code == 1 << SFC_STATIC
        assert static[:5].all(), (scope, code.tolist())                         # unschedulable, taint, selection, nodeName x2
        if scope:
            assert code[5] == 0 and static[6] and code[7] not in (0, 1 << SFC_STATIC), code.tolist()
    o.close()


MOVE_CASES = [("mix", dict(seed_no=103, n_nodes=95, n_workloads=40, max_replicas=7), 30000),
              ("c3", dict(n_nodes=400, n_workloads=80, replicas=10, n_apps=2, seed_no=21, gpu_pct=25), 40000)]


@pytest.mark.parametrize("kind,kw,n", MOVE_CASES, ids=[k for k, _kw, _n in MOVE_CASES])
def test_sampled_moves_match_checker_uncached(kind, kw, n):
    from test_moves_scope import _engine_vs_checker, _moves, _state
    _p, c, o, out = _state(kind, **kw)
    mv = _moves(out, c, n)
    for scope in (0, GPU | HARD):
        code = _engine_vs_checker(c, o, out, mv, scope, static_cache=False)
        assert (code == 0).any() and (code == 1).any(), scope
    o.close()


@pytest.mark.parametrize("name", sorted(BUILDERS))
def test_engine_limit_moves_match_checker_uncached(name):
    from oracle.binding import Oracle
    from simon_b200 import moves as M
    from test_moves_scope import _engine_vs_checker
    _p, c = LIM.case(name)
    o = Oracle(c)
    out = o.schedule()[0]
    hand = LIM._hand_picked(name, c, out)
    mv = np.concatenate([hand, M.sample_moves(len(out), c.n_nodes, 20000, seed=5, placement=out)]).astype(np.uint32)
    for scope in (0, GPU | HARD):
        code = _engine_vs_checker(c, o, out, mv, scope, static_cache=False)
        assert (code[len(hand):] != 0).any(), scope
    o.close()


def test_migration_plans_match_checkers_uncached():
    """A migration plan without and with a PodDisruptionBudget table, each against its checker."""
    from simon_b200 import disruption, rebalance
    from test_disruption import _plan_vs_checker, mixed_pdbs
    from test_moves_plan import _engine_vs_checker, _oracle_state
    from util import make_case
    _p, c = make_case("c3", n_nodes=400, n_workloads=80, replicas=10, n_apps=2, seed_no=21, gpu_pct=25)
    o, out = _oracle_state(c)
    o.close()
    mv = rebalance.candidates(c, out)
    mv = mv[np.sort(np.random.RandomState(3).choice(len(mv), min(len(mv), 200000), replace=False))]
    for scope in (0, HARD):
        r = _engine_vs_checker(c, mv, 25, 1, scope, rebuild=True, static_cache=False)
        assert len(r["steps"]) > 0
    t = disruption.compile_pdbs(mixed_pdbs(c, 7), c)
    r = _plan_vs_checker(c, mv, t, 40, HARD, static_cache=False)[2]
    assert len(r["steps"]) > 0


# ---- above the cache's cap -------------------------------------------------------------------------------------------------

OVER_NODES, OVER_TWINS = 16400, 1000


def over_cap_cluster(n_nodes=OVER_NODES, n_twins=OVER_TWINS):
    """n_nodes nodes and as many single-pod workloads, each with a static signature of its own, so that the verdict cache would
    take n_nodes^2 x 8 bytes, over 2 GiB.  A cluster may reference at most 1,024 label atoms, so the signatures are pairs: node j
    carries a = j % 128 and b = j // 128; workload i requires a in {i % 128, i % 128 + 1} and b not i // 128 (about 250 nodes
    each).  The first n_twins workloads each have a twin with the same selection and another CPU request, ordered right after
    it, so the first 2 x n_twins pods visit every signature twice."""
    from simon_b200 import simulator, synth
    from simon_b200.compiler import compile_cluster
    from simon_b200.objects import AppResource, ResourceTypes
    cluster = ResourceTypes()
    for j in range(n_nodes):
        cluster.Nodes.append(synth._node(f"n{j:05d}", 8 + 8 * (j % 7), f"z{j % 3}", "r", 100,
                                         {"st.test/a": f"a{j % 128}", "st.test/b": f"b{j // 128}"}))
    app = AppResource("app", ResourceTypes())

    def pod(name, i, cpu):
        aff = {"nodeAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": {"nodeSelectorTerms": [{"matchExpressions": [
            {"key": "st.test/a", "operator": "In", "values": [f"a{i % 128}", f"a{(i + 1) % 128}"]},
            {"key": "st.test/b", "operator": "NotIn", "values": [f"b{i // 128}"]}]}]}}}
        return {"apiVersion": "v1", "kind": "Pod", "metadata": {"name": name, "namespace": "default"},
                "spec": {"affinity": aff, "containers": [{"name": "c", "image": "registry.local/x:v1",
                                                          "resources": {"requests": {"cpu": cpu, "memory": "1Gi"}}}]}}
    for i in range(n_nodes):
        app.Resource.Pods.append(pod(f"w{i:05d}", i, "2"))
        if i < n_twins:
            app.Resource.Pods.append(pod(f"w{i:05d}-twin", i, "3"))
    p = simulator.plan(cluster, [app])
    return compile_cluster(p.nodes, p.pods, p.ctx)


def test_over_the_cache_cap_without_the_flag():
    """The first 2 x OVER_TWINS pods of over_cap_cluster() against the oracle, on the default engine: the cache would pass its cap,
    so every class switch evaluates the leader thread's nodes again, revisited signatures included."""
    from oracle.binding import Oracle
    from simon_b200.compiler import SCW_STATIC_SIG
    c = over_cap_cluster()
    assert c.pods_dims["n_static_sigs"] * c.n_nodes * 8 > 2 << 30
    cls = c.pods["pod_class"]
    sig = np.array([int(c.pods["class_blob"][int(c.pods["class_off"][k]) + SCW_STATIC_SIG]) for k in range(len(c.pods["class_off"]) - 1)])
    n = 2 * OVER_TWINS
    assert len(np.unique(sig[cls[:n]])) == OVER_TWINS and len(np.unique(cls[:n])) == n
    o = Oracle(c, threads=16)
    ref, _rs, rfc, rfp = o.schedule(0, n)
    rst = o.state()
    o.close()
    with _engine(c, record_scores=True) as eng:
        out, _score, fc, fp = eng.schedule(0, n)
        st, li = eng.stats(), eng.last_launch()
        state = eng.state()
    bad = np.nonzero(out != ref)[0]
    assert len(bad) == 0, f"{len(bad)} mismatches, first at pods {bad[:5]}: gpu {out[bad[:5]]} oracle {ref[bad[:5]]}"
    assert (ref >= 0).all()
    np.testing.assert_array_equal(fc, rfc)
    np.testing.assert_array_equal(fp, rfp)
    for k in rst:
        np.testing.assert_array_equal(state[k], rst[k], err_msg=k)
    # every switch evaluates the leader's nodes (at least N / threads of them): with a cache, the revisits would evaluate none
    per = c.n_nodes // (li["cluster_ctas"] * li["threads_per_cta"])
    assert st["class_switches"] >= n - 1 and st["static_evals"] >= per * st["class_switches"] and per >= 2, (st, li)
