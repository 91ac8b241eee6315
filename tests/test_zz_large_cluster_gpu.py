"""The large-cluster kernel variant past 65,536 nodes against the C oracle and its checkers.

Known answers at the flip word's old 16-bit wrap (csrc/simon_flip_word.h): a zone of Z identical nodes and one or two nodes of a
second zone, and a Deployment with required pod anti-affinity to itself on the zone key.  Ties go to the first node in scenario
order (nodeTree order, which interleaves the zones), so replica 1 lands on the first zone-a node; that makes every node of zone a
infeasible at once, Z flips with the last winner among them.  With one zone-b node replica 2 goes there with score 0 (one feasible
node is not scored) and replica 3 is unschedulable.  Z = 65,537 and 131,073 wrapped a 16-bit flip count to 1, which took the
single-node flip fast path with a feasible count too large by 65,536 k; Z = 65,536 and 65,538 are the near misses.  Engine.stats()
pins the path: the wrap decision is a flip with a full summary rebuild, never the fast path.  A small control on the same variant
shows the fast path does fire on a real single flip.

Zone flips of 3,000 to 65,537 nodes under hostname and rack spread: the net change of the counted set wraps the large variant's
12-bit field, so the predicted hostname size is wrong, and only the full summary's size check and the spread pass it redoes pick
the right winner.

Then C3-shaped clusters with GPU share of 70,000 nodes and of the 327,680-node cap: single runs (every score, zeros included,
failure records, state(), state_ext(), GPU slot words), a resume from half of the placement decisions, scenario batches, drains
and probes at both sizes; one run without the static-verdict cache and sampled moves against the scoped checker at 70,000; and
the Open-Local placement, drain and probe kernels on a 70,000-node Open-Local cluster.
"""
import functools
import os

import numpy as np
import pytest

from simon_b200 import abi, objects as O, simulator, synth
from simon_b200.compiler import compile_cluster

pytestmark = pytest.mark.gpu

R = "requiredDuringSchedulingIgnoredDuringExecution"
ZONE = "topology.kubernetes.io/zone"
THREADS = min(16, len(os.sched_getaffinity(0)))


def _engine(c, **kw):
    from simon_b200.engine import Engine
    return Engine(c, device=0, record_scores=True, **kw)


@functools.lru_cache(maxsize=None)
def zone_case(n_a, n_b, replicas):
    """n_a nodes in zone za, then n_b in zone zb (all 8 cores, 32 GiB), and `replicas` pods of a Deployment with required
    anti-affinity to itself on the zone key."""
    nodes = [synth._node(f"a{i:06d}", 8, "za", "", 100) for i in range(n_a)] + [synth._node(f"b{i}", 8, "zb", "", 100) for i in range(n_b)]
    lab = {"app": "anti"}
    ctr = {"name": "c", "image": "registry.local/anti:v1", "resources": {"requests": {"cpu": "1", "memory": "1Gi"}}}
    aff = {"podAntiAffinity": {R: [{"labelSelector": {"matchLabels": lab}, "topologyKey": ZONE}]}}
    dep = {"apiVersion": "apps/v1", "kind": "Deployment", "metadata": {"name": "anti", "namespace": "default"},
           "spec": {"replicas": replicas, "selector": {"matchLabels": lab},
                    "template": {"metadata": {"labels": lab}, "spec": {"containers": [ctr], "affinity": aff}}}}
    p = simulator.plan(O.ResourceTypes(Nodes=nodes), [O.AppResource("wrap", O.ResourceTypes(Deployments=[dep]))])
    return compile_cluster(p.nodes, p.pods, p.ctx)


_ORACLE = {}


def oracle_full(c):
    """The oracle's full run of the compiled cluster c (one of the cached cases above): (out, score, fail_counts, fail_pod,
    state(), state_ext(), GPU slot words)."""
    if id(c) not in _ORACLE:
        from oracle.binding import Oracle
        o = Oracle(c, threads=THREADS)
        _ORACLE[id(c)] = (c, o.schedule() + (o.state(), o.state_ext(), o.gpu_slot_words()))
        o.close()
    return _ORACLE[id(c)][1]


def _assert_run(c, eng, out, score, fc, fp, what):
    """Placements, EVERY scheduled pod's score (zeros included), failure records, state(), state_ext() and GPU slot words."""
    ref, rscore, rfc, rfp, rst, rext, rslots = oracle_full(c)
    bad = np.nonzero(out != ref)[0]
    assert len(bad) == 0, f"{what}: {len(bad)} mismatches, first at pods {bad[:5]}: gpu {out[bad[:5]]} oracle {ref[bad[:5]]}"
    sched = ref >= 0
    bad = np.nonzero(sched & (score != rscore))[0]
    assert len(bad) == 0, f"{what}: scores differ at pods {bad[:5]}: gpu {score[bad[:5]]} oracle {rscore[bad[:5]]}"
    np.testing.assert_array_equal(fp, rfp, err_msg=what)
    np.testing.assert_array_equal(fc, rfc, err_msg=what)
    st, ext = eng.state(), eng.state_ext()
    for k in rst:
        np.testing.assert_array_equal(st[k], rst[k], err_msg=f"{what}: {k}")
    for k in rext:
        np.testing.assert_array_equal(ext[k], rext[k], err_msg=f"{what}: {k}")
    np.testing.assert_array_equal(eng.gpu_slot_words(), rslots, err_msg=f"{what}: GPU slots")


def _assert_large(li, n_nodes, n_scenarios=1):
    slots = -(-n_nodes // (16 * 320))
    assert li["kernel"].endswith("_big") and li["large"], li
    assert (li["cluster_ctas"], li["threads_per_cta"], li["node_slots"]) == (16, 320, slots), li
    assert li["n_scenarios"] == n_scenarios, li


# ---- known answers at the wrap ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n_a", [65536, 65537, 65538, 131073])
def test_zone_flip_at_the_wrap(n_a):
    """Replica 1 on the first zone-a node, replica 2 on the one zone-b node with score 0 after n_a flips, replica 3 unschedulable
    (every node refused by the anti-affinity): a full summary rebuild decides replica 2, never the single-node fast path."""
    c = zone_case(n_a, 1, 3)
    names = c.node_names
    ref, rscore, rfc, rfp = oracle_full(c)[:4]
    assert [names[g] for g in ref[:2]] == ["a000000", "b0"] and ref[2] == -1
    assert rscore[0] > 0 and rscore[1] == 0 and list(rfp) == [2]
    with _engine(c) as eng:
        out, score, fc, fp = eng.schedule()
        _assert_large(eng.last_launch(), n_a + 1)
        st = eng.stats()
        _assert_run(c, eng, out, score, fc, fp, f"zone {n_a}")
    assert score[1] == 0
    # replica 1: first visit of the class, a full summary.  Replica 2: n_a flips -> a full summary, never the fast path.
    # Replica 3: one flip, the last winner, but it held the extremes and no feasible node is left -> a full summary as well.
    assert st["decisions"] == 3 and st["single_flip_fast"] == 0 and st["redone"] == 2 and st["summary_rebuilds"] == 3, st


def test_single_flip_fast_path_fires_on_the_large_variant():
    """The control: the same class on 1 + 2 nodes (forced onto the large variant) flips exactly one node, the last winner, and the
    fast path takes that decision."""
    c = zone_case(1, 2, 2)
    with _engine(c, force_large=True) as eng:
        out, score, fc, fp = eng.schedule()
        assert eng.last_launch()["large"]
        st = eng.stats()
        _assert_run(c, eng, out, score, fc, fp, "control")
    assert st["decisions"] == 2 and st["redone"] == 1 and st["single_flip_fast"] == 1 and st["summary_rebuilds"] == 1, st


@pytest.mark.parametrize("n_a", [65537, 131073])
def test_zone_flip_probe_stops_when_nothing_is_feasible(n_a):
    """A headroom probe of the Deployment's pod on the empty cluster places replica 1 on zone a, replica 2 on zone b after the
    wrap-sized flip (score 0) and stops at replica 3, where no node is feasible (the probe's stop reads the feasible count)."""
    import checkers
    from oracle.binding import Oracle
    c = zone_case(n_a, 1, 3)
    placed = np.full(c.pods_dims["n_pods"], -1, np.int32)
    o = Oracle(c, threads=THREADS)
    want = checkers.probe(o, placed, 0, 5)
    o.close()
    assert want["n_placed"] == 2 and want["stop_reason"] == abi.PROBE_STOP_UNSCHEDULABLE and want["score"][1] == 0
    with _engine(c) as eng:
        got = eng.probe_run(placed, [(0, 5)])[0]
        _assert_large(eng.last_launch(), n_a + 1)
        st = eng.stats()
    assert (got["n_placed"], got["stop_reason"]) == (want["n_placed"], want["stop_reason"])
    for k in ("node", "score", "gpu_slots", "fail_counts"):
        np.testing.assert_array_equal(got[k], want[k], err_msg=k)
    assert st["single_flip_fast"] == 0 and st["redone"] >= 1, st


# ---- a zone flip under hostname spread: the mispredicted topology size goes through sizes_ok and the spread redo ------------

RACK = "example.com/rack"
HOST = "kubernetes.io/hostname"


def _dep(name, replicas, labels, spec):
    ctr = {"name": "c", "image": f"registry.local/{name}:v1", "resources": {"requests": {"cpu": "1", "memory": "1Gi"}}}
    return {"apiVersion": "apps/v1", "kind": "Deployment", "metadata": {"name": name, "namespace": "default"},
            "spec": {"replicas": replicas, "selector": {"matchLabels": labels},
                     "template": {"metadata": {"labels": labels}, "spec": dict(containers=[ctr], **spec)}}}


@functools.lru_cache(maxsize=None)
def spread_case(n_a):
    """Zone za: n_a nodes, a000001..a000003 in rack r1 and the rest in rack r0.  Zone zb: b0 (rack rb0) and b1 (rack r1).  One
    tier=web pod pinned by nodeSelector to each of a000001..a000003 and b0, then two replicas of `anti` (tier=web): required
    anti-affinity to itself on the zone key, and ScheduleAnyway spread of tier=web over hostname and over rack.

    Replica 1 goes to a000000 (raw spread score 0, first in scenario order) and makes all n_a zone-a nodes infeasible.  Replica 2
    chooses between b0 (1 pod on the host, 1 in its rack) and b1 (0 on the host, 3 in rack r1 from the zone-a pods).  With the
    true sizes (2 counted hosts, 2 racks) both weights are log 4, so b0 scores 2 log 4 < 3 log 4 and wins.  The net change of the
    counted set is -n_a, which the large variant's 12-bit field wraps for n_a > 2,047: the hostname size predicted from it is
    some thousands, its weight near log n_a, and b0's 1 x log n_a + log 4 would lose to b1.  Only the full summary's size check
    (sizes_ok) and the spread pass it redoes under the true sizes give b0."""
    nodes = [synth._node(f"a{i:06d}", 8, "za", "", 100, labels={RACK: "r1" if 1 <= i <= 3 else "r0"}) for i in range(n_a)]
    nodes += [synth._node("b0", 8, "zb", "", 100, labels={RACK: "rb0"}), synth._node("b1", 8, "zb", "", 100, labels={RACK: "r1"})]
    fills = [_dep(f"fill-{h}", 1, {"app": f"fill-{h}", "tier": "web"}, {"nodeSelector": {HOST: h}})
             for h in ("a000001", "a000002", "a000003", "b0")]
    web = {"matchLabels": {"tier": "web"}}
    spec = {"affinity": {"podAntiAffinity": {R: [{"labelSelector": {"matchLabels": {"app": "anti"}}, "topologyKey": ZONE}]}},
            "topologySpreadConstraints": [
                {"topologyKey": HOST, "maxSkew": 1, "whenUnsatisfiable": "ScheduleAnyway", "labelSelector": web},
                {"topologyKey": RACK, "maxSkew": 1, "whenUnsatisfiable": "ScheduleAnyway", "labelSelector": web}]}
    apps = [O.AppResource("fill", O.ResourceTypes(Deployments=fills)),
            O.AppResource("anti", O.ResourceTypes(Deployments=[_dep("anti", 2, {"app": "anti", "tier": "web"}, spec)]))]
    p = simulator.plan(O.ResourceTypes(Nodes=nodes), apps)
    return compile_cluster(p.nodes, p.pods, p.ctx)


@pytest.mark.parametrize("n_a", [3000, 50000, 65537])
def test_zone_flip_under_hostname_spread_redoes_the_spread_pass(n_a):
    """n_a = 3,000 (forced onto the large variant): just past the 12-bit net-change field; 50,000: the dc range past 16 bits as
    well; 65,537: at the old flip-count wrap."""
    c = spread_case(n_a)
    names = c.node_names
    ref, rscore = oracle_full(c)[:2]
    assert [names[g] for g in ref[4:]] == ["a000000", "b0"] and rscore[5] > 0, (ref, rscore)
    with _engine(c, force_large=True) as eng:
        a = eng.schedule(0, 4)
        b = eng.schedule(4, 2)
        out, score = np.concatenate([a[0], b[0]]), np.concatenate([a[1], b[1]])
        li = eng.last_launch()
        assert li["kernel"] == "simon_place_kernel_big" and li["large"], li
        if n_a + 2 > 20480:
            _assert_large(li, n_a + 2)
        st = eng.stats()        # of the second call: the two replicas
        _assert_run(c, eng, out, score, b[2], b[3], f"spread {n_a}")
    assert names[out[5]] == "b0"
    # replica 1: first visit of the class; replica 2: n_a flips, a full summary whose size check fails and redoes the spread pass
    assert st["decisions"] == 2 and st["redone"] == 1 and st["single_flip_fast"] == 0 and st["summary_rebuilds"] == 2, st


# ---- the families at 70,000 nodes and at the 327,680-node cap ----------------------------------------------------------------

# C3 with GPU-share devices on ~20 % of the nodes, GPU-share requests and DoNotSchedule zone spreads on some workloads
SIZES = {"70k": dict(n_nodes=70000, n_workloads=40, replicas=10, n_apps=2, seed_no=7, gpu_pct=20),
         "cap": dict(n_nodes=327680, n_workloads=20, replicas=10, n_apps=2, seed_no=7, gpu_pct=20)}


@functools.lru_cache(maxsize=None)
def family_case(size):
    cluster, apps = synth.make_c3(**SIZES[size])
    p = simulator.plan(cluster, apps)
    return compile_cluster(p.nodes, p.pods, p.ctx)


def _free_pods(c):
    """Pods that reach the scheduler (not bound by spec.nodeName): the placement decisions, as opposed to the pre-bound prefill."""
    return c.pods["pod_fixed_node"] == -1


@pytest.mark.parametrize("size", sorted(SIZES))
def test_single_run(size):
    c = family_case(size)
    with _engine(c) as eng:
        out, score, fc, fp = eng.schedule()
        _assert_large(eng.last_launch(), c.n_nodes)
        _assert_run(c, eng, out, score, fc, fp, size)
    free = _free_pods(c)
    assert (free & (out >= 0)).sum() >= 150 and (free & (score > 0)).sum() >= 150
    assert (oracle_full(c)[6] != 0).sum() > 0       # GPU-share pods hold device slots


def test_single_run_without_static_cache():
    c = family_case("70k")
    with _engine(c, static_cache=False) as eng:
        out, score, fc, fp = eng.schedule()
        _assert_large(eng.last_launch(), c.n_nodes)
        _assert_run(c, eng, out, score, fc, fp, "70k static_cache=False")


@pytest.mark.parametrize("size", sorted(SIZES))
def test_resume_from_half(size):
    """simon_schedule_resume from the oracle's placement up to half of the placement decisions (all the pre-bound prefill comes
    first): the replay walks the prefix's counts, GPU-share device slots included, then the rest is placed."""
    c = family_case(size)
    ref, rscore, _fc, _fp, rst, rext, rslots = oracle_full(c)
    free = np.nonzero(_free_pods(c))[0]
    h = int(free[len(free) // 2])
    assert (rslots[:h] != 0).any() and (rslots[h:] != 0).any()
    with _engine(c) as eng:
        out, score, _, _ = eng.schedule_resume(ref[:h])
        _assert_large(eng.last_launch(), c.n_nodes)
        np.testing.assert_array_equal(out, ref)
        sched = ref[h:] >= 0
        np.testing.assert_array_equal(score[h:][sched], rscore[h:][sched])
        st, ext = eng.state(), eng.state_ext()
        for k in rst:
            np.testing.assert_array_equal(st[k], rst[k], err_msg=k)
        for k in rext:
            np.testing.assert_array_equal(ext[k], rext[k], err_msg=k)
        np.testing.assert_array_equal(eng.gpu_slot_words()[h:], rslots[h:])


@pytest.mark.parametrize("size", sorted(SIZES))
def test_scenario_batch(size):
    """Node lists: all nodes, every other node, and a subset of 65,537 + 1,000 active nodes (still past the wrap): nodes,
    unscheduled counts and the occupancy sums."""
    from oracle.binding import Oracle
    c = family_case(size)
    n = c.n_nodes
    lists = [np.arange(n), np.arange(0, n, 2), np.random.default_rng(3).permutation(n)[:66537]]
    with _engine(c) as eng:
        res, nodes = eng.run_scenarios(lists, want_nodes=True)
        _assert_large(eng.last_launch(), n, len(lists))
    o = Oracle(c, threads=THREADS)
    for i, act in enumerate(lists):
        o.set_active(act)
        o.reset()
        ref = o.schedule()[0]
        st = o.state()
        np.testing.assert_array_equal(nodes[i], ref, err_msg=f"{size} scenario {i}")
        assert res[i]["n_unscheduled"] == int((ref == -1).sum()), i
        assert (res[i]["req_mcpu"], res[i]["req_mem"]) == (int(st["req_mcpu"][act].sum()), int(st["req_mem"][act].sum())), i
    o.close()


def _live(size):
    """The case, a fresh oracle on it and the oracle's placement (each checker gets an oracle of its own)."""
    from oracle.binding import Oracle
    c = family_case(size)
    o = Oracle(c, threads=THREADS)
    return c, o, o.schedule()[0]


@pytest.mark.parametrize("size", sorted(SIZES))
def test_drains(size):
    import checkers
    from simon_b200 import scaledown
    from test_drain import _assert_drain_equal
    c, o, placed = _live(size)
    rng = np.random.default_rng(7)
    order = scaledown.NodeOrder(c)
    used = np.unique(placed[_free_pods(c) & (placed >= 0)])      # nodes holding pods the scheduler placed
    drains = [[int(g)] for g in rng.choice(used, 3, replace=False)] + [rng.choice(c.n_nodes, 500, replace=False).tolist()]
    remain = [order.remaining(d) for d in drains]
    with _engine(c) as eng:
        got = eng.drain_run(placed, remain)
        for li in eng.last_drain["launches"]:
            _assert_large(li, c.n_nodes, li["n_scenarios"])
    for d, rl, g in zip(drains, remain, got):
        want = checkers.drain(o, placed, rl)
        _assert_drain_equal(g, want, f"drain of {len(d)} nodes")
        pos = g["node"] >= 0
        np.testing.assert_array_equal(g["score"][pos], want["score"][pos])
    assert sum(g["n_evicted"] for g in got) > 0
    o.close()


@pytest.mark.parametrize("size", sorted(SIZES))
def test_probes(size):
    import checkers
    from test_zz_headroom_gpu import _probe_pods
    c, o, placed = _live(size)      # an oracle of its own: see test_open_local_place_drain_probe_70k
    probes = list(zip(_probe_pods(c, np.random.default_rng(11), 4), (1, 7, 40, 200)))
    with _engine(c) as eng:
        got = eng.probe_run(placed, probes)
        for li in eng.last_probe["launches"]:
            _assert_large(li, c.n_nodes, li["n_scenarios"])
    for (q, r), g in zip(probes, got):
        want = checkers.probe(o, placed, q, r)
        assert (g["n_placed"], g["stop_reason"]) == (want["n_placed"], want["stop_reason"]), (q, r)
        for k in ("node", "score", "gpu_slots", "fail_counts"):
            np.testing.assert_array_equal(g[k], want[k], err_msg=f"probe {q} of {r}: {k}")
    assert sum(g["n_placed"] for g in got) > 4
    o.close()


def test_sampled_moves_70k():
    """20,000 sampled moves (the move kernels have no large variant of their own: they score every node of a 70,000-node cluster)
    against the scoped checker, with the default scope and with GPU-share and hard-spread classes admitted."""
    from simon_b200 import abi as A, moves as M
    from test_moves_scope import _engine_vs_checker
    c, o, out = _live("70k")
    mv = M.sample_moves(len(out), c.n_nodes, 20000, seed=5, placement=out).astype(np.uint32)
    n_feasible = 0
    for scope in (0, A.MOVES_SCOPE_GPU_SHARE | A.MOVES_SCOPE_HARD_SPREAD):
        code = _engine_vs_checker(c, o, out, mv, scope)
        n_feasible += int((code == 0).sum())
    assert n_feasible > 0
    o.close()


# ---- Open-Local above 65,536 nodes: simon_local_kernel_big, simon_drain_local_kernel_big, simon_probe_local_kernel_big ----------

@functools.lru_cache(maxsize=None)
def local_case():
    """synth.make_open_local on 70,000 nodes: VGs and SSD / HDD devices on ~60 % of them, 288 pods of which 216 request LVM
    volumes, devices or both."""
    from test_drain_local import _synth_compiled
    return _synth_compiled(70000, 5)[1]


@functools.lru_cache(maxsize=None)
def local_oracle_full():
    from oracle.binding import Oracle
    o = Oracle(local_case(), threads=THREADS, open_local=True)
    try:
        return o.schedule() + (o.state(), o.state_ext(), o.gpu_slot_words()) + o.storage_state()
    finally:
        o.close()


def test_open_local_place_drain_probe_70k():
    import checkers
    from oracle.binding import Oracle
    from simon_b200 import scaledown
    from test_zz_headroom_gpu import _probe_pods
    from test_zz_open_local_oracle_gpu import assert_engine_matches
    c = local_case()
    st = c.storage
    ref = local_oracle_full()
    placed = ref[0]
    with _engine(c) as eng:
        out, score, fc, fp = eng.schedule()
        li = eng.last_launch()
        assert li["kernel"] == "simon_local_kernel_big" and li["local"], li
        _assert_large(li, c.n_nodes)
        assert_engine_matches(ref, eng, out, score, fc, fp, "open-local 70k")
    local_pods = st.class_local[c.pods["pod_class"]].astype(bool) & (placed >= 0) & (c.pods["pod_fixed_node"] == -1)
    assert local_pods.sum() > 0
    o = Oracle(c, threads=THREADS, open_local=True)
    try:
        # drains: three nodes that hold pods with local volumes, one at a time, and 300 nodes at once
        rng = np.random.default_rng(5)
        hold = np.unique(placed[local_pods])
        drains = [[int(g)] for g in rng.choice(hold, 3, replace=False)] + [rng.choice(c.n_nodes, 300, replace=False).tolist()]
        order = scaledown.NodeOrder(c)
        remain = [order.remaining(d) for d in drains]
        with _engine(c) as eng:
            got = eng.drain_run(placed, remain, local=True)
            for li in eng.last_drain["launches"]:
                assert li["kernel"] == "simon_drain_local_kernel_big", li
                _assert_large(li, c.n_nodes, li["n_scenarios"])
            states = [eng.scenario_storage_state(i) for i in range(len(drains))] if eng.last_drain["chunks"] == 1 else None
        for j, (d, rl, g) in enumerate(zip(drains, remain, got)):
            want = checkers.drain(o, placed, rl)
            for k in ("n_evicted", "n_placed", "n_unscheduled", "n_blocked", "n_vanished"):
                assert g[k] == want[k], (d, k)
            for k in ("evicted", "node", "score", "gpu_slots", "blocked", "fail_pod", "fail_counts"):
                np.testing.assert_array_equal(g[k], want[k], err_msg=f"drain {d}: {k}")
            vg, dev = o.storage_state()
            if states is not None:
                rl = np.asarray(rl)
                np.testing.assert_array_equal(states[j][0][:, rl], vg[:, rl], err_msg=f"drain {d}: VG state")
                if dev is not None:
                    np.testing.assert_array_equal(states[j][1][rl], dev[rl], err_msg=f"drain {d}: device state")
    finally:
        o.close()
    # probes, on an oracle of their own (the probe checker starts from the state the oracle holds, and the drain checker leaves it changed)
    o = Oracle(c, threads=THREADS, open_local=True)
    try:
        # pods with local volumes and without
        qs = _probe_pods(c, np.random.default_rng(9), 60)
        loc = [q for q in qs if st.class_local[int(c.pods["pod_class"][q])]][:3]
        plain = [q for q in qs if not st.class_local[int(c.pods["pod_class"][q])]][:2]
        assert loc
        probes = [(q, r) for q, r in zip(loc + plain, (1, 8, 30, 5, 60))]
        with _engine(c) as eng:
            gotp = eng.probe_run(placed, probes)
            for li in eng.last_probe["launches"]:
                assert li["kernel"] == "simon_probe_local_kernel_big", li
                _assert_large(li, c.n_nodes, li["n_scenarios"])
            pstates = [eng.scenario_storage_state(i) for i in range(len(probes))] if eng.last_probe["chunks"] == 1 else None
        for j, ((q, r), g) in enumerate(zip(probes, gotp)):
            want = checkers.probe(o, placed, q, r)
            assert (g["n_placed"], g["stop_reason"]) == (want["n_placed"], want["stop_reason"]), (q, r)
            for k in ("node", "score", "gpu_slots", "fail_counts"):
                np.testing.assert_array_equal(g[k], want[k], err_msg=f"probe {q} of {r}: {k}")
            vg, dev = o.storage_state()
            if pstates is not None:
                np.testing.assert_array_equal(pstates[j][0], vg, err_msg=f"probe {q}: VG state")
    finally:
        o.close()
