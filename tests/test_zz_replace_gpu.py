"""Node-pool replacement on the device (simon_wave_begin_pool / simon_wave_run_join / simon_wave_commit_retire, Engine.wave_*,
Simulator.PlanNodeReplacement) against the wave checker (tests/checkers.c): whole plans run in lockstep on both, every
batch and every committed base compared, at the four drain geometries, without the static-verdict cache and with PDBs; every wave
batch against the compile-and-resume definition on clusters without GPU share; a GPU-share case where a rebuild would give a moved pod
another device; the C-entry refusals; session safety."""
import copy
import re

import numpy as np
import pytest

import checkers
from simon_b200 import objects as O, replace, rolling, synth
from simon_b200.quantity import Quantity
from test_grow import session
from test_replace import _cluster, _dep, _spec
from test_zz_rolling_gpu import GEOMETRIES, _gpu_node, _gpu_pod, _pdbs_of_mix

pytestmark = pytest.mark.gpu

JOIN_KEYS = ("join_pods", "join_node", "join_gpu_slots", "join_score", "join_fail_pod", "join_fail_counts")


class LockstepRunner(rolling.WaveRunner):
    """The engine, checked at every step against the checker: each batch's evicted and join results and, after each commit, the
    base's placement, slot words, node states, node aggregates, scalars and GPU memory."""

    def __init__(self, eng, o, pdbs=None, kernel=None):
        self.eng, self.chk, self.kernel = eng, checkers.OracleRunner(o, pdbs), kernel
        self.dev = rolling.EngineRunner(eng)
        self.batches = self.commits = 0

    def begin(self, placed, present=None):
        self.dev.begin(placed, present)
        self.chk.begin(placed, present)
        self._check_base()

    def run(self, remain_lists, joins=None):
        got = self.dev.run(remain_lists, joins)
        want = self.chk.run(remain_lists, joins)
        if self.kernel:
            assert self.eng.last_launch()["kernel"] == self.kernel
        for i, (g, w) in enumerate(zip(got, want)):
            for k in ("n_evicted", "n_placed", "n_unscheduled", "n_blocked", "n_vanished", "n_pdb_violated", "req_mcpu", "req_mem",
                      "alloc_mcpu", "alloc_mem", "n_join", "n_join_placed", "n_join_unscheduled"):
                assert g[k] == w[k], (self.batches, i, k)
            for k in ("evicted", "node", "gpu_slots", "score", "blocked", "fail_pod", "fail_counts", "pdb_violated", "pdb_evicted") + JOIN_KEYS:
                assert np.array_equal(np.asarray(g[k]), np.asarray(w[k])), (self.batches, i, k)
        self.batches += 1
        return got

    def commit(self, i, retire=False):
        self.dev.commit(i, retire)
        self.chk.commit(i, retire)
        self.commits += 1
        self._check_base()

    def _check_base(self):
        pl, sl = self.dev.placement()
        cpl, csl = self.chk.placement()
        assert np.array_equal(pl, cpl) and np.array_equal(sl, csl)
        assert np.array_equal(self.eng.wave_presence(), self.chk.state)
        st, want = self.eng.state(), self.chk.o.state()
        for k, v in want.items():
            assert np.array_equal(st[k], v), k
        ext, wext = self.eng.state_ext(), self.chk.o.state_ext()
        for k, v in wext.items():
            assert np.array_equal(ext[k], v), k

    def placement(self):
        return self.dev.placement()


def _bigger(node, factor=2):
    """A copy of a node object with `factor` times its cores and memory, under a new name."""
    n = copy.deepcopy(node)
    n["metadata"]["name"] = "replacement"
    for part in ("allocatable", "capacity"):
        al = n["status"].get(part)
        if al:
            al["cpu"] = f"{Quantity.parse(al['cpu']).milli_value() * factor}m"
            al["memory"] = str(Quantity.parse(al["memory"]).int_value() * factor)
    return n


def _lockstep(sim, nodes, spec, eng_kw=None, pdb_objs=None, kernel=None, **kw):
    from oracle.binding import Oracle
    from simon_b200.disruption import compile_pdbs
    from simon_b200.engine import Engine
    c, placed, present, pool, copies, pdbs = replace.superset(sim, nodes, spec, kw.pop("kmax", len(nodes)))
    if pdb_objs:
        pdbs = compile_pdbs(pdb_objs, c)
    o = Oracle(c, threads=8)
    checkers.grow(o, placed, len(sim.placements), np.nonzero(present)[0].astype(np.uint32))
    with Engine(c, record_scores=True, **(eng_kw or {})) as eng:
        if pdbs is not None:
            eng.pdbs_upload(pdbs)
        r = LockstepRunner(eng, o, pdbs, kernel)
        plan = replace.plan_replacement(c, placed, r, present, pool, copies, caps=(100, 100), pdbs=pdbs, **kw)
        info = dict(eng.last_wave)
    o.close()
    return plan, r, info


def _mix_session(seed, n_nodes=40):
    cluster, apps = synth.make_mix(seed_no=seed, n_nodes=n_nodes)
    return session(cluster, apps), cluster


@pytest.mark.parametrize("kernel", sorted(GEOMETRIES))
def test_plans_match_checker_at_forced_geometries(kernel):
    cs, t, big = GEOMETRIES[kernel]
    for seed in (0, 3):
        sim, cluster = _mix_session(seed)
        names = list(sim.compiled.node_names)
        pool = names[:8]
        plan, r, info = _lockstep(sim, pool, _bigger(cluster.Nodes[0]), dict(cluster_ctas=cs, threads_per_cta=t, force_large=big),
                                  kernel=kernel, max_surge=2, max_unavailable=1)
        assert r.batches >= 1 + plan.TotalWaves and r.commits == plan.TotalWaves
        assert plan.TotalWaves + len(plan.Skipped) > 0


def test_plans_match_checker_without_static_cache_and_with_pdbs():
    from simon_b200 import simulator
    for seed in (1, 2):
        sim, cluster = _mix_session(seed)
        pool = list(sim.compiled.node_names)[-10:]
        p = simulator.plan(*synth.make_mix(seed_no=seed, n_nodes=40))
        from simon_b200.compiler import compile_cluster
        pdb_objs = _pdbs_of_mix(compile_cluster(p.nodes, p.pods, p.ctx))
        plan, r, _ = _lockstep(sim, pool, _bigger(cluster.Nodes[-1]), dict(static_cache=False), pdb_objs=pdb_objs, max_surge=1,
                               max_unavailable=2)
        assert r.commits == plan.TotalWaves
        _lockstep(sim, pool, _bigger(cluster.Nodes[-1], 1), pdb_objs=pdb_objs, max_surge=3, max_unavailable=0, order="given")


def test_hand_cases_match_checker():
    sim = session(_cluster([_dep("web", 6)]))
    plan, r, _ = _lockstep(sim, ["old-0", "old-1"], _spec("big", "5000m"))
    assert plan.Sizing.MinNodes == 2 and plan.TotalWaves == 2 and plan.MovedPods == 6
    plan, r, _ = _lockstep(sim, ["old-0", "old-1"], _spec("tiny", "100m"), kmax=2)
    assert plan.Sizing.MinNodes == -1 and plan.TotalWaves == 0


def test_c_entry_refusals():
    from oracle.binding import Oracle  # noqa: F401  (the checker builds alongside)
    from simon_b200.engine import Engine, lib
    sim = session(_cluster([_dep("web", 2)]))
    c, placed, present, pool, copies, pdbs = replace.superset(sim, ["old-0", "old-1"], _spec("big"), 2)
    a, b = copies
    with Engine(c) as eng:
        with pytest.raises(RuntimeError, match="without a wave base"):
            eng.wave_run([np.array([0, 1, a], np.uint32)], [np.array([a], np.uint32)])
        bad = placed.copy()
        bad[len(sim.placements)] = a             # a copy's DaemonSet pod placed on an absent node
        with pytest.raises(RuntimeError, match="not present"):
            eng.wave_begin(bad, present)
        eng.wave_begin(placed, present)
        with pytest.raises(RuntimeError, match="not in its remaining nodes"):
            eng.wave_run([np.array([0, 1], np.uint32)], [np.array([a], np.uint32)])
        with pytest.raises(RuntimeError, match="absent and does not join"):
            eng.wave_run([np.array([0, 1, a, b], np.uint32)], [np.array([a], np.uint32)])
        with pytest.raises(RuntimeError, match="not absent"):
            eng.wave_run([np.array([0, 1], np.uint32)], [np.array([0], np.uint32)])
        with pytest.raises(RuntimeError, match="absent and does not join"):
            eng.wave_run([np.array([0, a], np.uint32)])
        res = eng.wave_run([np.array([1, a], np.uint32)], [np.array([a], np.uint32)])
        assert res[0]["n_join"] == 1 and res[0]["n_join_unscheduled"] == 0
        with pytest.raises(RuntimeError, match="joined nodes"):
            eng.wave_commit(0)
        eng.wave_commit(0, retire=True)
        assert eng.wave_presence().tolist() == [2, 1, 1, 0]
        with pytest.raises(RuntimeError, match="retired"):
            eng.wave_run([np.array([0, 1, a], np.uint32)])
        with pytest.raises(RuntimeError, match="no wave batch"):
            eng._check(lib().simon_wave_commit_retire(eng.h, 0))
        # the old node's DaemonSet pod no longer exists; the copy's runs on it
        pl, _ = eng.wave_placement()
        guard = np.asarray(c.pods["pod_fixed_node"])
        recs = c.pod_recs
        agents = {recs[q].name: int(pl[q]) for q in range(len(recs)) if recs[q].name.startswith("agent")}
        assert sorted(agents.values()) == sorted([-3, 1, a, -1]), (agents, guard)


class ResumeCheckRunner(rolling.EngineRunner):
    """The engine's runner whose every wave batch is checked against the definition: remain compiled with the pod list [pods placed
    on remain in the base] + [join pods] + [evicted pods], resumed after the first part, gives the same nodes, GPU slot words and
    failure records (join pods' first, as the wave lists them)."""

    def __init__(self, eng, sim):
        super().__init__(eng)
        self.sim, self.c, self.checked = sim, eng.c, 0

    def run(self, remain_lists, joins=None):
        from simon_b200.compiler import compile_cluster
        from simon_b200.engine import Engine
        got = super().run(remain_lists, joins)
        base = self.placement()[0]
        c = self.c
        ctx = self.sim._plan().ctx
        for rl, r in zip(remain_lists, got):
            rl = np.asarray(rl).tolist()
            on = set(rl)
            stay = [q for q in range(len(base)) if base[q] >= 0 and int(base[q]) in on]
            order = stay + r["join_pods"].tolist() + r["evicted"].tolist()
            nodes = [c.node_objs[g] for g in sorted(rl, key=lambda g: c.node_orig_index[g])]
            c2 = compile_cluster(nodes, [c.pod_recs[q] for q in order], ctx)
            assert c2.node_names == [c.node_names[g] for g in rl]
            to2 = {g: i for i, g in enumerate(rl)}
            with Engine(c2, record_scores=True) as e2:
                out, _score, fc, fp = e2.schedule_resume(np.array([to2[int(base[q])] for q in stay], np.int32))
                slots = e2.gpu_slot_words()
            n0, nj = len(stay), len(r["join_pods"])
            back = lambda v: np.array([rl[x] if x >= 0 else x for x in v.tolist()], np.int32)   # noqa: E731
            assert np.array_equal(back(out[n0:n0 + nj]), r["join_node"]) and np.array_equal(back(out[n0 + nj:]), r["node"])
            assert np.array_equal(slots[n0:n0 + nj], r["join_gpu_slots"]) and np.array_equal(slots[n0 + nj:], r["gpu_slots"])
            assert np.array_equal(fc, np.concatenate([r["join_fail_counts"], r["fail_counts"]]))
            assert [order[q] for q in fp.tolist()] == r["join_fail_pod"].tolist() + r["fail_pod"].tolist()
            self.checked += 1
        return got


def _strip_gpu_share(cluster):
    for n in cluster.Nodes:
        for sect in ("allocatable", "capacity"):
            n["status"].get(sect, {}).pop("alibabacloud.com/gpu-count", None)
            n["status"].get(sect, {}).pop("alibabacloud.com/gpu-mem", None)
    return cluster


def test_wave_batches_equal_compile_and_resume():
    """Without GPU share every wave batch of a plan (sizing, joins and retirements) equals the compile-and-resume definition."""
    from simon_b200.engine import Engine
    for seed in (2, 6):
        cluster, apps = synth.make_mix(seed_no=seed, n_nodes=30)
        sim = session(_strip_gpu_share(cluster), apps)
        names = list(sim.compiled.node_names)
        c, placed, present, pool, copies, _ = replace.superset(sim, names[:6], _bigger(cluster.Nodes[0]), 6)
        with Engine(c, record_scores=True) as eng:
            r = ResumeCheckRunner(eng, sim)
            plan = replace.plan_replacement(c, placed, r, present, pool, copies, count=6, caps=(100, 100), max_surge=2,
                                            max_unavailable=1)
        assert plan.TotalWaves > 0 and plan.JoinedNodes > 0 and r.checked > plan.TotalWaves


def test_gpu_share_wave_follows_the_carried_devices():
    """node-x has two 12 GiB devices, pods p1 and p2 (6 GiB each) sit on its device 0; p0 (5 GiB, first in pod order) sits on node-y,
    which it prefers.  Replacing node-y by a copy without GPUs (count 1) joins the copy, whose DaemonSet pod runs there, and moves p0
    to node-x, where only device 1 has room.  A pod-order rebuild of the final placement gives p0 device 0."""
    from simon_b200.engine import Engine
    nodes = [_gpu_node("node-x", 24, 2), _gpu_node("node-y", 24, 2)]
    pods = [_gpu_pod("p0", "node-y", 5), _gpu_pod("p1", "node-x", 6), _gpu_pod("p2", "node-x", 6)]
    na = pods[0]["spec"]["affinity"]["nodeAffinity"]
    na["preferredDuringSchedulingIgnoredDuringExecution"] = [
        {"weight": 100, "preference": na.pop("requiredDuringSchedulingIgnoredDuringExecution")["nodeSelectorTerms"][0]}]
    from test_grow import _ds
    sim = session(O.ResourceTypes(Nodes=nodes, Pods=pods, DaemonSets=[_ds("agent")]))
    x, y = sim.compiled.node_index("node-x"), sim.compiled.node_index("node-y")
    q0 = next(q for q, rec in enumerate(sim.compiled.pod_recs) if rec.name == "p0")
    assert sim.placements[q0] == y and int(sim.gpu_slots[q0]) == 1
    plan, r, _ = _lockstep(sim, ["node-y"], _spec("plain"), count=1, max_surge=1, max_unavailable=0, order="given")
    assert [w.Nodes for w in plan.Waves] == [["node-y"]] and len(plan.Waves[0].Joined) == 1
    assert [(p.Pod.name.split("-")[0], p.Node) for p in plan.Waves[0].JoinPods] == [("agent", plan.Waves[0].Joined[0])]
    assert [(e.Pod.name, e.To, e.GpuIndex) for e in plan.Waves[0].Evicted] == [("p0", "node-x", "1")]
    assert plan.FinalPlacement["default/p0"] == ("node-x", "1")
    final, slots = r.chk.placement()          # equal to the engine's base at every commit (LockstepRunner)
    assert int(slots[q0]) == 1 << 4
    with Engine(r.chk.o.c) as e2:
        e2.schedule_resume(np.where(final == -3, -1, final))
        assert int(e2.gpu_slot_words()[q0]) == 1           # the pod-order replay: device 0


def test_more_c_entry_refusals():
    from simon_b200.engine import Engine
    # a join pod bound by spec.nodeName: the superset's first copy's DaemonSet pod marked bound to a present node
    sim = session(_cluster([_dep("web", 2)]))
    c, placed, present, pool, copies, _ = replace.superset(sim, ["old-0", "old-1"], _spec("big"), 2)
    a, b = copies
    with Engine(c) as eng:
        eng.wave_begin(placed, present)
        for join, msg in (([c.n_nodes], "out of range"), ([a, a], "twice")):
            with pytest.raises(RuntimeError, match=msg):
                eng.wave_run([np.array([0, 1, a], np.uint32)], [np.array(join, np.uint32)])
    q = next(q for q in range(len(sim.placements), c.pods_dims["n_pods"]) if np.asarray(c.pods["pod_pin_node"])[q] == a)
    bound = copy.copy(c)
    bound.pods = dict(c.pods)
    bound.pods["pod_fixed_node"] = np.array(c.pods["pod_fixed_node"]).copy()
    bound.pods["pod_fixed_node"][q] = 0
    pl = placed.copy()
    pl[q] = 0
    with Engine(bound) as eng:
        eng.wave_begin(pl, present)
        with pytest.raises(RuntimeError, match="bound by spec.nodeName"):
            eng.wave_run([np.array([0, 1, a], np.uint32)], [np.array([a], np.uint32)])
    # a join pod with Open-Local volumes
    import test_open_local_oracle as T
    from simon_b200 import simulator
    cl = _cluster([_dep("web", 2)], ds=False)
    ds = _ds_local()
    T._annotate(ds["spec"]["template"].setdefault("metadata", {}), [{"size": str(5 << 30), "kind": "LVM", "scName": "open-local-lvm"}])
    cl.DaemonSets.append(ds)
    cl.StorageClasss.extend(T.STORAGE_CLASSES)
    sim = session(cl, (), simulator.WithOpenLocal(devices=True))
    c, placed, present, pool, copies, _ = replace.superset(sim, ["old-0", "old-1"], _spec("big"), 1)
    with Engine(c) as eng:
        eng.wave_begin(placed, present)
        with pytest.raises(RuntimeError, match="Open-Local volumes"):
            eng.wave_run([np.array([0, 1, copies[0]], np.uint32)], [np.array(copies, np.uint32)])
    # a batch that joins a node without DaemonSet pods still joins it: simon_wave_commit refuses it
    sim = session(_cluster([_dep("web", 2)], ds=False))
    c, placed, present, pool, copies, _ = replace.superset(sim, ["old-0", "old-1"], _spec("big"), 1)
    with Engine(c) as eng:
        eng.wave_begin(placed, present)
        res = eng.wave_run([np.array([1, copies[0]], np.uint32)], [np.array(copies, np.uint32)])
        assert res[0]["n_join"] == 0
        with pytest.raises(RuntimeError, match="joined nodes"):
            eng.wave_commit(0)
        eng.wave_commit(0, retire=True)
        assert eng.wave_presence().tolist() == [2, 1, 1]


def _ds_local():
    from test_grow import _ds
    return _ds("store")


def test_pending_daemonset_pods_of_a_retired_node_stop_existing():
    """A DaemonSet pod that was pending on an old node (too large for it) does not exist once its node retires."""
    from test_grow import _ds
    cl = _cluster([_dep("web", 2)])
    cl.DaemonSets.append(_ds("huge", cpu="9000m"))
    sim = session(cl)
    plan, r, _ = _lockstep(sim, ["old-0", "old-1"], _spec("big", "16000m"), count=2, max_surge=1)
    assert plan.TotalWaves == 2
    final, _ = r.chk.placement()              # equal to the engine's base at every commit (LockstepRunner)
    recs = r.chk.o.c.pod_recs
    for q, rec in enumerate(recs):
        if rec.name.startswith("huge") and "old" in rec.name:
            assert final[q] == -3, rec.name


def test_session_answers_unchanged_by_a_plan():
    from simon_b200 import simulator
    cluster, apps = synth.make_mix(seed_no=0, n_nodes=24)
    sim = simulator.NewSimulator(simulator.WithPodDisruptionBudgets())
    sim.RunCluster(cluster)
    for app in apps:
        sim.ScheduleApp(app)
    names = list(sim.compiled.node_names)
    pod = next(f"{r.tmpl.namespace}/{r.name}" for q, r in enumerate(sim.compiled.pod_recs) if sim.placements[q] >= 0)
    wl = next(f"{r.tmpl.workload_kind}/{r.tmpl.workload_namespace}/{r.workload_name}" for r in sim.compiled.pod_recs
              if r.tmpl.workload_kind in ("ReplicaSet", "StatefulSet"))

    def answers():
        m = sim.PlanMigrations(max_moves=5)
        m.KernelMs = 0.0                                               # a device time, not an answer
        return (repr(sim.DrainNodes([names[:2]])), repr(sim.PlanRollingMaintenance(names[:3])), repr(m),
                repr(sim.Headroom([wl], max_replicas=50)), repr(sim.Explain([pod])[0]))
    before = answers()
    placements = sim.placements.copy()
    plan = sim.PlanNodeReplacement(names[:4], _bigger(cluster.Nodes[0]), max_surge=2)
    assert plan.Count == (plan.Sizing.MinNodes if plan.Sizing.MinNodes >= 0 else 4)
    assert np.array_equal(sim.placements, placements)
    assert answers() == before
    sim.Close()
