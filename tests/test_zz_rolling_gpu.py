"""Rolling node maintenance on the device (simon_wave_*, Engine.wave_*, Simulator.PlanRollingMaintenance) against the wave checker
(tests/checkers.c): full plans run in lockstep on both, every batch and every committed base compared; wave batches against
simon_drain_run from the same placement; a GPU-share case where a rebuild would give a moved pod other devices; session safety."""
import numpy as np
import pytest

from simon_b200 import abi, objects as O, rolling, simulator, synth
from simon_b200.compiler import compile_cluster

pytestmark = pytest.mark.gpu

# (CTAs per scenario, threads per CTA, force_large): the geometries the drain GPU tests force, one per drain kernel
GEOMETRIES = {"simon_drain_kernel_256": (2, 128, False), "simon_drain_kernel_320": (2, 288, False),
              "simon_drain_kernel_384": (1, 352, False), "simon_drain_kernel_big": (4, 64, True)}


def _plan_compiled(cluster, apps):
    p = simulator.plan(cluster, apps)
    return p, compile_cluster(p.nodes, p.pods, p.ctx)


class LockstepRunner(rolling.WaveRunner):
    """The engine, checked at every step against the checker: each batch's results (counts, evicted pods, nodes, GPU slot words,
    scores, blocked pods, failures, requested sums) and, after each commit, the base's placement, slot words, node aggregates and
    scalars and GPU memory.  drain_eng: a second engine on the same cluster, whose simon_drain_run from the base placement must give
    the same batch (clusters without GPU share)."""

    def __init__(self, eng, o, pdbs=None, drain_eng=None, kernel=None):
        import checkers
        self.eng, self.chk, self.drain_eng, self.kernel = eng, checkers.OracleRunner(o, pdbs), drain_eng, kernel
        self.dev = rolling.EngineRunner(eng)
        self.batches = 0

    def begin(self, placed):
        self.dev.begin(placed)
        self.chk.begin(placed)
        self._check_base()

    def run(self, remain_lists):
        got = self.dev.run(remain_lists)
        want = self.chk.run(remain_lists)
        if self.kernel:
            assert self.eng.last_launch()["kernel"] == self.kernel
        for i, (g, w) in enumerate(zip(got, want)):
            for k in ("n_evicted", "n_placed", "n_unscheduled", "n_blocked", "n_vanished", "n_pdb_violated", "req_mcpu", "req_mem",
                      "alloc_mcpu", "alloc_mem"):
                assert g[k] == w[k], (self.batches, i, k)
            for k in ("evicted", "node", "gpu_slots", "score", "blocked", "fail_pod", "fail_counts", "pdb_violated", "pdb_evicted"):
                assert np.array_equal(np.asarray(g[k]), np.asarray(w[k])), (self.batches, i, k)
        if self.drain_eng is not None:
            base = self.dev.placement()[0]
            ref = self.drain_eng.drain_run(base, remain_lists, detail=True)
            for i, (g, r) in enumerate(zip(got, ref)):
                for k, v in r.items():
                    assert np.array_equal(np.asarray(g[k]), np.asarray(v)), ("drain_run", self.batches, i, k)
        self.batches += 1
        return got

    def commit(self, i):
        self.dev.commit(i)
        self.chk.commit(i)
        self._check_base()

    def _check_base(self):
        pl, sl = self.dev.placement()
        cpl, csl = self.chk.placement()
        assert np.array_equal(pl, cpl) and np.array_equal(sl, csl)
        st, want = self.eng.state(), self.chk.o.state()
        for k, v in want.items():
            assert np.array_equal(st[k], v), k
        ext, wext = self.eng.state_ext(), self.chk.o.state_ext()
        for k, v in wext.items():
            assert np.array_equal(ext[k], v), k

    def placement(self):
        return self.dev.placement()


def _lockstep_plan(c, eng_kw=None, b=3, pdb_objs=None, drain_check=False, kernel=None, **kw):
    from oracle.binding import Oracle
    from simon_b200.disruption import compile_pdbs
    from simon_b200.engine import Engine
    eng_kw = dict(eng_kw or {})
    o = Oracle(c, threads=8)
    placed = o.schedule()[0]
    pdbs = compile_pdbs(pdb_objs, c) if pdb_objs else None
    with Engine(c, record_scores=True, **eng_kw) as eng:
        out = eng.schedule()[0]
        assert np.array_equal(out, placed)
        if pdbs is not None:
            eng.pdbs_upload(pdbs)
        drain_eng = Engine(c, record_scores=True) if drain_check else None
        try:
            if drain_eng is not None and pdbs is not None:
                drain_eng.pdbs_upload(pdbs)
            r = LockstepRunner(eng, o, pdbs, drain_eng, kernel)
            plan = rolling.plan_rolling(c, placed, r, max_unavailable=b, caps=(100, 100), pdbs=pdbs, **kw)
        finally:
            if drain_eng is not None:
                drain_eng.close()
        return plan, r, eng.last_wave


def _pdbs_of_mix(c):
    """A maxUnavailable 1 PDB on the first label of each of the first four labelled workloads."""
    seen, out = set(), []
    for r in c.pod_recs:
        labels = r.tmpl.labels
        if not labels or r.tmpl.workload_kind == "Pod" or (r.tmpl.namespace, r.tmpl.workload_name) in seen or len(out) == 4:
            continue
        seen.add((r.tmpl.namespace, r.tmpl.workload_name))
        k, v = sorted(labels.items())[0]
        out.append({"apiVersion": "policy/v1beta1", "kind": "PodDisruptionBudget",
                    "metadata": {"name": f"pdb-{len(out)}", "namespace": r.tmpl.namespace},
                    "spec": {"maxUnavailable": 1, "selector": {"matchLabels": {k: v}}}})
    assert out
    return out


@pytest.mark.parametrize("kernel", sorted(GEOMETRIES))
def test_plans_match_checker_at_forced_geometries(kernel):
    cs, t, big = GEOMETRIES[kernel]
    for seed in (0, 3):
        p, c = _plan_compiled(*synth.make_mix(seed_no=seed, n_nodes=40))
        plan, r, info = _lockstep_plan(c, dict(cluster_ctas=cs, threads_per_cta=t, force_large=big), b=3, kernel=kernel)
        assert plan.TotalWaves > 0 and r.batches >= plan.TotalWaves
        assert info["commits"] == plan.TotalWaves


def test_plans_match_checker_without_static_cache_and_with_pdbs():
    for seed in (1, 4):
        p, c = _plan_compiled(*synth.make_mix(seed_no=seed, n_nodes=40))
        _lockstep_plan(c, dict(static_cache=False), b=4)
        _lockstep_plan(c, b=2, pdb_objs=_pdbs_of_mix(c), order="given", candidates=list(range(c.n_nodes))[::-1])


def test_plans_match_checker_past_the_shared_memory_budget():
    """The large-cluster variant (per-node arrays in global memory, as past the shared-memory budget) on a 2,500-node C3."""
    p, c = _plan_compiled(*synth.make_c3(n_nodes=2500, n_workloads=120, replicas=10, n_apps=2, seed_no=11))
    plan, r, info = _lockstep_plan(c, dict(force_large=True), b=4, candidates=list(range(0, c.n_nodes, 97)))
    assert plan.TotalWaves > 0 and all(l["large"] for l in info["launches"])


def test_wave_batches_equal_drains_from_the_same_placement():
    """Without GPU share a wave batch equals simon_drain_run from the placement the earlier waves leave."""
    for seed in (2, 6):
        p, c = _plan_compiled(*synth.make_mix(seed_no=seed, n_nodes=40))
        if np.asarray(c.snap["gpu_count"]).any():
            cl, apps = synth.make_mix(seed_no=seed, n_nodes=40)
            for n in cl.Nodes:
                for sect in ("allocatable", "capacity"):
                    n["status"][sect].pop("alibabacloud.com/gpu-count", None)
                    n["status"][sect].pop("alibabacloud.com/gpu-mem", None)
            p, c = _plan_compiled(cl, apps)
        _lockstep_plan(c, b=3, drain_check=True)


def _gpu_node(name, mem_gi, count, cpu="16000m"):
    n = {"apiVersion": "v1", "kind": "Node", "metadata": {"name": name, "labels": {"kubernetes.io/hostname": name}},
         "status": {"allocatable": {"cpu": cpu, "memory": "64Gi", "pods": "110"},
                    "capacity": {"cpu": cpu, "memory": "64Gi", "pods": "110"}}}
    if count:
        for sect in ("allocatable", "capacity"):
            n["status"][sect]["alibabacloud.com/gpu-count"] = str(count)
            n["status"][sect]["alibabacloud.com/gpu-mem"] = f"{mem_gi}Gi"
    return n


def _gpu_pod(name, node, mem_gi):
    return {"apiVersion": "v1", "kind": "Pod", "metadata": {"name": name, "namespace": "default",
                                                            "annotations": {"alibabacloud.com/gpu-mem": f"{mem_gi}Gi", "alibabacloud.com/gpu-count": "1"}},
            "spec": {"affinity": {"nodeAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": {"nodeSelectorTerms": [
                {"matchExpressions": [{"key": "kubernetes.io/hostname", "operator": "In", "values": [node]}]}]}}},
                "containers": [{"name": "c", "image": "x", "resources": {"requests": {"cpu": "100m", "memory": "128Mi"}}}]}}


def test_gpu_share_wave_follows_the_carried_devices():
    """node-x has two 12 GiB devices, pods p1 and p2 (6 GiB each) sit on its device 0; p0 (5 GiB, first in pod order) sits on node-y,
    which it prefers.
    Draining node-y moves p0 to node-x, where only device 1 has room: its slot word is device 1.  A rebuild of that placement replays
    Reserve in pod order (p0, p1, p2) and gives p0 device 0.  The plan follows the carried state, and the checker agrees."""
    from simon_b200.engine import Engine
    nodes = [_gpu_node("node-x", 24, 2), _gpu_node("node-y", 24, 2)]
    pods = [_gpu_pod("p0", "node-y", 5), _gpu_pod("p1", "node-x", 6), _gpu_pod("p2", "node-x", 6)]
    na = pods[0]["spec"]["affinity"]["nodeAffinity"]         # p0 prefers node-y but may move
    na["preferredDuringSchedulingIgnoredDuringExecution"] = [
        {"weight": 100, "preference": na.pop("requiredDuringSchedulingIgnoredDuringExecution")["nodeSelectorTerms"][0]}]
    cluster = O.ResourceTypes(Nodes=nodes, Pods=pods)
    p, c = _plan_compiled(cluster, [])
    x, y = c.node_index("node-x"), c.node_index("node-y")
    from oracle.binding import Oracle
    o = Oracle(c)
    placed = o.schedule()[0]
    assert placed.tolist() == [y, x, x] and o.gpu_slot_words().tolist() == [1, 1, 1]
    plan, r, _ = _lockstep_plan(c, b=1, order="given", candidates=[y])
    assert [w.Nodes for w in plan.Waves] == [["node-y"]]
    assert [(e.To, e.GpuIndex) for e in plan.Waves[0].Evicted] == [("node-x", "1")]
    final, slots = r.chk.placement()          # equal to the engine's base at every commit (LockstepRunner)
    assert int(slots[0]) == 1 << 4
    with Engine(c) as e2:
        e2.schedule_resume(final)
        assert int(e2.gpu_slot_words()[0]) == 1           # the pod-order replay: device 0


def test_wave_refusals_and_session_safety():
    from simon_b200.engine import Engine
    p, c = _plan_compiled(*synth.make_mix(seed_no=3, n_nodes=40))
    with Engine(c) as eng:
        placed = eng.schedule()[0]
        L = eng
        with pytest.raises(RuntimeError, match="wave base"):
            L.wave_run([np.arange(1, c.n_nodes)])
        L.wave_begin(placed)
        with pytest.raises(RuntimeError, match="no simon_wave_run batch"):
            L.wave_commit(0)
        with pytest.raises(RuntimeError, match="leaves no node"):
            L.wave_run([np.zeros(0, np.uint32)])
        eng.moves_upload(np.array([[0, 0]], np.uint32))
        for call in (lambda: eng.moves_plan(4), eng.pdbs_allowed):         # the pool holds the base, not the live state
            with pytest.raises(RuntimeError, match="no placement"):
                call()
        res = L.wave_run([np.arange(1, c.n_nodes)])
        with pytest.raises(RuntimeError, match="of a batch of 1"):
            from simon_b200.engine import lib
            L._check(lib().simon_wave_commit(L.h, 5))
        eng.drain_run(placed, [np.arange(1, c.n_nodes)])          # rebuilds: drops the base
        with pytest.raises(RuntimeError, match="wave base"):
            L.wave_commit(0)
        assert res[0]["n_evicted"] >= 0


def test_session_answers_unchanged_by_a_rolling_plan():
    cluster, apps = synth.make_mix(seed_no=5, n_nodes=40)
    with simulator.NewSimulator() as sim:
        sim.RunCluster(simulator.PrepareCluster(cluster))
        for a in apps:
            sim.ScheduleApp(a)
        names = sim.compiled.node_names
        pod = next(f"{r.tmpl.namespace}/{r.name}" for q, r in enumerate(sim.compiled.pod_recs) if sim.placements[q] >= 0)
        wl = next(f"{r.tmpl.workload_kind}/{r.tmpl.workload_namespace}/{r.workload_name}" for r in sim.compiled.pod_recs
                  if r.tmpl.workload_kind in ("ReplicaSet", "StatefulSet"))

        def answers():
            d = sim.DrainNodes([[names[0]], [names[1], names[2]]])
            m = sim.PlanMigrations(max_moves=5)
            m.KernelMs = 0.0                                               # a device time, not an answer
            x = sim.Explain([pod])[0]
            h = sim.Headroom([wl], max_replicas=50)
            return repr(d), repr(m), repr(x), repr(h)
        placements = sim.placements.copy()
        before = answers()
        plan = sim.PlanRollingMaintenance(max_unavailable=3)
        assert plan.TotalWaves > 0
        assert np.array_equal(sim.placements, placements)
        assert answers() == before
        plan2 = sim.PlanRollingMaintenance(names[:5], max_unavailable=2, order="given")
        assert sorted([n for w in plan2.Waves for n in w.Nodes] + [s.Node for s in plan2.Skipped]) == sorted(names[:5])
        assert plan2.Order == names[:5] and all(len(w.Nodes) <= 2 for w in plan2.Waves)
        for kw, msg in ((dict(nodes=["nope"]), "no node named"), (dict(max_unavailable=0), "max_unavailable"),
                        (dict(order="random"), "unknown order")):
            with pytest.raises(ValueError, match=msg):
                sim.PlanRollingMaintenance(**kw)
        with pytest.raises(TypeError):
            sim.PlanRollingMaintenance(local_volumes=True)
