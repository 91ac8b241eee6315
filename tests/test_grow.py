"""Nodes to add to the live cluster (simon_grow_run, Engine.grow_run, simon_b200.grow, Simulator.PlanAddNodes) on the CPU.

The superset a session grows into: its pod list first and unchanged, then the pool DaemonSet pods guarded by their copies, then the
apps' pods; the placements remapped by node name; scenario k = 0 in the session's node order.  The search (grow.plan) runs here on the
grow checker (tests/checkers.c) on hand-derived cases; the shared k search gives apply.auto_add_nodes what its own loop gave; and
the host refusals."""
import copy

import numpy as np
import pytest

from simon_b200 import apply as A, capacity, grow, objects as O, simulator, synth
from simon_b200.compiler import compile_cluster
from simon_b200.scaledown import pod_guard


def _node(name, mcpu="4000m", zone=None):
    labels = {"kubernetes.io/hostname": name}
    if zone:
        labels["topology.kubernetes.io/zone"] = zone
    al = {"cpu": mcpu, "memory": "16Gi", "pods": "110"}
    return {"apiVersion": "v1", "kind": "Node", "metadata": {"name": name, "labels": labels},
            "status": {"allocatable": dict(al), "capacity": dict(al)}}


def _dep(name, n, cpu="1000m"):
    spec = {"containers": [{"name": "c", "image": "nginx", "resources": {"requests": {"cpu": cpu, "memory": "1Gi"}}}]}
    return {"apiVersion": "apps/v1", "kind": "Deployment", "metadata": {"name": name, "namespace": "default"},
            "spec": {"replicas": n, "selector": {"matchLabels": {"app": name}}, "template": {"metadata": {"labels": {"app": name}},
                                                                                           "spec": spec}}}


def _ds(name, cpu="200m"):
    spec = {"containers": [{"name": "c", "image": "agent", "resources": {"requests": {"cpu": cpu, "memory": "100Mi"}}}]}
    return {"apiVersion": "apps/v1", "kind": "DaemonSet", "metadata": {"name": name, "namespace": "kube-system"},
            "spec": {"selector": {"matchLabels": {"app": name}}, "template": {"metadata": {"labels": {"app": name}}, "spec": spec}}}


class _Closed:
    def close(self):
        pass


def session(cluster, apps=(), *opts):
    """A Simulator after RunCluster(PrepareCluster(cluster)) and ScheduleApp per app, its placements from the CPU oracle (no device)."""
    from oracle.binding import Oracle
    sim = simulator.NewSimulator(*opts)
    sim.cluster = simulator.PrepareCluster(cluster)
    sim._cluster_pods = [copy.copy(r) for r in sim.cluster.Pods]
    sim.apps = list(apps)
    p = sim._plan()
    c = compile_cluster(p.nodes, p.pods, p.ctx, open_local=sim.options.openLocal,
                        storage_classes=list(cluster.StorageClasss) + [sc for a in apps for sc in a.Resource.StorageClasss]
                        if sim.options.openLocal else None, local_devices=sim.options.openLocalDevices)
    o = Oracle(c, open_local=sim.options.openLocal)
    sim.placements = o.schedule()[0]
    sim.gpu_slots = o.gpu_slot_words()
    o.close()
    sim.compiled, sim._segments, sim.engine = c, list(p.segments), _Closed()
    return sim


class CheckerEngine:
    """Engine.grow_run on the CPU: the grow checker per scenario, plus the occupancy sums of its end state."""

    def __init__(self, c):
        from oracle.binding import Oracle
        self.c = c
        self.o = Oracle(c, open_local=c.storage is not None)
        self.batches = []

    def grow_run(self, placed, n_prefix, scenarios, detail=True, chunk=None):
        import checkers
        out = []
        for nodes in scenarios:
            r = checkers.grow(self.o, placed, n_prefix, nodes)
            st = self.o.state()
            act = np.asarray(nodes, np.int64)
            r.update(req_mcpu=int(st["req_mcpu"][act].sum()), alloc_mcpu=int(self.c.snap["alloc_mcpu"][act].sum()),
                     req_mem=int(st["req_mem"][act].sum()), alloc_mem=int(self.c.snap["alloc_mem"][act].sum()))
            out.append(r)
        self.batches.append(len(scenarios))
        self.last_grow = dict(chunks=1)
        return out


# the hand-derived cluster: 2 nodes of 4000m, a DaemonSet of 200m per node and 6 web pods of 1000m (3 per node): 800m free on each,
# so no pod of 1000m fits the running cluster.  The new app: 4 pods of 1000m.  A copy of a spec runs the DaemonSet pod too.
def _hand():
    cluster = O.ResourceTypes(Nodes=[_node("node-0"), _node("node-1")], Deployments=[_dep("web", 6)], DaemonSets=[_ds("agent")])
    app = O.AppResource("new", O.ResourceTypes(Deployments=[_dep("new", 4)]))
    specs = [_node("spec-small", "1000m"), _node("spec-big", "2400m"), _node("spec-mid", "1200m")]
    return cluster, app, specs


def _plan(sim, app, specs, kmax, method="sweep", **caps):
    gs = grow.build(sim, [app], specs, kmax)
    return gs, grow.plan(CheckerEngine(gs.compiled), gs, [O.name_of(s) for s in specs], method, **caps)


def test_superset_pod_list_guards_and_remap():
    cluster, app, specs = _hand()
    earlier = O.AppResource("earlier", O.ResourceTypes(Deployments=[_dep("e", 2, "100m")], DaemonSets=[_ds("logger", "100m")]))
    sim = session(cluster, [earlier])
    p = sim._plan()
    gs = grow.build(sim, [app], specs[:2], 3)
    c = gs.compiled
    recs = c.pod_recs
    assert gs.n_prefix == len(p.pods) == len(sim.placements)
    assert [(r.name, r.tmpl.workload_kind) for r in recs[:gs.n_prefix]] == [(r.name, r.tmpl.workload_kind) for r in p.pods]
    # the tail: the cluster's DaemonSet on every copy, the earlier app's DaemonSet on every copy, then the new app
    assert [s[0] for s in gs.segments] == ["cluster-daemonsets", "earlier", "new"]
    pool = [f"simon-{s:02d}-{i:05d}" for s in range(2) for i in range(3)]
    guard = pod_guard(c)
    for what, first, count in gs.segments[:2]:
        assert count == len(pool)
        assert [c.node_names[guard[q]] for q in range(first, first + count)] == pool
        assert all(recs[q].tmpl.workload_kind == "DaemonSet" for q in range(first, first + count))
    assert [recs[q].tmpl.workload_name for q in range(*gs.segments[2][1:2], sum(gs.segments[2][1:]))] == ["new"] * 4
    assert all(recs[q].app_name == "earlier" for q in range(gs.segments[1][1], gs.segments[1][1] + gs.segments[1][2]))
    # the remap keeps every placed pod on the node of the same name
    for q, g in enumerate(sim.placements.tolist()):
        if g >= 0:
            assert c.node_names[gs.placed[q]] == sim.compiled.node_names[g]
        else:
            assert gs.placed[q] == g
    # scenario k = 0 of every spec is the session's node order; k copies add that spec's first k copies
    for s in range(2):
        assert [c.node_names[g] for g in gs.scenario(s, 0).nodes] == sim.compiled.node_names
        assert sorted(c.node_names[g] for g in gs.scenario(s, 2).nodes) == sorted(sim.compiled.node_names + pool[3 * s:3 * s + 2])


def test_k0_tail_order_is_schedule_app_order():
    """An app without DaemonSets: the tail at k = 0 is the pod list ScheduleApp would append."""
    cluster, apps = synth.make_c3(n_nodes=40, n_workloads=10, replicas=4, n_apps=2, seed_no=9)
    sim = session(cluster, apps[:1])
    gs = grow.build(sim, apps[1:], [cluster.Nodes[0]], 2)
    sim.apps.append(apps[1])
    p = sim._plan()
    sim.apps.pop()
    what, first, count = gs.segments[-1]
    tail = [(r.tmpl.workload_name, r.name) for r in gs.compiled.pod_recs[first:first + count]]
    assert what == apps[1].Name and tail == [(r.tmpl.workload_name, r.name) for r in p.pods[gs.n_prefix:]]
    # the pool DaemonSet pods before it do not exist at k = 0
    guard = pod_guard(gs.compiled)
    active = set(gs.scenario(0, 0).nodes.tolist())
    assert all(guard[q] >= 0 and guard[q] not in active for q in range(gs.n_prefix, first))


def test_hand_derived_answers():
    cluster, app, specs = _hand()
    sim = session(cluster)
    assert sorted(sim.placements[:6].tolist()) == [0, 0, 0, 1, 1, 1]
    gs, res = _plan(sim, app, specs, 5)
    small, big, mid = res.Specs
    # 1000m copies hold 800m next to their DaemonSet pod: never a 1000m pod
    assert small.NewNodeNum == -1 and small.K == 5 and len(small.UnscheduledPods) == 4
    assert small.UnscheduledPods[0].Reason.endswith("Unschedulable: 0/7 nodes are available: 7 Insufficient cpu.")
    assert all(small.PerK[k]["n_unscheduled"] == 4 for k in range(6))
    # 2400m copies hold two pods each: k = 2 fits, k = 1 leaves two
    assert big.NewNodeNum == 2 and big.PerK[1]["n_unscheduled"] == 2
    assert sorted(p.Node for p in big.Pods if p.Pod.tmpl.workload_name == "new") == ["simon-01-00000"] * 2 + ["simon-01-00001"] * 2
    assert [p.Node for p in big.Pods if p.Pod.tmpl.workload_kind == "DaemonSet"] == ["simon-01-00000", "simon-01-00001"]
    assert not big.UnscheduledPods
    # 1200m copies hold one pod each
    assert mid.NewNodeNum == 4 and mid.PerK[3]["n_unscheduled"] == 1
    assert res.Best == {"spec": 1, "Spec": "spec-big", "k": 2}
    # the DaemonSet pods on the copies take room: 2 x 200m + 6 x 1000m + 200m per copy + 4 x 1000m requested
    assert big.PerK[2]["req_mcpu"] == 400 + 6000 + 400 + 4000 and big.PerK[2]["alloc_mcpu"] == 8000 + 4800
    # MaxCPU decides k: 10,800 / 12,800 = 84 %, at k = 3 11,000 / 15,200 = 72 %, at k = 4 11,200 / 17,600 = 63 %, at k = 5
    # 11,400 / 20,000 = 57 %
    for cap, want in ((90, 2), (80, 3), (70, 4), (60, 5), (50, -1)):
        for method in ("sweep", "bisect"):
            _gs, r = _plan(sim, app, specs[1:2], 5, method, max_cpu=cap)
            assert r.Specs[0].NewNodeNum == want, (cap, method)


def test_apps_that_fit_need_no_node():
    cluster, app, specs = _hand()
    sim = session(cluster)
    light = O.AppResource("light", O.ResourceTypes(Deployments=[_dep("light", 2, "500m")]))
    _gs, res = _plan(sim, light, specs, 3, "bisect")
    assert [s.NewNodeNum for s in res.Specs] == [0, 0, 0] and res.Best == {"spec": 0, "Spec": "spec-small", "k": 0}
    assert res.ScenariosEvaluated == 6 and res.Rounds == 1     # (s, 0) and (s, kmax) of each spec
    assert {p.Node for p in res.Specs[0].Pods} <= {"node-0", "node-1"}


def test_search_min_k_bisect_finds_the_sweep():
    """A fake monotone runner: bisection finds the sweep's k for every threshold, in at most 1 + ceil(log2 kmax) rounds."""
    kmax = 37
    for thresholds in ([0, 5, 37, 99], [1, 2, 36, 17], [38, 0, 0, 13]):
        calls = []
        ok = lambda s, k: k >= thresholds[s]
        sweep, r1 = capacity.search_min_k(4, kmax, "sweep", calls.append, ok)
        bis, r2 = capacity.search_min_k(4, kmax, "bisect", calls.append, ok)
        assert sweep == bis == [t if t <= kmax else -1 for t in thresholds]
        assert r1 == 1 and r2 <= 1 + 6


def _old_auto_add_nodes(cluster, apps, new_node, runner_factory, kmax=64, method="sweep"):
    """apply.auto_add_nodes as its own loop ran it before the shared search (the CPU-only path, without Open-Local)."""
    max_cpu, max_mem = capacity.env_caps()
    ks = list(range(0, kmax + 1))
    ss = capacity.build_scenarios(cluster, apps, [new_node], ks)
    runner = runner_factory(ss)
    by_k = {sc.k: sc for sc in ss.scenarios}
    per_k = {}
    keys = ("n_unscheduled", "n_scheduled", "req_mcpu", "alloc_mcpu", "req_mem", "alloc_mem")

    def evaluate(klist):
        todo = [by_k[k] for k in klist if k not in per_k]
        for sc, res in zip(todo, runner(ss, todo)):
            per_k[sc.k] = {q: int(res[q]) for q in keys}

    def ok(k):
        r = per_k[k]
        return r["n_unscheduled"] == 0 and capacity.occupancy_ok(r, max_cpu, max_mem, 100)
    if method == "sweep":
        evaluate(ks)
        rounds = 1
        best = next((k for k in sorted(per_k) if ok(k)), -1)
    else:
        evaluate([0, kmax])
        rounds = 1
        if ok(0):
            best = 0
        elif not ok(kmax):
            best = -1
        else:
            lo, hi = 0, kmax
            while hi - lo > 1:
                mid = (lo + hi) // 2
                evaluate([mid])
                rounds += 1
                if ok(mid):
                    hi = mid
                else:
                    lo = mid
            best = hi
    return A.ApplyResult(best, per_k[0]["n_unscheduled"] if 0 in per_k else -1, len(per_k), rounds, per_k)


@pytest.mark.parametrize("method", ["sweep", "bisect"])
def test_auto_add_nodes_unchanged_by_the_shared_search(method):
    from test_capacity import _oracle_factory
    cluster, apps, specs = synth.make_c4(n_nodes=12, n_workloads=8, replicas=15, seed_no=4)
    for kmax in (0, 1, 24):
        got = A.auto_add_nodes(cluster, apps, specs[1], _oracle_factory, kmax=kmax, method=method)
        want = _old_auto_add_nodes(cluster, apps, specs[1], _oracle_factory, kmax=kmax, method=method)
        assert got == want, kmax


def test_refusals():
    cluster, app, specs = _hand()
    with pytest.raises(RuntimeError, match="RunCluster"):
        simulator.NewSimulator().PlanAddNodes([app], specs)
    sim = session(cluster)
    with pytest.raises(ValueError, match="kmax"):
        sim.PlanAddNodes([app], specs, kmax=-1)
    with pytest.raises(ValueError, match="not a Node"):
        sim.PlanAddNodes([app], [specs[0], _dep("x", 1)])
    with pytest.raises(ValueError, match="unknown method"):
        sim.PlanAddNodes([app], specs, method="binary")
    # a pool name that is a node of the session
    clash = session(O.ResourceTypes(Nodes=[_node("node-0"), _node("simon-00-00001")], Deployments=[_dep("web", 2)]))
    with pytest.raises(ValueError, match="simon-00-00001"):
        grow.build(clash, [app], specs[:1], 2)
    grow.build(clash, [app], specs[:1], 1)
    # past the engine's node limit
    with pytest.raises(ValueError, match="exceed the engine"):
        grow.build(sim, [app], specs, grow.ENGINE_MAX_NODES // 3 + 1)
    sim.Close()
    with pytest.raises(RuntimeError, match="closed"):
        sim.PlanAddNodes([app], specs)
