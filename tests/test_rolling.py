"""Rolling node maintenance (simon_b200.rolling, simon_wave_*) on the CPU: the planner on the wave checker (tests/checkers.c)
against hand-derived answers, the planner's rules and refusals on fake runners, the ABI and the session's refusals without a
device."""
import numpy as np
import pytest

from simon_b200 import abi, objects as O, rolling, scaledown, simulator, synth
from simon_b200.compiler import compile_cluster


def _compiled(cluster, apps):
    p = simulator.plan(cluster, apps)
    return compile_cluster(p.nodes, p.pods, p.ctx)


def _node(name, mcpu="4000m", mem="16Gi"):
    return {"apiVersion": "v1", "kind": "Node", "metadata": {"name": name, "labels": {"kubernetes.io/hostname": name}},
            "status": {"allocatable": {"cpu": mcpu, "memory": mem, "pods": "110"}, "capacity": {"cpu": mcpu, "memory": mem, "pods": "110"}}}


def _deployment(name, replicas, cpu="1000m"):
    return {"apiVersion": "apps/v1", "kind": "Deployment", "metadata": {"name": name, "namespace": "default"},
            "spec": {"replicas": replicas, "selector": {"matchLabels": {"app": name}},
                     "template": {"metadata": {"labels": {"app": name}},
                                  "spec": {"containers": [{"name": "c", "image": "nginx",
                                                           "resources": {"requests": {"cpu": cpu, "memory": "1Gi"}}}]}}}}


def _bound_pod(name, node):
    return {"apiVersion": "v1", "kind": "Pod", "metadata": {"name": name, "namespace": "default"},
            "spec": {"nodeName": node, "containers": [{"name": "c", "image": "nginx",
                                                       "resources": {"requests": {"cpu": "100m", "memory": "128Mi"}}}]}}


def _pdb(name, app, **spec):
    return {"apiVersion": "policy/v1beta1", "kind": "PodDisruptionBudget", "metadata": {"name": name, "namespace": "default"},
            "spec": dict(spec, selector={"matchLabels": {"app": app}})}


def four_nodes(replicas=8, pods=()):
    """4 nodes of 4000m; a Deployment `web` of `replicas` pods of 1000m (8: two per node in the live state)."""
    cluster = O.ResourceTypes(Nodes=[_node(f"node-{i}") for i in range(4)], Pods=list(pods))
    return cluster, [O.AppResource("web", O.ResourceTypes(Deployments=[_deployment("web", replicas)]))]


def _checker_plan(c, pdb_objs=None, **kw):
    import checkers
    from oracle.binding import Oracle
    from simon_b200.disruption import compile_pdbs
    o = Oracle(c)
    placed = o.schedule()[0]
    pdbs = compile_pdbs(pdb_objs, c) if pdb_objs else None
    runner = checkers.OracleRunner(o, pdbs)
    kw.setdefault("caps", (100, 100))
    return rolling.plan_rolling(c, placed, runner, pdbs=pdbs, **kw), placed, runner


def _per_node(plan, c):
    cnt = {nm: 0 for nm in c.node_names}
    for node, _gpu in plan.FinalPlacement.values():
        if node is not None:
            cnt[node] += 1
    return [cnt[nm] for nm in c.node_names]


# ---- the planner on the checker, against hand-derived answers ---------------------------------------------------------------------

def test_one_node_at_a_time_rolls_every_node():
    c = _compiled(*four_nodes())
    plan, placed, _ = _checker_plan(c)
    assert np.bincount(placed, minlength=4).tolist() == [2, 2, 2, 2]
    assert [w.Nodes for w in plan.Waves] == [["node-0"], ["node-1"], ["node-2"], ["node-3"]]
    assert plan.Skipped == [] and plan.TotalWaves == 4 and plan.MovedPods == sum(len(w.Evicted) for w in plan.Waves)
    assert [len(w.Evicted) for w in plan.Waves][0] == 2
    assert all(e.To is not None and e.To not in w.Nodes for w in plan.Waves for e in w.Evicted)
    assert sum(_per_node(plan, c)) == 8


def test_two_at_a_time_fits_only_because_the_first_wave_came_back():
    """b = 2: wave 1 takes node-0 and node-1 out, their 4 pods fill node-2 and node-3 (4 x 1000m each).  Wave 2 takes node-2 and node-3
    out: their 8 pods fit only on node-0 and node-1, which came back empty.  Three nodes at once never fit (6 pods onto one node)."""
    c = _compiled(*four_nodes())
    for b in (2, 3):
        plan, _placed, runner = _checker_plan(c, max_unavailable=b)
        assert [w.Nodes for w in plan.Waves] == [["node-0", "node-1"], ["node-2", "node-3"]], b
        assert [len(w.Evicted) for w in plan.Waves] == [4, 8] and plan.MovedPods == 12
        assert _per_node(plan, c) == [4, 4, 0, 0]
        assert {e.To for e in plan.Waves[1].Evicted} == {"node-0", "node-1"}
        assert plan.Waves[0].Occupancy["req_mcpu"] == 8000 and plan.Waves[0].Occupancy["alloc_mcpu"] == 8000
        assert runner.runs == ([2, 2] if b == 2 else [3, 2])


def test_a_node_with_a_bound_pod_is_skipped_with_its_reason():
    c = _compiled(*four_nodes(pods=[_bound_pod("pinned", "node-1")]))
    plan, _placed, runner = _checker_plan(c, order="given", candidates=[0, 1, 2, 3])
    assert [w.Nodes for w in plan.Waves] == [["node-0"], ["node-2"], ["node-3"]]
    assert [(s.Node, s.BeforeWave) for s in plan.Skipped] == [("node-1", 1)]
    assert plan.Skipped[0].Reasons == [f"pod default/pinned {scaledown.BLOCK_NODE_NAME}"]
    assert plan.Skipped[0].Drain is None and runner.runs == [1, 1, 1]     # skipped without a device run
    assert plan.FinalPlacement["default/pinned"] == ("node-1", None)
    # b = 3: the first batch stops before node-1 (the prefixes past it are not run), then node-1 is skipped; node-2 and node-3
    # together do not fit on node-0 and node-1, so they go one at a time
    plan, _placed, runner = _checker_plan(c, order="given", candidates=[0, 1, 2, 3], max_unavailable=3)
    assert [w.Nodes for w in plan.Waves] == [["node-0"], ["node-2"], ["node-3"]] and runner.runs[0] == 1
    assert [(s.Node, s.BeforeWave) for s in plan.Skipped] == [("node-1", 1)]


def test_a_pdb_with_max_unavailable_one_splits_the_wave():
    """4 replicas, one per node: without a PDB b = 2 rolls two nodes per wave.  With maxUnavailable 1 a wave may evict one of them:
    wave 1 is node-0 alone, and its pod lands on node-1 (all three remaining nodes tie; the first wins).  node-1 then holds two
    replicas, so even alone it would evict 2 > 1: it is skipped before wave 1 and not retried.  node-2 and node-3 follow, one each."""
    c = _compiled(*four_nodes(replicas=4))
    plan, placed, _ = _checker_plan(c, max_unavailable=2)
    assert np.bincount(placed, minlength=4).tolist() == [1, 1, 1, 1]
    assert [len(w.Nodes) for w in plan.Waves] == [2, 2]
    plan, _placed, runner = _checker_plan(c, [_pdb("web-pdb", "web", maxUnavailable=1)], max_unavailable=2)
    assert [w.Nodes for w in plan.Waves] == [["node-0"], ["node-2"], ["node-3"]]
    assert [(e.From, e.To) for e in plan.Waves[0].Evicted] == [("node-0", "node-1")]
    assert [(s.Node, s.BeforeWave, s.Reasons) for s in plan.Skipped] == \
        [("node-1", 1, ["PodDisruptionBudget default/web-pdb: evicts 2, allows 1"])]
    assert all(w.PdbEvicted == {"default/web-pdb": 1} for w in plan.Waves)
    assert runner.runs == [2, 2, 2, 1]
    # maxUnavailable 0: no node can go
    plan, _placed, _ = _checker_plan(c, [_pdb("web-pdb", "web", maxUnavailable=0)], max_unavailable=2)
    assert plan.Waves == [] and [s.Node for s in plan.Skipped] == ["node-0", "node-1", "node-2", "node-3"]
    assert plan.Skipped[0].Reasons == ["PodDisruptionBudget default/web-pdb: evicts 1, allows 0"]


def test_caps_shorten_a_wave():
    """Two nodes out leave 8000m requested on 8000m: 100 % > MaxCPU 75; one node out leaves 8000m on 12000m."""
    c = _compiled(*four_nodes())
    plan, _placed, _ = _checker_plan(c, max_unavailable=2, caps=(75, 100))
    assert [len(w.Nodes) for w in plan.Waves] == [1, 1, 1, 1]
    plan, _placed, _ = _checker_plan(c, max_unavailable=2, caps=(60, 100))
    assert plan.Waves == [] and all(s.Reasons == [rolling.CAPS_REASON] for s in plan.Skipped)


def test_given_order_against_utilisation():
    c = _compiled(*four_nodes())
    plan, _placed, _ = _checker_plan(c, order="given", candidates=[3, 1, 3, 0])
    assert plan.Order == ["node-3", "node-1", "node-0"]
    assert [w.Nodes for w in plan.Waves] == [["node-3"], ["node-1"], ["node-0"]]
    plan, _placed, _ = _checker_plan(c, candidates=[3, 1, 0])              # equal utilisation: nodeTree order
    assert plan.Order == ["node-0", "node-1", "node-3"]
    placed = np.array([0, 0, 0, 1, 1, 2, 3, 3], np.int32)                  # node-2 least used, then node-1 / node-3, then node-0
    assert rolling.order_candidates(c, placed, None, "utilisation") == [2, 1, 3, 0]
    assert rolling.order_candidates(c, placed, [0, 2], "given") == [0, 2]


@pytest.mark.parametrize("seed", [0, 5])
def test_checker_waves_keep_the_state_consistent_on_mixed_clusters(seed):
    """On a mixed cluster each committed base equals the state its placement leaves when every pod sits where the base says, up to
    GPU devices: node sums and pod counts match a drain checker run with nothing removed from that placement."""
    import checkers
    from oracle.binding import Oracle
    c = _compiled(*synth.make_mix(seed_no=seed, n_nodes=30))
    plan, _placed, runner = _checker_plan(c, max_unavailable=3)
    assert plan.TotalWaves + len(plan.Skipped) <= c.n_nodes and plan.TotalWaves > 0
    final, _slots = runner.placement()
    o2 = Oracle(c)
    checkers.drain(o2, final, np.arange(c.n_nodes, dtype=np.uint32))
    want, got = o2.state(), runner.o.state()
    for k in ("req_mcpu", "req_mem", "req_eph", "nz_mcpu", "nz_mem", "num_pods"):
        assert np.array_equal(got[k], want[k]), k


# ---- the planner's rules and refusals on fake runners ---------------------------------------------------------------------------

class FakeRunner(rolling.WaveRunner):
    """Drains whose verdict is ok(removed node set); records the calls."""

    def __init__(self, c, ok):
        self.c, self.ok, self.calls, self.commits = c, ok, [], []

    def begin(self, placed):
        self.placed = np.array(placed, np.int32)

    def run(self, remain_lists):
        self.calls.append([sorted(set(range(self.c.n_nodes)) - set(np.asarray(r).tolist())) for r in remain_lists])
        self.last = self.calls[-1]
        out = []
        for rm in self.last:
            good = self.ok(frozenset(rm))
            out.append(dict(n_evicted=0, n_placed=0, n_unscheduled=0 if good else 1, n_blocked=0, n_vanished=0, n_pdb_violated=0,
                            req_mcpu=0, alloc_mcpu=1, req_mem=0, alloc_mem=1, evicted=np.zeros(0, np.uint32), node=np.zeros(0, np.int32),
                            gpu_slots=np.zeros(0, np.uint32), score=np.zeros(0, np.int64), blocked=np.zeros(0, np.uint32),
                            fail_counts=np.zeros((0 if good else 1, abi.N_FAIL_CODES), np.uint32),
                            fail_pod=np.zeros(0 if good else 1, np.uint32), pdb_violated=np.zeros(0, np.uint32),
                            pdb_evicted=np.zeros(0, np.uint32)))
        return out

    def commit(self, i):
        self.commits.append(self.last[i])

    def placement(self):
        return self.placed, np.zeros(len(self.placed), np.uint32)


def _fake(ok, **kw):
    c = _compiled(*four_nodes())
    r = FakeRunner(c, ok)
    plan = rolling.plan_rolling(c, np.repeat(np.arange(4), 2).astype(np.int32), r, caps=(100, 100), **kw)
    return plan, r


def test_planner_prefix_rule_and_skips():
    # {0, 1} fails while {0, 1, 2} would pass: the first failing prefix ends the wave (no monotonicity assumed)
    plan, r = _fake(lambda s: s != {0, 1}, max_unavailable=3)
    assert r.calls[0] == [[0], [0, 1], [0, 1, 2]] and r.commits[0] == [0]
    assert [w.Nodes for w in plan.Waves][0] == ["node-0"]
    # node 1 never drains: skipped once, before wave 1, and the plan goes on
    plan, r = _fake(lambda s: 1 not in s, max_unavailable=2)
    assert [(s.Node, s.BeforeWave) for s in plan.Skipped] == [("node-1", 1)]
    assert [w.Nodes for w in plan.Waves] == [["node-0"], ["node-2", "node-3"]]
    assert sum(1 for call in r.calls if call[0] == [1]) == 1                # tried in one run only
    # never more than N - 1 nodes at once
    plan, r = _fake(lambda s: True, max_unavailable=10)
    assert r.calls[0] == [[0], [0, 1], [0, 1, 2]] and [len(w.Nodes) for w in plan.Waves] == [3, 1]


def test_planner_one_node_cluster_skips_it():
    c = _compiled(O.ResourceTypes(Nodes=[_node("only")]), [])
    r = FakeRunner(c, lambda s: True)
    plan = rolling.plan_rolling(c, np.zeros(0, np.int32), r, caps=(100, 100))
    assert plan.Waves == [] and [(s.Node, s.Reasons) for s in plan.Skipped] == [("only", [rolling.LAST_NODE_REASON])]
    assert r.calls == []


def test_planner_refusals_before_any_run():
    for kw, msg in ((dict(max_unavailable=0), "max_unavailable"), (dict(order="random"), "unknown order")):
        with pytest.raises(ValueError, match=msg):
            _fake(lambda s: True, **kw)
    c = _compiled(*four_nodes())
    r = FakeRunner(c, lambda s: True)
    with pytest.raises(ValueError):
        rolling.plan_rolling(c, np.zeros(8, np.int32), r, max_unavailable=-1)
    assert not hasattr(r, "placed")                                      # nothing began


def test_pdb_allowed_on_a_placement():
    from simon_b200.disruption import compile_pdbs
    c = _compiled(*four_nodes(replicas=4))
    t = compile_pdbs([_pdb("a", "web", maxUnavailable=1), _pdb("b", "web", minAvailable=4)], c)
    assert rolling.pdb_allowed(t, np.array([0, 1, 2, 3], np.int32)).tolist() == [1, 0]
    assert rolling.pdb_allowed(t, np.array([0, -1, 2, 3], np.int32)).tolist() == [0, 0]


# ---- ABI and the session without a device -------------------------------------------------------------------------------------

def test_wave_entry_points_are_declared():
    for name in ("simon_wave_begin", "simon_wave_run", "simon_wave_commit", "simon_wave_download", "simon_wave_times"):
        assert name in abi.SIGNATURES


def test_session_refusals_without_a_device():
    sim = simulator.NewSimulator()
    with pytest.raises(RuntimeError, match="RunCluster"):
        sim.PlanRollingMaintenance()
    sim.Close()
    with pytest.raises(RuntimeError, match="closed"):
        sim.PlanRollingMaintenance(["node-0"], max_unavailable=2)
