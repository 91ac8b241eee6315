"""Node-pool replacement (simon_b200.replace, Simulator.PlanNodeReplacement, simon_wave_run_join / simon_wave_commit_retire) on the
CPU: the planner on the wave checker (tests/checkers.c) against hand-derived answers, and the host refusals."""
import numpy as np
import pytest

import checkers
from checkers import OracleRunner
from simon_b200 import grow, objects as O, replace, simulator
from test_grow import _dep, _ds, _node, session


def _spec(name, mcpu="8000m", mem="32Gi"):
    al = {"cpu": mcpu, "memory": mem, "pods": "110"}
    return {"apiVersion": "v1", "kind": "Node", "metadata": {"name": name, "labels": {"pool": "new"}},
            "status": {"allocatable": dict(al), "capacity": dict(al)}}


def _anti(name, n):
    d = _dep(name, n, cpu="500m")
    d["spec"]["template"]["spec"]["affinity"] = {"podAntiAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": [
        {"labelSelector": {"matchLabels": {"app": name}}, "topologyKey": "kubernetes.io/hostname"}]}}
    return d


def plan_cpu(sim, nodes, spec, kmax=None, caps=(100, 100), **kw):
    """PlanNodeReplacement's plan on the checker: the same superset, its first base built by the grow checker."""
    from oracle.binding import Oracle
    kmax = len(nodes) if kmax is None else kmax
    c, placed, present, pool, copies, pdbs = replace.superset(sim, nodes, spec, kmax)
    o = Oracle(c)
    n_prefix = len(sim.placements)
    checkers.grow(o, placed, n_prefix, np.nonzero(present)[0].astype(np.uint32))
    runner = OracleRunner(o, pdbs)
    plan = replace.plan_replacement(c, placed, runner, present, pool, copies, caps=caps, pdbs=pdbs, **kw)
    o.close()
    return plan, c


def _cluster(extra=(), n_nodes=2, mcpu="4000m", ds=True):
    return O.ResourceTypes(Nodes=[_node(f"old-{i}", mcpu) for i in range(n_nodes)], Deployments=list(extra),
                           DaemonSets=[_ds("agent")] if ds else [])


def test_one_to_one_by_a_larger_spec():
    # each old node: the agent (200m) and 3 x 1000m; a 5000m copy takes 3.2 cores, so two copies are needed, one per wave
    sim = session(_cluster([_dep("web", 6)]))
    plan, c = plan_cpu(sim, ["old-0", "old-1"], _spec("big", "5000m"))
    assert plan.Sizing.MinNodes == 2 and plan.Count == 2
    assert plan.Sizing.PerK[1]["n_unscheduled"] > 0 and 0 not in plan.Sizing.PerK     # k = 0 leaves no node
    assert plan.TotalWaves == 2 and not plan.Skipped and not plan.NeverJoined
    assert [len(w.Joined) for w in plan.Waves] == [1, 1] and [len(w.Nodes) for w in plan.Waves] == [1, 1]
    for w in plan.Waves:
        assert [p.Pod.name.split("-")[0] for p in w.JoinPods] == ["agent"] and w.JoinPods[0].Node == w.Joined[0]
    assert plan.MovedPods == 6 and plan.JoinedNodes == 2 and plan.RetiredNodes == 2
    # every web pod ends on a copy; the old nodes' agents do not exist any more, the copies' agents run on them
    for name, (node, _g) in plan.FinalPlacement.items():
        if "web" in name:
            assert node.startswith(O.NEW_NODE_NAME_PREFIX)
    assert sorted(v[0] for k, v in plan.FinalPlacement.items() if "agent" in k and v[0]) == sorted(w.Joined[0] for w in plan.Waves)


def test_consolidation_onto_fewer_larger_nodes():
    # four old nodes of 3.2 cores each onto 16-core copies: 12 web cores + 0.2 per copy fit on one
    sim = session(_cluster([_dep("web", 12)], n_nodes=4))
    plan, c = plan_cpu(sim, [f"old-{i}" for i in range(4)], _spec("huge", "16000m", "64Gi"), max_surge=1, max_unavailable=3)
    assert plan.Sizing.MinNodes == 1 < 4 and plan.Count == 1
    assert plan.TotalWaves == 1 and plan.Waves[0].Joined and len(plan.Waves[0].Nodes) == 4 and plan.MovedPods == 12


def test_anti_affinity_needs_surge():
    # one replica per old node with required hostname anti-affinity: without surge a drained replica has nowhere to go
    sim = session(_cluster([_anti("db", 2)]))
    plan, _ = plan_cpu(sim, ["old-0", "old-1"], _spec("big"), max_surge=0, max_unavailable=1)
    assert plan.Sizing.MinNodes == 2
    assert plan.TotalWaves == 0 and [s.Node for s in plan.Skipped] == plan.Pool and len(plan.NeverJoined) == 2
    assert all(any("anti-affinity" in r or "didn't match" in r for r in s.Reasons) for s in plan.Skipped)
    plan, _ = plan_cpu(sim, ["old-0", "old-1"], _spec("big"), max_surge=1, max_unavailable=0)
    assert plan.TotalWaves == 2 and not plan.Skipped and plan.MovedPods == 2


def test_spec_too_small_for_the_daemonset():
    sim = session(_cluster([_dep("web", 2)]))
    plan, _ = plan_cpu(sim, ["old-0", "old-1"], _spec("tiny", "100m"), kmax=2)
    assert plan.Sizing.MinNodes == -1 and plan.Count == 2
    assert plan.TotalWaves == 0 and sorted(s.Node for s in plan.Skipped) == ["old-0", "old-1"]
    for s in plan.Skipped:
        assert any(r.startswith("new-node pod kube-system/agent") and "Insufficient cpu" in r for r in s.Reasons), s.Reasons
    assert len(plan.NeverJoined) == 2


def test_node_name_pod_is_skipped_without_a_run():
    bound = {"apiVersion": "v1", "kind": "Pod", "metadata": {"name": "pinned", "namespace": "default"},
             "spec": {"nodeName": "old-0", "containers": [{"name": "c", "image": "x", "resources": {"requests": {"cpu": "100m"}}}]}}
    cl = _cluster([_dep("web", 2)])
    cl.Pods.append(bound)
    sim = session(cl)
    plan, _ = plan_cpu(sim, ["old-0", "old-1"], _spec("big"), order="given")
    assert [s.Node for s in plan.Skipped] == ["old-0"] and plan.Skipped[0].Drain is None
    assert plan.TotalWaves == 1 and plan.Waves[0].Nodes == ["old-1"]


def test_caps_split_the_waves():
    # 4 old nodes (3.2 cores each: 12 web cores and 4 agents of 0.2) onto 8-core copies.  Two copies hold 12.4 of 16 cores (77 %), three
    # hold 12.6 of 24 (52 %): MinNodes is 2 at MaxCPU 100 and 3 at MaxCPU 60
    sim = session(_cluster([_dep("web", 12)], n_nodes=4))
    loose, _ = plan_cpu(sim, [f"old-{i}" for i in range(4)], _spec("big"), max_surge=2, max_unavailable=0, caps=(100, 100))
    tight, _ = plan_cpu(sim, [f"old-{i}" for i in range(4)], _spec("big"), max_surge=2, max_unavailable=0, caps=(60, 100))
    assert loose.Sizing.MinNodes == 2 and tight.Sizing.MinNodes == 3
    assert [len(w.Nodes) for w in loose.Waves] == [2, 2] and loose.JoinedNodes == 2
    assert tight.JoinedNodes == 3 and tight.RetiredNodes == 4 and not tight.Skipped


def _db_pdb():
    return {"apiVersion": "policy/v1", "kind": "PodDisruptionBudget", "metadata": {"name": "db", "namespace": "default"},
            "spec": {"minAvailable": 2, "selector": {"matchLabels": {"app": "db"}}}}


def test_pdb_splits_a_wave():
    # one db replica per old node (required hostname anti-affinity), a PDB that allows one disruption: with max_surge 3 every wave
    # may take three old nodes, but only the prefix of one keeps the PDB, so each wave retires one node
    cl = _cluster([_anti("db", 3)], n_nodes=3)
    cl.PodDisruptionBudgets.append(_db_pdb())
    sim = session(cl, (), simulator.WithPodDisruptionBudgets())
    plan, _ = plan_cpu(sim, ["old-0", "old-1", "old-2"], _spec("big"), max_surge=3, max_unavailable=0, count=3)
    assert [len(w.Nodes) for w in plan.Waves] == [1, 1, 1] and not plan.Skipped
    assert [len(w.Joined) for w in plan.Waves] == [3, 0, 0]
    assert all(w.PdbEvicted == {"default/db": 1} for w in plan.Waves)


def test_pdb_blocks_every_node():
    pdb = {"apiVersion": "policy/v1", "kind": "PodDisruptionBudget", "metadata": {"name": "web", "namespace": "default"},
           "spec": {"minAvailable": 3, "selector": {"matchLabels": {"app": "web"}}}}
    cl = _cluster([_dep("web", 4, cpu="500m")])
    cl.PodDisruptionBudgets.append(pdb)
    sim = session(cl, (), simulator.WithPodDisruptionBudgets())
    plan, _ = plan_cpu(sim, ["old-0", "old-1"], _spec("big"), max_surge=2, max_unavailable=0)
    # 2 web pods per old node; the PDB allows one disruption, so no wave may drain an old node (2 evictions): every node is skipped
    assert plan.TotalWaves == 0 and all(any("PodDisruptionBudget default/web" in r for r in s.Reasons) for s in plan.Skipped)


def test_pinned_nodes_stay_out_of_the_sizing():
    bound = {"apiVersion": "v1", "kind": "Pod", "metadata": {"name": "pinned", "namespace": "default"},
             "spec": {"nodeName": "old-0", "containers": [{"name": "c", "image": "x", "resources": {"requests": {"cpu": "100m"}}}]}}
    cl = _cluster([_dep("web", 6)])
    cl.Pods.append(bound)
    sim = session(cl)
    plan, _ = plan_cpu(sim, ["old-0", "old-1"], _spec("big", "5000m"))
    # old-0 can never retire; retiring old-1 alone needs one copy
    assert plan.Sizing.MinNodes == 1 and plan.Sizing.PerK[1]["n_blocked"] == 0 and plan.Count == 1


def test_refusals():
    with pytest.raises(RuntimeError, match="RunCluster"):
        simulator.NewSimulator().PlanNodeReplacement(["old-0"], _spec("big"))
    sim = session(_cluster([_dep("web", 2)]))
    with pytest.raises(ValueError, match="no node named 'nope'"):
        sim.PlanNodeReplacement(["old-0", "nope"], _spec("big"))
    with pytest.raises(ValueError, match="'old-0' is listed twice"):
        sim.PlanNodeReplacement(["old-0", "old-1", "old-0"], _spec("big"))
    with pytest.raises(ValueError, match="not a Node"):
        sim.PlanNodeReplacement(["old-0"], _dep("x", 1))
    with pytest.raises(ValueError, match="max_surge"):
        sim.PlanNodeReplacement(["old-0"], _spec("big"), max_surge=0, max_unavailable=0)
    with pytest.raises(ValueError, match="unknown order"):
        sim.PlanNodeReplacement(["old-0"], _spec("big"), order="random")
    with pytest.raises(ValueError, match="count"):
        sim.PlanNodeReplacement(["old-0"], _spec("big"), count=3, kmax=2)
    with pytest.raises(ValueError, match="exceed the engine"):
        sim.PlanNodeReplacement(["old-0"], _spec("big"), kmax=grow.ENGINE_MAX_NODES)
    sim.Close()
    with pytest.raises(RuntimeError, match="closed"):
        sim.PlanNodeReplacement(["old-0"], _spec("big"))
