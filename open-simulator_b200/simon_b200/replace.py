"""Node-pool replacement: move a set of the live cluster's nodes (the old pool) to a new node spec, as a surge upgrade does.  Each wave
first joins up to max_surge new nodes, then drains up to max_surge + max_unavailable old nodes, which leave for good.  The operator asks
how many new nodes replace the pool, whether every wave fits within the PDBs and the caps, how many waves it takes, which old nodes
cannot be replaced and why, and where each moved pod ends up.

The cluster is the superset of grow.build with no apps: the session's nodes plus kmax copies of the spec (capacity.pool_nodes), and
the session's pod list followed by the copies' DaemonSet pods, pending.  A wave starts from the state the waves before it leave (the
wave base, include/simon_gpu.h simon_wave_begin_pool / simon_wave_run_join / simon_wave_commit_retire): the joined copies hold their
DaemonSet pods, the moved pods stay where they went with the GPU-share devices Reserve gave them, and the retired nodes are gone.

Sizing is one wave batch from the first base: scenario k (k = 0 .. kmax) joins the first k copies and retires the pool, less the old
nodes holding pods that never move (rolling.pinned_pods: they can never retire, and would fail every scenario).  MinNodes
is the least k whose scenario is committable (every join and evicted pod placed, nothing blocked, no PDB violated, the MaxCPU / MaxMemory
caps over the remaining nodes), -1 when none is.  The plan joins `count` copies (MinNodes by default) through rolling.run_waves.

Left out: pods with Open-Local volumes moving in waves (they block; join pods with volumes are refused), several specs in one plan,
returning the old nodes, retrying skipped nodes and pending pods, sharding over several GPUs, the native host side and a command line.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence

import numpy as np

from . import rolling, scaledown
from .capacity import env_caps, occupancy_ok

OCC_KEYS = ("req_mcpu", "alloc_mcpu", "req_mem", "alloc_mem")


@dataclass
class Sizing:
    PerK: Dict[int, Dict[str, int]] = field(default_factory=dict)   # k -> counts and occupancy of joining k copies, retiring the pool
    MinNodes: int = -1                                              # the least committable k, -1: none up to kmax


@dataclass
class ReplacementPlan:
    Pool: List[str]                    # the old nodes, in plan order
    Spec: str                          # the new node's name
    Sizing: Sizing
    Count: int                         # copies the plan may join: `count`, or Sizing.MinNodes
    Waves: List[rolling.Wave] = field(default_factory=list)
    Skipped: List[rolling.SkippedNode] = field(default_factory=list)
    NeverJoined: List[str] = field(default_factory=list)            # copies of the first Count that no wave joined
    FinalPlacement: Dict[str, tuple] = field(default_factory=dict)   # pod "namespace/name" -> (node or None, gpu-index or None)
    TotalWaves: int = 0
    MovedPods: int = 0
    JoinedNodes: int = 0
    RetiredNodes: int = 0


def superset(sim, nodes: Sequence[str], new_node, kmax: int):
    """The superset of a session (simulator.Simulator after RunCluster) for replacing `nodes` by copies of new_node: (compiled,
    placement of its pod list with the copies' DaemonSet pods pending, present nodes, the pool and the copies as compiled indices, and
    the session's PodDisruptionBudgets compiled on it or None)."""
    from . import objects as O
    from .capacity import pool_nodes
    from .grow import build
    gs = build(sim, [], [new_node], kmax)
    c = gs.compiled
    pool = [c.node_index(nm) for nm in nodes]
    # compiled indices follow the nodeTree order, not the build order: the copies are found by name
    copies = [c.node_index(O.name_of(n)) for (_s, _i, n) in pool_nodes([new_node], kmax)]
    present = np.ones(c.n_nodes, bool)
    present[copies] = False
    placed = np.concatenate([gs.placed, np.full(c.pods_dims["n_pods"] - gs.n_prefix, -1, np.int32)])
    pdbs = None
    if sim.options.pdbs:
        from .disruption import compile_pdbs
        pdbs = compile_pdbs(list(sim.cluster.PodDisruptionBudgets) + [d for a in sim.apps for d in a.Resource.PodDisruptionBudgets] +
                            sim.options.extraPdbs, c)
    return c, placed, present, pool, copies, pdbs


def committable(r: dict, max_cpu: int, max_mem: int) -> bool:
    """A wave_run(joins=...) result that may be committed: every join and evicted pod placed, nothing blocked, no PDB violated, and
    the caps over the remaining nodes."""
    return scaledown.drainable(r) and r.get("n_join_unscheduled", 0) == 0 and occupancy_ok(r, max_cpu, max_mem)


def sizing(compiled, runner: rolling.WaveRunner, present: np.ndarray, pool: Sequence[int], copies: Sequence[int],
           caps: Optional[tuple] = None) -> Sizing:
    """One wave batch from the runner's first base: scenario k joins copies[:k] and retires `pool` (k = 0 .. len(copies)); an empty
    pool gives no scenario."""
    max_cpu, max_mem = caps if caps is not None else env_caps()
    nodes = scaledown.NodeOrder(compiled)
    absent = np.nonzero(np.asarray(present) == 0)[0].tolist()
    remain, joins = [], []
    for k in range(len(copies) + 1):
        j = set(copies[:k])
        remain.append(nodes.remaining([g for g in absent if g not in j] + list(pool)))
        joins.append(np.asarray(copies[:k], np.uint32))
    keep = [k for k in range(len(remain)) if len(remain[k])] if len(pool) else []   # a scenario that leaves no node is not run
    raw = runner.run([remain[k] for k in keep], [joins[k] for k in keep]) if keep else []
    out = Sizing()
    for k, r in zip(keep, raw):
        out.PerK[k] = {q: int(r[q]) for q in ("n_evicted", "n_unscheduled", "n_blocked", "n_pdb_violated", "n_join", "n_join_unscheduled")
                       + OCC_KEYS}
        if out.MinNodes < 0 and committable(r, max_cpu, max_mem):
            out.MinNodes = k
    return out


def plan_replacement(compiled, placed: np.ndarray, runner: rolling.WaveRunner, present: np.ndarray, pool: Sequence[int],
                     copies: Sequence[int], count: Optional[int] = None, max_surge: int = 1, max_unavailable: int = 0,
                     order: str = "utilisation", caps: Optional[tuple] = None, pdbs=None) -> ReplacementPlan:
    """The replacement plan of `pool` (compiled node indices of present nodes) by `copies` (compiled indices of absent nodes, in join
    order) on the placement `placed` of the superset, driven through `runner`."""
    if max_surge < 0 or max_unavailable < 0 or max_surge + max_unavailable < 1:
        raise ValueError(f"max_surge + max_unavailable must be at least 1, neither below 0 (got {max_surge} and {max_unavailable})")
    names = compiled.node_names
    cand = rolling.order_candidates(compiled, placed, pool, order)
    runner.begin(placed, present)
    pinned = rolling.pinned_pods(compiled, placed)
    size = sizing(compiled, runner, present, [g for g in cand if g not in pinned], copies, caps)
    use = size.MinNodes if count is None else int(count)
    if use < 0:
        use = len(copies)
    if use > len(copies):
        raise ValueError(f"count {use} exceeds the {len(copies)} copies of the spec (kmax)")
    plan = ReplacementPlan(Pool=[names[c] for c in cand], Spec="", Sizing=size, Count=use)
    waves, skipped, moved, left = rolling.run_waves(compiled, placed, runner, cand, max_surge + max_unavailable, caps, pdbs,
                                                    present=present, copies=list(copies[:use]), max_surge=max_surge)
    plan.Waves, plan.Skipped, plan.MovedPods = waves, skipped, moved
    plan.NeverJoined = [names[g] for g in left]
    plan.FinalPlacement = rolling.final_placement(compiled, runner)
    plan.TotalWaves = len(waves)
    plan.JoinedNodes = sum(len(w.Joined) for w in waves)
    plan.RetiredNodes = sum(len(w.Nodes) for w in waves)
    return plan
