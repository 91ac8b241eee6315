"""Rolling node maintenance: take nodes out in waves of at most `max_unavailable`, bring each wave back empty apart from its DaemonSet
pods, and report whether every evicted pod finds a place each time, how many waves it takes and which nodes cannot be rolled.  This
is the operator's question before a kernel, OS or kubelet upgrade, built on the drain definition of scaledown.py.

A wave starts from the state the waves before it leave (the wave base, include/simon_gpu.h simon_wave_*): the pods the earlier waves
evicted stay where they went, with the GPU-share devices Reserve gave them there, and the earlier waves' nodes are back.  Rebuilding
each wave's state from its placement instead would replay GPU-share Reserve in pod order and could give a moved pod other devices.

plan_rolling orders the candidates once (by live utilisation ascending, ties in nodeTree order, as PlanScaleDown orders them; or as
given).  Each wave evaluates, in one batch from the current base, the prefixes of length 1 .. min(max_unavailable, remaining) of the
remaining candidates.  The wave is the longest prefix k such that every prefix up to k drains (scaledown.drainable) within the MaxCPU /
MaxMemory caps, the rule of PlanScaleDown; that scenario is committed and becomes the next base.  When k = 0 the first remaining
candidate is skipped with its drain result and not retried.  The plan ends when no candidate remains.  A node holding pods that never
move (pinned_pods: bound by spec.nodeName, or with Open-Local volumes) fails every drain: it is skipped without a device run, and the
prefixes past it are not evaluated, which changes no wave.

run_waves is that loop, shared with node-pool replacement (replace.py), whose waves also join new nodes and retire the drained ones.

Left out: pods with Open-Local volumes moving in waves (they block, and the base's VG and device state is never changed), surge
nodes (see replace.py), retrying skipped nodes, pending pods of the live state (they stay pending and are not retried), sharding over several GPUs,
the native host side and a command line.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence

import numpy as np

from . import scaledown
from .capacity import env_caps, occupancy_ok

ORDERS = ("utilisation", "given")
CAPS_REASON = "the remaining nodes would exceed the MaxCPU / MaxMemory caps"
LAST_NODE_REASON = "no other node would remain"


@dataclass
class Wave:
    Nodes: List[str]                                          # taken out together, back at the end of the wave (retired: gone for good)
    Evicted: List[scaledown.EvictedPod] = field(default_factory=list)
    PdbEvicted: Dict[str, int] = field(default_factory=dict)  # PDB "namespace/name" -> members the wave evicts
    Occupancy: Dict[str, int] = field(default_factory=dict)   # req_mcpu / alloc_mcpu / req_mem / alloc_mem over the remaining nodes
    Joined: List[str] = field(default_factory=list)           # node-pool replacement: the new nodes that join first
    JoinPods: list = field(default_factory=list)              # their DaemonSet pods (grow.NewPod), with their nodes and gpu-index


@dataclass
class SkippedNode:
    Node: str
    BeforeWave: int                 # the index of the wave before which it was tried (len(Waves) when tried after the last one)
    Reasons: List[str]
    Drain: Optional[scaledown.DrainResult] = None             # its drain alone from that wave's base (None: not run, see pinned_pods)


@dataclass
class RollingPlan:
    Order: List[str]
    Waves: List[Wave] = field(default_factory=list)
    Skipped: List[SkippedNode] = field(default_factory=list)
    FinalPlacement: Dict[str, tuple] = field(default_factory=dict)   # pod "namespace/name" -> (node or None, gpu-index or None)
    TotalWaves: int = 0
    MovedPods: int = 0


class WaveRunner:
    """What run_waves drives.  begin(placed, present) makes the first base (present: None, or the nodes in the cluster);
    run(remain_lists, joins) drains each entry from the base, joining the nodes joins[i] first (joins None: no join), and returns
    Engine.wave_run(detail=True) dicts; commit(i, retire) makes entry i of the last run the base; placement() -> (node per pod, GPU slot
    word per pod) of the base."""

    def begin(self, placed, present=None):
        raise NotImplementedError

    def run(self, remain_lists, joins=None):
        raise NotImplementedError

    def commit(self, i: int, retire: bool = False):
        raise NotImplementedError

    def placement(self):
        raise NotImplementedError


class EngineRunner(WaveRunner):
    """The device: Engine.wave_begin / wave_run / wave_commit / wave_placement."""

    def __init__(self, eng):
        self.eng = eng

    def begin(self, placed, present=None):
        self.eng.wave_begin(placed, present)

    def run(self, remain_lists, joins=None):
        return self.eng.wave_run(remain_lists, joins, detail=True)

    def commit(self, i: int, retire: bool = False):
        self.eng.wave_commit(i, retire)

    def placement(self):
        return self.eng.wave_placement()


def pdb_allowed(pdbs, placed: np.ndarray) -> np.ndarray:
    """Per PDB of disruption.PdbTables: max(0, placed members - desired) on `placed`."""
    off = np.asarray(pdbs.pod_off, dtype=np.int64)
    ids = np.asarray(pdbs.pod_pdb, dtype=np.int64)
    owner = np.repeat(np.arange(len(off) - 1), np.diff(off))
    healthy = np.bincount(ids[np.asarray(placed)[owner] >= 0], minlength=len(pdbs.desired))
    return np.maximum(0, healthy - np.asarray(pdbs.desired, dtype=np.int64))


def order_candidates(compiled, placed: np.ndarray, candidates: Optional[Sequence[int]], order: str) -> List[int]:
    """The candidates (all nodes by default; repeats dropped, first kept) in plan order."""
    if order not in ORDERS:
        raise ValueError(f"unknown order {order!r} (one of {', '.join(ORDERS)})")
    cand = list(range(compiled.n_nodes)) if candidates is None else list(dict.fromkeys(int(c) for c in candidates))
    if order == "utilisation":
        util = scaledown.node_utilisation(compiled, placed)
        cand.sort(key=lambda c: (util[c], c))              # compiled index order is nodeTree order
    return cand


def pinned_pods(compiled, placed: np.ndarray) -> Dict[int, List[tuple]]:
    """Per node, the placed pods that block every drain of it from any base: bound by spec.nodeName or with Open-Local volumes, and no
    DaemonSet pod of any node.  They never move (a wave that would evict them is never committed), so such a node is skipped without a
    device run, and a wave ends before it."""
    placed = np.asarray(placed)
    fixed = np.asarray(compiled.pods["pod_fixed_node"])
    guard = scaledown.pod_guard(compiled)
    local = compiled.storage.class_local if getattr(compiled, "storage", None) is not None else None
    cls = np.asarray(compiled.pods["pod_class"])
    out: Dict[int, List[tuple]] = {}
    for q in np.nonzero((placed >= 0) & (guard < 0))[0].tolist():
        if fixed[q] >= 0:
            out.setdefault(int(placed[q]), []).append((q, scaledown.BLOCK_NODE_NAME))
        elif local is not None and local[int(cls[q])]:
            out.setdefault(int(placed[q]), []).append((q, scaledown.BLOCK_LOCAL_STORAGE))
    return out


def _reasons(d: scaledown.DrainResult) -> List[str]:
    out = [f"pod {b.Pod.tmpl.namespace}/{b.Pod.name} {b.Reason}" for b in d.BlockedPods]
    out += [f"pod {u.Pod.tmpl.namespace}/{u.Pod.name}: {u.Reason}" for u in d.UnscheduledPods]
    out += [f"PodDisruptionBudget {v.Name}: evicts {v.Evicted}, allows {v.Allowed}" for v in d.PdbViolations]
    if not out and not d.CapsOk:
        out.append(CAPS_REASON)
    return out


def plan_rolling(compiled, placed: np.ndarray, runner: WaveRunner, candidates: Optional[Sequence[int]] = None, order: str = "utilisation",
                 max_unavailable: int = 1, caps: Optional[tuple] = None, pdbs=None) -> RollingPlan:
    """The rolling plan of `candidates` (compiled node indices; all nodes by default) on the live placement `placed`, driven through
    `runner`.  caps: (MaxCPU, MaxMemory) percentages (default: the environment's, env_caps()); pdbs: disruption.PdbTables the runner
    honours, used to name PDBs in the results."""
    if max_unavailable < 1:
        raise ValueError(f"max_unavailable must be at least 1 (got {max_unavailable})")
    cand = order_candidates(compiled, placed, candidates, order)
    plan = RollingPlan(Order=[compiled.node_names[c] for c in cand])
    runner.begin(placed)
    plan.Waves, plan.Skipped, plan.MovedPods, _ = run_waves(compiled, placed, runner, cand, max_unavailable, caps, pdbs)
    plan.FinalPlacement = final_placement(compiled, runner)
    plan.TotalWaves = len(plan.Waves)
    return plan


def final_placement(compiled, runner: WaveRunner) -> Dict[str, tuple]:
    """Pod "namespace/name" -> (node or None, gpu-index or None) of the runner's base."""
    names = compiled.node_names
    final, slots = runner.placement()
    out = {}
    for q, rec in enumerate(compiled.pod_recs):
        g = int(final[q])
        out[f"{rec.tmpl.namespace}/{rec.name}"] = (names[g] if g >= 0 else None, scaledown.gpu_index(int(slots[q])) if g >= 0 else None)
    return out


def join_pods(compiled, r: dict) -> list:
    """The join pods of one wave_run(joins=..., detail=True) dict as grow.NewPod: their nodes (None: unschedulable) and gpu-index."""
    from .grow import NewPod
    names, recs = compiled.node_names, compiled.pod_recs
    return [NewPod(recs[q], names[g] if g >= 0 else None, scaledown.gpu_index(int(w)) if g >= 0 else None)
            for q, g, w in zip(r["join_pods"].tolist(), r["join_node"].tolist(), r["join_gpu_slots"].tolist())]


def join_reasons(compiled, r: dict, remain: np.ndarray) -> List[str]:
    """The FitError text of each unscheduled join pod of one wave_run(joins=..., detail=True) dict."""
    from .simulator import format_fit_error
    recs = compiled.pod_recs
    active = np.asarray(remain).tolist()
    memo: dict = {}
    return [f"new-node pod {recs[q].tmpl.namespace}/{recs[q].name}: "
            + format_fit_error(compiled, recs[q], r["join_fail_counts"][j], active=active, static_memo=memo)
            for j, q in enumerate(r["join_fail_pod"].tolist())]


def run_waves(compiled, placed: np.ndarray, runner: WaveRunner, cand: List[int], per_wave: int, caps: Optional[tuple], pdbs,
              present: Optional[np.ndarray] = None, copies: Sequence[int] = (), max_surge: int = 0):
    """The wave loop on a runner that holds the first base (begin done): each wave evaluates, in one batch, the prefixes of length
    1 .. min(per_wave, remaining) of the remaining candidates and commits the longest one whose every prefix is committable.  Without
    `present` (rolling maintenance) the drained nodes return.  With it (node-pool replacement; present: the nodes in the cluster)
    each wave first joins the next min(max_surge, left) nodes of `copies`, every prefix is evaluated with those joins, a committable
    prefix also places every join pod, and the drained nodes retire; when no prefix is committable the first candidate is skipped and
    the wave is tried again with the same joins.  -> (waves, skipped, moved pods, copies never joined)."""
    max_cpu, max_mem = caps if caps is not None else env_caps()
    names = compiled.node_names
    n = compiled.n_nodes
    nodes = scaledown.NodeOrder(compiled)
    pool = present is not None
    state = np.array(present, dtype=np.int8) if pool else None          # 0 absent, 1 present, 2 retired
    left = list(copies)
    waves: List[Wave] = []
    skipped: List[SkippedNode] = []
    moved = 0
    base = np.array(placed, dtype=np.int32)
    remaining = list(cand)
    pinned = pinned_pods(compiled, placed)
    recs = compiled.pod_recs
    while remaining:
        join = left[:max_surge] if pool else []
        out_nodes = np.nonzero(state != 1)[0].tolist() if pool else []       # absent or retired
        n_in = n - len(out_nodes) + len(join)
        m = min(per_wave, len(remaining), n_in - 1)
        if m == 0:
            skipped += [SkippedNode(names[c], len(waves), [LAST_NODE_REASON]) for c in remaining]
            break
        if remaining[0] in pinned:
            skipped.append(SkippedNode(names[remaining[0]], len(waves),
                                       [f"pod {recs[q].tmpl.namespace}/{recs[q].name} {why}" for q, why in pinned[remaining[0]]]))
            remaining.pop(0)
            continue
        m = next((j for j in range(1, m) if remaining[j] in pinned), m)       # the prefixes past a pinned node fail
        removed = [remaining[:j] for j in range(1, m + 1)]
        if pool:
            gone = [g for g in out_nodes if g not in set(join)]
            remain = [nodes.remaining(gone + r) for r in removed]
            raw = runner.run(remain, [np.asarray(join, np.uint32)] * len(remain))
        else:
            remain = [nodes.remaining(r) for r in removed]
            raw = runner.run(remain)
        k = 0
        for r in raw:
            if not (scaledown.drainable(r) and occupancy_ok(r, max_cpu, max_mem) and r.get("n_join_unscheduled", 0) == 0):
                break
            k += 1
        if k == 0:
            allowed = pdb_allowed(pdbs, base) if pdbs is not None else None
            d = scaledown.drain_results(compiled, base, removed[:1], remain[:1], raw[:1], max_cpu, max_mem, pdbs=pdbs, allowed=allowed)[0]
            why = join_reasons(compiled, raw[0], remain[0]) if pool else []
            skipped.append(SkippedNode(names[remaining[0]], len(waves), why + _reasons(d), d))
            remaining.pop(0)
            continue
        r = raw[k - 1]
        d = scaledown.drain_results(compiled, base, removed[k - 1:k], remain[k - 1:k], [r], max_cpu, max_mem)[0]
        w = Wave(Nodes=[names[c] for c in removed[k - 1]], Evicted=d.EvictedPods, Occupancy=d.Occupancy)
        if pool:
            w.Joined = [names[g] for g in join]
            w.JoinPods = join_pods(compiled, r)
        if pdbs is not None:
            for q in r["evicted"].tolist():
                for j in pdbs.pod_pdb[pdbs.pod_off[q]:pdbs.pod_off[q + 1]]:
                    nm = pdbs.names[int(j)]
                    w.PdbEvicted[nm] = w.PdbEvicted.get(nm, 0) + 1
        if pool:
            runner.commit(k - 1, True)
            state[join] = 1
            state[removed[k - 1]] = 2
            left = left[len(join):]
        else:
            runner.commit(k - 1)
        base = np.array(runner.placement()[0], dtype=np.int32)
        waves.append(w)
        moved += len(w.Evicted)
        remaining = remaining[k:]
    return waves, skipped, moved, left
