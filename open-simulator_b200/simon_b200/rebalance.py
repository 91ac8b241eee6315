"""Migration plans for defragmentation: the reference's "Pods Migration" use case (README.md:16), which it names without code.  The
definition is this project's (include/simon_gpu.h, simon_moves_plan): starting from the live state, the best feasible candidate move
by (gain descending, move index ascending) is applied, then every candidate is scored again on the state it leaves, until max_moves
migrations are planned or no move gains at least min_gain.  Each pod moves at most once.  Gains, filters and the move scope are those
of the candidate-move scoring (moves.py).  The whole plan runs on the device; the live state is not changed.

With PodDisruptionBudgets (disruption.py) each PDB starts with the disruptions it allows on the live state; a pod with a PDB at 0 is not
moved, and each migration spends one unit of every PDB of its pod.  Budgets are not restored within a plan: its migrations are one
batch of evictions that violates no PDB.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence

import numpy as np

from . import abi
from .compiler import Compiled
from .scaledown import NodeOrder, gpu_index
from .workloads import PodRec

MAX_CANDIDATES = 1 << 26            # 512 MiB of moves on the device, and as much scoring output per step
STOP_REASONS = {abi.PLAN_STOP_NO_MOVE: "NoMove", abi.PLAN_STOP_MAX_MOVES: "MaxMoves"}


@dataclass
class Migration:
    Pod: PodRec
    From: str
    To: str
    Gain: int
    GpuIndex: Optional[str] = None  # alibabacloud.com/gpu-index on the target of a GPU-share pod: one device id per slot, "-"-joined


@dataclass
class MigrationPlan:
    Migrations: List[Migration] = field(default_factory=list)
    StopReason: str = ""             # "NoMove": no remaining move gains min_gain; "MaxMoves": max_moves migrations planned
    Excluded: int = 0                # GPU-share pods whose slot word is saturated on a device: never moved
    NodePods: Dict[str, List[str]] = field(default_factory=dict)     # pod names per node after the plan (nodes in index order)
    KernelMs: float = 0.0
    PdbBlocked: int = 0              # placed pods a PDB without budget on the live state keeps in place
    PdbExhausted: List[str] = field(default_factory=list)            # PDBs whose budget the plan used up


def candidates(compiled: Compiled, placement, sources: Optional[Sequence[int]] = None, targets: Optional[Sequence[int]] = None,
               cap: int = MAX_CANDIDATES) -> np.ndarray:
    """Every pod placed on a source node x every target node other than its own, as a uint32 [n, 2] move list (pod, target).
    Pod-major, pods ascending, targets in nodeTree order, so equal gains go to the lowest pod, then the first target in that order.
    sources / targets: node indices (None: every node).  Raises ValueError when the list would exceed `cap` moves."""
    placement = np.asarray(placement, dtype=np.int64)
    n = compiled.n_nodes
    order = NodeOrder(compiled).remaining([]).astype(np.int64)
    if targets is not None:
        want = np.zeros(n, bool)
        want[np.asarray(list(targets), dtype=np.int64)] = True
        order = order[want[order]]
    src = np.ones(n, bool) if sources is None else np.zeros(n, bool)
    if sources is not None:
        src[np.asarray(list(sources), dtype=np.int64)] = True
    pods = np.nonzero((placement >= 0) & src[np.maximum(placement, 0)])[0]
    in_targets = np.zeros(n, bool)
    in_targets[order] = True
    total = len(pods) * len(order) - int(in_targets[placement[pods]].sum())
    if total > cap:
        raise ValueError(f"{total} candidate moves exceed the cap of {cap}: narrow the sources or targets")
    mv = np.empty((len(pods), len(order), 2), np.uint32)
    mv[:, :, 0] = pods[:, None]
    mv[:, :, 1] = order[None, :]
    keep = mv[:, :, 1].astype(np.int64) != placement[pods][:, None]
    return mv[keep].reshape(-1, 2)


def from_raw(compiled: Compiled, steps: np.ndarray, stop_reason: int, excluded: int, placement, kernel_ms: float = 0.0) -> MigrationPlan:
    """MigrationPlan from the engine's raw plan: steps with fields pod, from, to, gain, gpu_slots (Engine.moves_plan) and the plan's
    end placement (Engine.moves_plan_download)."""
    names, recs = compiled.node_names, compiled.pod_recs
    out = MigrationPlan(StopReason=STOP_REASONS.get(int(stop_reason), str(stop_reason)), Excluded=int(excluded), KernelMs=float(kernel_ms))
    gpu_cls = _gpu_classes(compiled)
    cls = np.asarray(compiled.pods["pod_class"], dtype=np.int64)
    for s in steps:
        q = int(s["pod"])
        out.Migrations.append(Migration(recs[q], names[int(s["from"])], names[int(s["to"])], int(s["gain"]),
                                        gpu_index(int(s["gpu_slots"])) if gpu_cls[cls[q]] else None))
    placement = np.asarray(placement)
    out.NodePods = {nm: [] for nm in names}
    for q in np.nonzero(placement >= 0)[0].tolist():
        out.NodePods[names[int(placement[q])]].append(recs[q].name)
    return out


def _gpu_classes(compiled: Compiled) -> np.ndarray:
    from .compiler import SCW_GPU_MEM
    off = np.asarray(compiled.pods["class_off"], dtype=np.int64)
    blob = np.asarray(compiled.pods["class_blob"], dtype=np.int64)
    return blob[off[:-1] + SCW_GPU_MEM] > 0


def plan(engine, compiled: Compiled, moves: np.ndarray, max_moves: int, min_gain: int = 1, scope: int = 0, pdbs=None) -> MigrationPlan:
    """A migration plan over `moves` (e.g. candidates(...)) on the engine's live state, under the move scope `scope`
    (abi.MOVES_SCOPE_* bits); pdbs: disruption.PdbTables of the engine's pod list, uploaded and honoured.  The engine's live state is
    not changed; its move list, scope and PDB table are."""
    from . import disruption
    engine.moves_set_scope(scope)
    engine.moves_upload(moves, 0)
    if pdbs is not None:
        engine.pdbs_upload(pdbs)
        allowed = engine.pdbs_allowed()
    r = engine.moves_plan(max_moves, min_gain)
    placement, _ = engine.moves_plan_download()
    out = from_raw(compiled, r["steps"], r["stop_reason"], r["excluded"], placement, r["kernel_ms"])
    out.PdbBlocked = r["pdb_blocked"]
    if pdbs is not None:
        out.PdbExhausted = [pdbs.names[j] for j in disruption.exhausted(pdbs, allowed, r["steps"]["pod"])]
    return out
