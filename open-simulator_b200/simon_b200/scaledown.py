"""Node drains and cluster scale-down planning: the reference's third use case (README.md:16, "Pods Migration: scaling down
cluster, defragmentation, etc."), which it names but has no code for.  The definition is this project's (include/simon_gpu.h,
simon_drain_run):

  * the live state is `placed`, the out_node of a full placement of the pod list (Simulate / the session's placements);
  * a drain removes some nodes; the remaining nodes keep their own nodeTree.list() order;
  * pods of DaemonSets of a removed node vanish with it; pods bound by spec.nodeName and pods with Open-Local volumes block the drain
    (they cannot be recreated elsewhere); every other pod of a removed node is evicted and placed again, in pod-list order, on the
    remaining nodes, on the live state minus the removed nodes' pods;
  * a drain is drainable when nothing blocks it, every evicted pod finds a node and, with PodDisruptionBudgets uploaded
    (disruption.py, Engine.pdbs_upload), it evicts no more members of any PDB than the PDB allows on the live state.  Vanished and
    blocked pods do not count against a PDB.  The result is the end state, not an eviction sequence.

With local volumes (local_volumes=True, on a cluster compiled with open_local=True; Engine.drain_run(..., local=True)) pods with
Open-Local volumes are evicted instead of blocking: they are placed again with the other evicted pods, through Open-Local's Filter,
Score and Bind on the remaining nodes, and their volumes are provisioned again there at the same sizes.  Their data is not carried
over, and the removed nodes' VGs and devices go with them: this answers whether the volumes fit elsewhere, not how to move the data.
Such drains also carry the VG sums of the remaining annotated nodes, and the MaxVG cap applies to them.

ScaleDownPlan sweeps every candidate node alone, orders the drainable ones by utilisation and removes the longest prefix of that order
whose every prefix drains and meets the satisfyResourceSetting caps (MaxCPU / MaxMemory, and MaxVG for drains with VG sums).  With
PDBs a prefix that violates one does not drain, so the first such prefix ends the plan, and the sweep marks such single-node drains
not drainable.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import abi
from .capacity import env_caps, env_vg_cap, occupancy_ok
from .compiler import SCW_GUARD_NODE, SCW_REQ_MCPU, SCW_REQ_MEM, Compiled, get_zone_key
from .objects import AppResource, ResourceTypes
from .workloads import PodRec

BLOCK_NODE_NAME = "bound to its node by spec.nodeName"
BLOCK_LOCAL_STORAGE = "has Open-Local volumes, which do not move"


@dataclass
class EvictedPod:
    Pod: PodRec
    From: str
    To: Optional[str]               # None: unschedulable on the remaining nodes
    GpuIndex: Optional[str] = None  # alibabacloud.com/gpu-index of a GPU-share pod that landed: one device id per GPU slot, "-"-joined


@dataclass
class BlockedPod:
    Pod: PodRec
    Node: str
    Reason: str


@dataclass
class PdbViolation:
    Name: str                       # "namespace/name"
    Evicted: int                    # members the drain evicts
    Allowed: int                    # disruptions the PDB allows on the live state


@dataclass
class DrainResult:
    RemovedNodes: List[str]
    Drainable: bool
    EvictedPods: List[EvictedPod] = field(default_factory=list)
    BlockedPods: List[BlockedPod] = field(default_factory=list)
    UnscheduledPods: list = field(default_factory=list)      # simulator.UnscheduledPod, FitError texts over the remaining nodes
    VanishedPods: int = 0
    Occupancy: Dict[str, int] = field(default_factory=dict)  # req_mcpu / alloc_mcpu / req_mem / alloc_mem over the remaining nodes
    CapsOk: bool = True                                       # occupancy_ok under MaxCPU / MaxMemory
    PdbViolations: List[PdbViolation] = field(default_factory=list)


@dataclass
class NodeSweep:
    """One candidate node drained alone."""
    Node: str
    Drainable: bool
    Utilisation: float              # max(cpu requested / allocatable, memory requested / allocatable) in the live state
    Evicted: int
    Unscheduled: int
    Blocked: int
    PdbViolated: int = 0            # PDBs the drain would violate


@dataclass
class ScaleDownPlan:
    RemovedNodes: List[str]          # the plan: remove these together
    Order: List[str]                 # drainable candidates by utilisation (ties in nodeTree order)
    Sweep: List[NodeSweep]
    Prefixes: List[dict]             # the raw results of the evaluated prefixes k = 1, 2, ... (each with k, ok)


# ---- remaining-node orders ---------------------------------------------------------------------------------------------------------

class NodeOrder:
    """nodeTree.list() of the nodes that remain after a drain, as compiled node indices.  node_tree_list over the remaining node
    objects, vectorised for sweeps: zones in order of their first remaining node (in the cluster's node order), round-robin over
    them, each zone's nodes in cluster order."""

    def __init__(self, compiled: Compiled):
        self.c = compiled
        n = compiled.n_nodes
        self.n = n
        orig = np.asarray(compiled.node_orig_index, dtype=np.int64)
        self.by_orig = np.argsort(orig, kind="stable")            # compiled indices in the cluster's node order
        zones: Dict[str, int] = {}
        zid = np.zeros(n, np.int64)
        for r, ci in enumerate(self.by_orig.tolist()):
            zid[r] = zones.setdefault(get_zone_key(compiled.node_objs[ci]), len(zones))
        self.zid = zid                                            # zone of the r-th node in cluster order
        self.nz = len(zones)
        self.rank_of_compiled = np.empty(n, np.int64)
        self.rank_of_compiled[self.by_orig] = np.arange(n)

    def remaining(self, removed: Sequence[int]) -> np.ndarray:
        keep = np.ones(self.n, bool)
        keep[self.rank_of_compiled[np.asarray(list(removed), dtype=np.int64)]] = False
        r = np.nonzero(keep)[0]                                   # remaining nodes, cluster order
        z = self.zid[r]
        by_zone = np.argsort(z, kind="stable")
        zs = z[by_zone]
        starts = np.r_[0, np.nonzero(np.diff(zs))[0] + 1] if len(zs) else np.zeros(0, np.int64)
        pos = np.empty(len(r), np.int64)                          # position within its zone among the remaining nodes
        pos[by_zone] = np.arange(len(r)) - np.repeat(starts, np.diff(np.r_[starts, len(r)]))
        first = np.full(max(self.nz, 1), self.n, np.int64)        # zones in order of their first remaining node
        np.minimum.at(first, z, r)
        zrank = np.argsort(np.argsort(first, kind="stable"), kind="stable")
        o = np.lexsort((zrank[z], pos))                           # round-robin: position first, then zone
        return self.by_orig[r[o]].astype(np.uint32)


# ---- live-state facts on the host ----------------------------------------------------------------------------------------------------

def _class_word(compiled: Compiled, word: int) -> np.ndarray:
    off = np.asarray(compiled.pods["class_off"], dtype=np.int64)
    blob = np.asarray(compiled.pods["class_blob"], dtype=np.int64)
    return blob[off[:-1] + word]


def pod_guard(compiled: Compiled) -> np.ndarray:
    """Per pod: the node whose removal makes it vanish (a DaemonSet pod's node), -1 none, -2 names no node."""
    cls = np.asarray(compiled.pods["pod_class"], dtype=np.int64)
    g = _class_word(compiled, SCW_GUARD_NODE)[cls]
    pin = compiled.pods.get("pod_pin_node")
    if pin is not None:
        g = np.where(g == -3, np.asarray(pin, dtype=np.int64), g)
    return g


def classify(compiled: Compiled, placed: np.ndarray, removed: Sequence[int], local_volumes: bool = False
             ) -> Tuple[List[int], List[Tuple[int, str]], List[int]]:
    """The pods of the removed nodes in pod order: (evicted, blocked as (pod, reason), vanished).  local_volumes: pods with
    Open-Local volumes are evicted instead of blocked (Engine.drain_run(..., local=True))."""
    placed = np.asarray(placed)
    rm = np.zeros(compiled.n_nodes, bool)
    rm[np.asarray(list(removed), dtype=np.int64)] = True
    guard = pod_guard(compiled)
    fixed = np.asarray(compiled.pods["pod_fixed_node"])
    local = compiled.storage.class_local if getattr(compiled, "storage", None) is not None else None
    cls = compiled.pods["pod_class"]
    ev, bl, va = [], [], []
    for q in np.nonzero((placed >= 0) & rm[np.maximum(placed, 0)])[0].tolist():
        if guard[q] >= 0 and rm[guard[q]]:
            va.append(q)
        elif fixed[q] >= 0:
            bl.append((q, BLOCK_NODE_NAME))
        elif local is not None and local[int(cls[q])] and not local_volumes:
            bl.append((q, BLOCK_LOCAL_STORAGE))
        else:
            ev.append(q)
    return ev, bl, va


def node_utilisation(compiled: Compiled, placed: np.ndarray) -> np.ndarray:
    """Per node of the live state: max(cpu requested / allocatable, memory requested / allocatable)."""
    placed = np.asarray(placed)
    cls = np.asarray(compiled.pods["pod_class"], dtype=np.int64)
    on = placed >= 0
    n = compiled.n_nodes
    rc = np.zeros(n, np.float64)
    rm = np.zeros(n, np.float64)
    np.add.at(rc, placed[on], _class_word(compiled, SCW_REQ_MCPU)[cls[on]].astype(np.float64))
    np.add.at(rm, placed[on], _class_word(compiled, SCW_REQ_MEM)[cls[on]].astype(np.float64))
    ac = np.asarray(compiled.snap["alloc_mcpu"], dtype=np.float64)
    am = np.asarray(compiled.snap["alloc_mem"], dtype=np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        u = np.maximum(np.where(ac > 0, rc / ac, 0.0), np.where(am > 0, rm / am, 0.0))
    return u


# ---- results -------------------------------------------------------------------------------------------------------------------------

def gpu_index(word: int) -> Optional[str]:
    """The alibabacloud.com/gpu-index value of a GPU-slot word (4 bits per device = the pod's slots on it): the device of every slot,
    ascending, joined by "-" as AllocateGpuId writes it (pkg/type/open-gpu-share/cache/gpunodeinfo.go:281-284) and GpuIdStrToIntList
    reads it back (utils/pod.go:101-105); None without slots."""
    devs = [d for d in range(8) for _ in range((word >> (4 * d)) & 15)]
    return "-".join(str(d) for d in devs) if devs else None


def drainable(r: dict) -> bool:
    """A drain result of Engine.drain_run: nothing blocked, every evicted pod placed, no PDB violated."""
    return r["n_blocked"] == 0 and r["n_unscheduled"] == 0 and r.get("n_pdb_violated", 0) == 0


def drain_results(compiled: Compiled, placed: np.ndarray, removed_lists: Sequence[Sequence[int]], remain_lists: Sequence[np.ndarray],
                  raw: Sequence[dict], max_cpu: Optional[int] = None, max_mem: Optional[int] = None, pdbs=None,
                  allowed: Optional[np.ndarray] = None, max_vg: Optional[int] = None) -> List[DrainResult]:
    """DrainResult per drain from Engine.drain_run(..., detail=True) results; pdbs (disruption.PdbTables) and allowed
    (Engine.pdbs_allowed on the live state) name the violated PDBs.  Results of drains with local volumes carry the VG sums: they go
    into Occupancy (vg_requested / vg_capacity) and CapsOk applies max_vg to them (default: env_vg_cap())."""
    from .simulator import UnscheduledPod, format_fit_error
    if max_cpu is None or max_mem is None:
        max_cpu, max_mem = env_caps()
    names = compiled.node_names
    recs = compiled.pod_recs
    placed = np.asarray(placed)
    fixed = np.asarray(compiled.pods["pod_fixed_node"])
    memo: dict = {}
    out = []
    for removed, remain, r in zip(removed_lists, remain_lists, raw):
        active = [int(x) for x in remain]
        res = DrainResult(RemovedNodes=[names[g] for g in removed], Drainable=drainable(r), VanishedPods=int(r["n_vanished"]))
        for j, e in zip(r.get("pdb_violated", []), r.get("pdb_evicted", [])):
            res.PdbViolations.append(PdbViolation(pdbs.names[int(j)] if pdbs is not None else str(int(j)), int(e),
                                                  int(allowed[int(j)]) if allowed is not None else -1))
        fails = {int(p): j for j, p in enumerate(r["fail_pod"])}
        for q, g, w in zip(r["evicted"].tolist(), r["node"].tolist(), r["gpu_slots"].tolist()):
            res.EvictedPods.append(EvictedPod(recs[q], names[placed[q]], names[g] if g >= 0 else None, gpu_index(w) if g >= 0 else None))
            if g < 0:
                j = fails.get(q)
                counts = r["fail_counts"][j] if j is not None else np.zeros(abi.N_FAIL_CODES, np.uint32)
                res.UnscheduledPods.append(UnscheduledPod(recs[q], format_fit_error(compiled, recs[q], counts, active=active, static_memo=memo)))
        for q in r["blocked"].tolist():
            res.BlockedPods.append(BlockedPod(recs[q], names[placed[q]], BLOCK_NODE_NAME if fixed[q] >= 0 else BLOCK_LOCAL_STORAGE))
        res.Occupancy = {k: int(r[k]) for k in ("req_mcpu", "alloc_mcpu", "req_mem", "alloc_mem")}
        if "vg_capacity" in r:
            if max_vg is None:
                max_vg = env_vg_cap()
            res.Occupancy.update(vg_requested=int(r["vg_requested"]), vg_capacity=int(r["vg_capacity"]))
            res.CapsOk = occupancy_ok(res.Occupancy, max_cpu, max_mem, max_vg)
        else:
            res.CapsOk = occupancy_ok(res.Occupancy, max_cpu, max_mem)
        out.append(res)
    return out


# ---- the planner ---------------------------------------------------------------------------------------------------------------------

def plan_scale_down(compiled: Compiled, placed: np.ndarray, runner: Callable[[List[np.ndarray]], List[dict]],
                    candidates: Optional[Sequence[int]] = None, max_remove: Optional[int] = None, batch: int = 64,
                    max_cpu: Optional[int] = None, max_mem: Optional[int] = None, max_vg: Optional[int] = None) -> ScaleDownPlan:
    """runner(remain_lists) -> per drain a dict with n_blocked, n_unscheduled, n_evicted, n_pdb_violated and the occupancy sums
    (Engine.drain_run with detail=False; on an engine with a PDB table the PDBs are honoured).  1. every candidate drained alone, in one run; 2. the drainable ones ordered by utilisation ascending, ties
    in nodeTree order; 3. prefixes k = 1, 2, ... of that order removed together, `batch` consecutive k per run; 4. the plan is the
    largest k such that every prefix up to k drains and meets the caps: the first failing k ends it (no monotonicity is assumed).
    max_vg (default env_vg_cap(), read at the first result with VG sums) applies to results that carry the VG sums (drains with local
    volumes) and is ignored for the others."""
    if max_cpu is None or max_mem is None:
        max_cpu, max_mem = env_caps()

    def caps_ok(r):
        nonlocal max_vg
        if "vg_capacity" not in r:
            return occupancy_ok(r, max_cpu, max_mem)
        if max_vg is None:
            max_vg = env_vg_cap()
        return occupancy_ok(r, max_cpu, max_mem, max_vg)
    names = compiled.node_names
    n = compiled.n_nodes
    cand = list(range(n)) if candidates is None else list(dict.fromkeys(int(c) for c in candidates))     # repeats dropped, order kept
    order = NodeOrder(compiled)
    util = node_utilisation(compiled, placed)
    sweep_raw = runner([order.remaining([c]) for c in cand]) if cand and n > 1 else []
    sweep = []
    good = []
    for c, r in zip(cand, sweep_raw):
        ok = drainable(r)
        sweep.append(NodeSweep(names[c], ok, float(util[c]), int(r["n_evicted"]), int(r["n_unscheduled"]), int(r["n_blocked"]),
                               int(r.get("n_pdb_violated", 0))))
        if ok:
            good.append(c)
    good.sort(key=lambda c: (util[c], c))            # compiled index order is nodeTree order
    kmax = min(len(good), n - 1)
    if max_remove is not None:
        kmax = min(kmax, int(max_remove))
    prefixes = []
    best = 0
    k = 1
    while k <= kmax:
        ks = list(range(k, min(k + batch, kmax + 1)))
        raw = runner([order.remaining(good[:j]) for j in ks])
        stop = False
        for j, r in zip(ks, raw):
            ok = drainable(r) and caps_ok(r)
            prefixes.append(dict(r, k=j, ok=ok))
            if not ok:
                stop = True
                break
            best = j
        if stop:
            break
        k = ks[-1] + 1
    return ScaleDownPlan(RemovedNodes=[names[c] for c in good[:best]], Order=[names[c] for c in good], Sweep=sweep, Prefixes=prefixes)


# ---- entry points on objects ---------------------------------------------------------------------------------------------------------

def drain(cluster: ResourceTypes, apps: List[AppResource], drains: List[List[str]], *opts, pdbs: Optional[List[dict]] = None,
          local_volumes: bool = False) -> List[DrainResult]:
    """NewSimulator(*opts), RunCluster(PrepareCluster(cluster)), ScheduleApp per app, then DrainNodes(drains, local_volumes).  pdbs: PDB
    objects to honour besides the cluster's and the apps' (given, even empty, the session runs WithPodDisruptionBudgets);
    local_volumes needs WithOpenLocal among opts."""
    from .simulator import NewSimulator, PrepareCluster, WithPodDisruptionBudgets
    if pdbs is not None:
        opts = opts + (WithPodDisruptionBudgets(pdbs),)
    with NewSimulator(*opts) as sim:
        sim.RunCluster(PrepareCluster(cluster))
        for app in apps:
            sim.ScheduleApp(app)
        return sim.DrainNodes(drains, local_volumes=local_volumes)
