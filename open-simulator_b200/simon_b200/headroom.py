"""Scheduling headroom of the live cluster: how many more replicas of a pod fit, where they go and what stops the next one.

A probe (pod q, max_replicas R) places replicas of q one at a time, each through the full scheduling cycle on the state the ones before
it leave, until one does not fit (Unschedulable) or R are placed (MaxReplicas).  It runs on the device as one scenario of a probe batch
(Engine.probe_run, simon_probe_run); the live state itself is not changed.  This is the capacity-planning use case of the reference
(README.md:14) asked of the running cluster; the reference has no code for it, so the definition is this library's
(include/simon_gpu.h)."""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import abi
from .compiler import Compiled
from .objects import AppResource, ResourceTypes
from .scaledown import gpu_index, pod_guard

# the kind a workload's pods record (workloads.py): a Deployment's pods are owned by its ReplicaSet of the same name, a CronJob's by
# its Job, as the reference expands them
_POD_OWNER_KIND = {"Deployment": "ReplicaSet", "CronJob": "Job"}
STOPPED = {abi.PROBE_STOP_UNSCHEDULABLE: "Unschedulable", abi.PROBE_STOP_MAX_REPLICAS: "MaxReplicas"}


@dataclass
class HeadroomResult:
    Probe: str                       # the workload reference "Kind/namespace/name", or "Pod/namespace/name" of a template
    Replicas: int                    # replicas placed
    Stopped: str                     # "Unschedulable" or "MaxReplicas"
    Reason: Optional[str] = None     # Unschedulable: the FitError text of the replica that did not fit
    Nodes: List[str] = field(default_factory=list)                   # the node of each replica, in order
    GpuIndex: List[Optional[str]] = field(default_factory=list)      # per replica, alibabacloud.com/gpu-index (scaledown.gpu_index)
    Occupancy: Dict[str, int] = field(default_factory=dict)          # req_mcpu / alloc_mcpu / req_mem / alloc_mem after the replicas,
    #                                                                   and vg_requested / vg_capacity with Open-Local


def free_pod_slots(compiled: Compiled, placed: np.ndarray) -> int:
    """Sum over the nodes of max(0, allocatable pods - pods placed there): no probe can place more replicas than this."""
    placed = np.asarray(placed)
    on = np.bincount(placed[placed >= 0], minlength=compiled.n_nodes)[:compiled.n_nodes]
    return int(np.maximum(0, np.asarray(compiled.snap["alloc_pods"], np.int64) - on).sum())


def workload_pods(compiled: Compiled, refs: Sequence[str]) -> List[int]:
    """Per reference "Kind/namespace/name" (a bare pod: "Pod/namespace/name"), the first pod of that workload in pod-list order."""
    first: Dict[Tuple[str, str, str], int] = {}
    for q, r in enumerate(compiled.pod_recs):
        first.setdefault((r.tmpl.workload_kind, r.tmpl.workload_namespace, r.workload_name), q)
    out = []
    for ref in refs:
        parts = ref.split("/")
        if len(parts) != 3 or not all(parts):
            raise ValueError(f"Headroom: {ref!r} is not a workload reference Kind/namespace/name")
        q = first.get((_POD_OWNER_KIND.get(parts[0], parts[0]), parts[1], parts[2]))
        if q is None:
            raise ValueError(f"Headroom: no workload {ref!r} in the session's cluster or apps")
        out.append(q)
    return out


def workload_pod(compiled: Compiled, ref: str) -> int:
    """workload_pods of one reference."""
    return workload_pods(compiled, [ref])[0]


def check_probe(compiled: Compiled, q: int, replicas: int, what: str, guard: Optional[np.ndarray] = None) -> None:
    """The host's refusals of one probe, before any device work (guard: scaledown.pod_guard(compiled), if already at hand)."""
    if replicas < 1:
        raise ValueError(f"Headroom: max_replicas must be at least 1 (got {replicas})")
    guard = pod_guard(compiled) if guard is None else guard
    if compiled.pod_recs[q].tmpl.workload_kind == "DaemonSet" or guard[q] >= 0:
        raise ValueError(f"Headroom: {what} is a DaemonSet pod: its replicas are one per node, not a count that fits")
    if int(compiled.pods["pod_fixed_node"][q]) != -1:
        raise ValueError(f"Headroom: {what} is bound by spec.nodeName and never reaches the scheduler")
    n = compiled.pods_dims["n_pods"]
    limit = compiled.class_pod_limit[int(compiled.pods["pod_class"][q])]
    if n + replicas > limit:
        raise ValueError(f"Headroom: {what}: {n} pods + {replicas} replicas exceed the int32 bounds of its class's tables "
                         f"({limit} pods); lower max_replicas")


def results(compiled: Compiled, labels: Sequence[str], pods: Sequence[int], raw: Sequence[dict]) -> List[HeadroomResult]:
    """HeadroomResult per probe from Engine.probe_run(..., detail=True).  Reason carries the histogram's reasons and counts, without
    the per-node Open-Gpu-Share and Open-Local detail."""
    from .simulator import format_fit_error
    names = compiled.node_names
    memo: dict = {}
    out = []
    for label, q, r in zip(labels, pods, raw):
        res = HeadroomResult(Probe=label, Replicas=int(r["n_placed"]), Stopped=STOPPED[int(r["stop_reason"])],
                             Nodes=[names[g] for g in r["node"].tolist()], GpuIndex=[gpu_index(w) for w in r["gpu_slots"].tolist()])
        if r["stop_reason"] == abi.PROBE_STOP_UNSCHEDULABLE:
            res.Reason = format_fit_error(compiled, compiled.pod_recs[q], r["fail_counts"], static_memo=memo)
        res.Occupancy = {k: int(r[k]) for k in ("req_mcpu", "alloc_mcpu", "req_mem", "alloc_mem", "vg_requested", "vg_capacity") if k in r}
        out.append(res)
    return out


def run(eng, compiled: Compiled, placed: np.ndarray, probes: Sequence[Tuple[str, int, int]]) -> List[HeadroomResult]:
    """probes: (label, pod, max_replicas) each, checked (check_probe) before the batch runs on `eng` from the live state `placed`."""
    guard = pod_guard(compiled)
    for label, q, rr in probes:
        check_probe(compiled, q, rr, label, guard)
    raw = eng.probe_run(placed, [(q, rr) for _l, q, rr in probes], detail=True)
    return results(compiled, [p[0] for p in probes], [p[1] for p in probes], raw)


def estimate(cluster: ResourceTypes, apps: List[AppResource], probes: list, *opts, max_replicas: Optional[int] = None
             ) -> List[HeadroomResult]:
    """NewSimulator(*opts), RunCluster(PrepareCluster(cluster)), ScheduleApp per app, then Headroom(probes, max_replicas)."""
    from .simulator import NewSimulator, PrepareCluster
    with NewSimulator(*opts) as sim:
        sim.RunCluster(PrepareCluster(cluster))
        for app in apps:
            sim.ScheduleApp(app)
        return sim.Headroom(probes, max_replicas=max_replicas)
