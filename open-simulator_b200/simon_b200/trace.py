"""Replay traces of pod arrivals and departures on the live session, and size the cluster a trace needs (include/simon_gpu.h,
simon_trace_run).

A trace is an ordered list of Events.  A create is a Pod object that reaches the scheduler when its event comes; a delete names a pod of
the session or an earlier create as "namespace/name", and takes it off its node with RemovePod semantics.  A create that fails is not
retried.  The cluster is compiled as a grow superset (grow.build's machinery): the session's nodes plus kmax copies of `new_node`, the
session's pods, the copies' pods of the cluster's and the session apps' DaemonSets, then the trace's pods in event order, pending.
Scenario k is the session's nodes plus the first k copies; every k runs in one batch from the live state."""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import abi, capacity
from . import objects as O
from .compiler import compile_cluster
from .objects import Obj, ResourceTypes
from .scaledown import gpu_index
from .workloads import PodRec, generate_valid_pods_from_app_resources, make_valid_pod_by_pod, make_valid_pods_by_daemonset

CREATE, DELETE = "create", "delete"


@dataclass
class Event:
    time: float
    op: str                    # CREATE or DELETE
    pod: object                # CREATE: a Pod object; DELETE: "namespace/name" of a session pod or of an earlier create


def pod_key(pod) -> str:
    """"namespace/name" of a Pod object or a PodRec."""
    if isinstance(pod, PodRec):
        return f"{pod.tmpl.namespace}/{pod.name}"
    ns = O.namespace_of(pod) or "default"
    return f"{ns}/{O.name_of(pod)}"


def from_lifetimes(items: Sequence[Tuple[Obj, float, Optional[float]]]) -> List[Event]:
    """Events of (pod, start, end | None) lifetimes, ordered by time; at equal times deletes go before creates, and otherwise the order
    of `items` is kept.  A lifetime must end after it starts."""
    keyed = []
    for i, (pod, start, end) in enumerate(items):
        keyed.append(((start, 1, i), Event(start, CREATE, pod)))
        if end is not None:
            if not end > start:
                raise ValueError(f"from_lifetimes: pod {pod_key(pod)!r} ends at {end}, not after its start {start}")
            keyed.append(((end, 0, i), Event(end, DELETE, pod_key(pod))))
    keyed.sort(key=lambda t: t[0])
    return [e for _, e in keyed]


@dataclass
class TraceSet:
    """A compiled superset with a trace: what simon_trace_run needs of it."""
    compiled: object
    n_prefix: int
    placed: np.ndarray
    events: np.ndarray             # [n_events][2] (op, pod)
    times: List[float]
    n_base: int
    kmax: int
    scenarios: List[capacity.Scenario]


def build(sim, events: Sequence[Event], new_node: Optional[Obj] = None, kmax: int = 0) -> TraceSet:
    """The superset of a session with the trace's pods appended (see the module docstring).  Refused before any device work: an event
    that is neither a create nor a delete, a create of an object that is not a Pod or that sets spec.nodeName, a create whose name a
    pod of the session or an earlier create already holds, a delete of a name no pod holds at that point, a delete of a DaemonSet pod,
    and a superset past a class's pod-count bound (Compiled.class_pod_limit)."""
    from . import grow
    p = sim._plan()
    if p.segments != sim._segments or len(p.pods) != len(sim.placements):
        raise RuntimeError("ReplayTrace: the session's pods expand differently now: were the cluster or app objects changed?")
    base = list(p.nodes)
    specs = [new_node] if new_node is not None and kmax > 0 else []
    pool = [n for (_s, _i, n) in capacity.pool_nodes(specs, kmax)] if specs else []
    names = {O.name_of(n) for n in base}
    clash = next((O.name_of(n) for n in pool if O.name_of(n) in names), None)
    if clash is not None:
        raise ValueError(f"ReplayTrace: the new node name {clash!r} is a node of the session")
    nodes = base + pool
    pods: List[PodRec] = list(p.pods)
    n_prefix = len(pods)
    if pool:
        pods.extend(r for ds in sim.cluster.DaemonSets for r in make_valid_pods_by_daemonset(ds, pool))
        for app in sim.apps:
            pods.extend(generate_valid_pods_from_app_resources(pool, app.Name, ResourceTypes(DaemonSets=list(app.Resource.DaemonSets))))
    index: Dict[str, int] = {}
    for q, rec in enumerate(pods[:n_prefix]):
        index.setdefault(pod_key(rec), q)
    ev = [(abi.TRACE_CREATE, q) for q in range(n_prefix, len(pods))]        # the copies' DaemonSet pods are created at the start
    times = [events[0].time if events else 0.0] * len(ev)
    memo: dict = {}
    for k, e in enumerate(events):
        if e.op == CREATE:
            if not isinstance(e.pod, dict) or e.pod.get("kind", "Pod") != "Pod":
                raise ValueError(f"ReplayTrace: event {k} creates {type(e.pod).__name__}, not a Pod")
            rec = make_valid_pod_by_pod(e.pod, memo)
            if rec.node_name:
                raise ValueError(f"ReplayTrace: event {k} creates pod {pod_key(rec)!r}, which sets spec.nodeName")
            key = pod_key(rec)
            if key in index:
                raise ValueError(f"ReplayTrace: event {k} creates pod {key!r}, a name that exists already")
            index[key] = len(pods)
            ev.append((abi.TRACE_CREATE, len(pods)))
            pods.append(rec)
        elif e.op == DELETE:
            q = index.pop(str(e.pod), None)
            if q is None:
                raise ValueError(f"ReplayTrace: event {k} deletes {e.pod!r}, which no pod holds")
            if pods[q].tmpl.guard_node_name:
                raise ValueError(f"ReplayTrace: event {k} deletes {e.pod!r}, a DaemonSet pod")
            ev.append((abi.TRACE_DELETE, q))
        else:
            raise ValueError(f"ReplayTrace: event {k} has op {e.op!r}, not {CREATE!r} or {DELETE!r}")
        times.append(e.time)
    o = sim.options
    compiled = compile_cluster(nodes, pods, p.ctx, extra_plugins=sim._extra_plugins or None, open_local=o.openLocal,
                               storage_classes=list(sim.cluster.StorageClasss) if o.openLocal else None, local_devices=o.openLocalDevices)
    limit = compiled.class_pod_limit
    if limit is not None:
        cls = np.asarray(compiled.pods["pod_class"])
        over = np.nonzero(len(pods) > np.asarray(limit, dtype=np.int64)[cls])[0]
        if len(over):
            raise ValueError(f"ReplayTrace: {len(pods)} pods exceed the int32 bounds of the class of pod {int(over[0])}")
    scen = capacity.scenario_nodes(compiled, nodes, len(base), kmax, 1, range(kmax + 1)) if pool else \
        capacity.scenario_nodes(compiled, nodes, len(base), 0, 1, [0])
    return TraceSet(compiled, n_prefix, grow.remap(sim.compiled, compiled, sim.placements), np.array(ev, np.uint32).reshape(-1, 2),
                    times, len(base), kmax if pool else 0, scen)


@dataclass
class TraceK:
    K: int
    Creates: int                       # creates of pods that exist in the scenario
    Failures: list                     # simulator.UnscheduledPod of each failed create, with its event time as .Time
    Deletes: int                       # deletes that took a pod off a node
    FirstFailureTime: Optional[float]
    Samples: Dict[str, np.ndarray] = field(default_factory=dict)     # the simon_trace_point fields, and "time"


@dataclass
class CreatedPod:
    Pod: PodRec
    Node: Optional[str]                # None: unschedulable
    GpuIndex: Optional[str] = None


@dataclass
class TraceResult:
    PerK: List[TraceK]
    MinNodes: int                      # the least k with no failed create, -1 if none up to kmax
    AllFromMinNodes: bool              # every k from MinNodes to kmax has no failed create (feasibility is not monotone in k)
    K: int                             # the k the placement below describes: MinNodes, or kmax when none
    Pods: List[CreatedPod]


def sample_events(n_events: int, samples: int) -> List[int]:
    """Up to `samples` event indices spread evenly over [0, n_events), the last event included."""
    if n_events == 0 or samples <= 0:
        return []
    m = min(samples, n_events)
    return [(i + 1) * n_events // m - 1 for i in range(m)]


def replay(eng, ts: TraceSet, samples: int = 100) -> TraceResult:
    """Every k of `ts` as one trace batch on `eng` (an Engine holding ts.compiled), with detail."""
    from .simulator import UnscheduledPod, format_fit_error
    c = ts.compiled
    sm = sample_events(len(ts.events), samples)
    raw = eng.trace_run(ts.placed, ts.n_prefix, ts.events, [s.nodes for s in ts.scenarios], samples=sm, detail=True)
    create_time = {int(q): ts.times[i] for i, (op, q) in enumerate(ts.events.tolist()) if op == abi.TRACE_CREATE}
    per_k, memo = [], {}
    for k, (s, r) in enumerate(zip(ts.scenarios, raw)):
        active = s.nodes.tolist()
        fails = []
        for j, q in enumerate(r["fail_pod"].tolist()):
            rec = c.pod_recs[q]
            u = UnscheduledPod(rec, format_fit_error(c, rec, r["fail_counts"][j], active=active, static_memo=memo))
            u.Time = create_time[q]
            fails.append(u)
        pts = r["samples"]
        smp = {f: np.asarray(pts[f]) for f in abi.TRACE_POINT_DTYPE.names if f != "reserved"}
        smp["time"] = np.array([ts.times[int(e)] for e in pts["event"]], np.float64)
        exists = int((r["node"] != -3).sum())
        per_k.append(TraceK(k, exists, fails, r["n_removed"], fails[0].Time if fails else None, smp))
    ok = [not t.Failures for t in per_k]
    min_nodes = next((k for k, v in enumerate(ok) if v), -1)
    K = min_nodes if min_nodes >= 0 else len(per_k) - 1
    pods = []
    r = raw[K]
    for t, (g, w) in enumerate(zip(r["node"].tolist(), r["gpu_slots"].tolist())):
        if g == -3:
            continue
        pods.append(CreatedPod(c.pod_recs[ts.n_prefix + t], c.node_names[g] if g >= 0 else None, gpu_index(w) if g >= 0 else None))
    return TraceResult(per_k, min_nodes, min_nodes >= 0 and all(ok[min_nodes:]), K, pods)
