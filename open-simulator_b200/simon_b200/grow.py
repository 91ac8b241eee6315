"""Nodes to add to the live cluster for new apps: the add-node search of `simon apply` on a running cluster (the reference's second use
case, README.md:15, where `simon apply` with cluster.kubeConfig reads the running cluster and adds nodes to it), on the session's state.

A grow batch (include/simon_gpu.h) runs on a superset cluster compiled once: the session's nodes plus kmax copies of every candidate
spec, and the session's pod list followed by a pending tail (the DaemonSet pods of the pool copies, then the new apps' pods).  Scenario
(spec, k) activates the session's nodes plus the first k copies of the spec and places the tail from the live state, so the running
pods stay where they are and keep their GPU-share devices and Open-Local volumes.  The search over k is capacity.search_min_k, the one
`apply.auto_add_nodes` runs."""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import abi, capacity
from . import objects as O
from .algo import order_app_pods
from .compiler import Compiled, compile_cluster
from .objects import AppResource, Obj, ResourceTypes
from .scaledown import gpu_index
from .workloads import PodRec, generate_valid_pods_from_app_resources, make_valid_pods_by_daemonset

# the largest cluster a placement kernel takes: 16 CTAs x 320 threads x 64 node slots (the large-cluster variant)
ENGINE_MAX_NODES = 16 * 320 * 64
METHODS = ("sweep", "bisect")


@dataclass
class GrowSet:
    """A compiled superset and what a grow batch needs of it."""
    compiled: Compiled
    n_prefix: int                      # the session's pods, first in compiled.pod_recs
    placed: np.ndarray                 # their placements as superset node indices
    n_base: int
    kmax: int
    n_specs: int
    scenarios: List[capacity.Scenario]     # every (spec, k <= kmax), spec by spec (sid = spec * (kmax + 1) + k)
    segments: List[Tuple[str, int, int]]   # (what, first, count) of the tail: "cluster-daemonsets", one per earlier app, one per new app

    def scenario(self, spec: int, k: int) -> capacity.Scenario:
        return self.scenarios[spec * (self.kmax + 1) + k]


@dataclass
class NewPod:
    Pod: PodRec
    Node: Optional[str]                # None: unschedulable
    GpuIndex: Optional[str] = None     # alibabacloud.com/gpu-index (scaledown.gpu_index)


@dataclass
class SpecPlan:
    Spec: str                          # the candidate node's name
    NewNodeNum: int                    # minimal k (0: the apps fit already), -1: none up to kmax
    PerK: Dict[int, Dict[str, int]] = field(default_factory=dict)   # counts and occupancy of every k evaluated
    K: int = 0                         # the k the detail below describes: NewNodeNum, or kmax when none fits
    Pods: List[NewPod] = field(default_factory=list)               # the tail pods that exist at K, in pod order
    UnscheduledPods: list = field(default_factory=list)            # simulator.UnscheduledPod of the tail at K


@dataclass
class AddNodesPlan:
    Specs: List[SpecPlan]
    Best: Optional[Dict[str, object]]  # {"spec": index, "Spec": name, "k": k}: min k, ties to the lowest spec; None if none fits
    Rounds: int
    ScenariosEvaluated: int


def build(sim, apps: Sequence[AppResource], specs: Sequence[Obj], kmax: int) -> GrowSet:
    """The superset of a session (simulator.Simulator after RunCluster): its nodes plus kmax copies of every spec
    (capacity.pool_nodes), its pod list exactly as Simulator._plan() gives it, then the pool copies' pods of the cluster's DaemonSets,
    those of every earlier app's DaemonSets in app order (a DaemonSet covers nodes that join later), then each new app's pods generated
    over the session's nodes and the pool and ordered as ScheduleApp orders them."""
    p = sim._plan()
    if p.segments != sim._segments or len(p.pods) != len(sim.placements):
        raise RuntimeError("PlanAddNodes: the session's pods expand differently now: were the cluster or app objects changed?")
    base = list(p.nodes)
    names = {O.name_of(n) for n in base}
    n_nodes = len(base) + kmax * len(specs)
    if n_nodes > ENGINE_MAX_NODES:
        raise ValueError(f"PlanAddNodes: {len(base)} nodes + {kmax} x {len(specs)} candidates = {n_nodes} nodes exceed the engine's "
                         f"{ENGINE_MAX_NODES}; lower kmax")
    pool = [n for (_s, _i, n) in capacity.pool_nodes(specs, kmax)]
    clash = next((O.name_of(n) for n in pool if O.name_of(n) in names), None)
    if clash is not None:
        raise ValueError(f"PlanAddNodes: the candidate name {clash!r} is a node of the session")
    nodes = base + pool
    pods: List[PodRec] = list(p.pods)
    n_prefix = len(pods)
    segments = []

    def add(what, recs):
        segments.append((what, len(pods), len(recs)))
        pods.extend(recs)
    add("cluster-daemonsets", [r for ds in sim.cluster.DaemonSets for r in make_valid_pods_by_daemonset(ds, pool)])
    for app in sim.apps:
        add(app.Name, generate_valid_pods_from_app_resources(pool, app.Name, ResourceTypes(DaemonSets=list(app.Resource.DaemonSets))))
    for app in apps:
        app_pods = generate_valid_pods_from_app_resources(nodes, app.Name, app.Resource)
        order_app_pods(app_pods)
        add(app.Name, app_pods)
    o = sim.options
    storage_classes = None
    if o.openLocal:
        storage_classes = list(sim.cluster.StorageClasss) + [sc for a in list(sim.apps) + list(apps) for sc in a.Resource.StorageClasss]
    compiled = compile_cluster(nodes, pods, p.ctx, extra_plugins=sim._extra_plugins or None, open_local=o.openLocal,
                               storage_classes=storage_classes, local_devices=o.openLocalDevices)
    return GrowSet(compiled, n_prefix, remap(sim.compiled, compiled, sim.placements), len(base), kmax, len(specs),
                   capacity.scenario_nodes(compiled, nodes, len(base), kmax, len(specs), range(kmax + 1)), segments)


def remap(src: Compiled, dst: Compiled, placed: np.ndarray) -> np.ndarray:
    """Placements on `src`'s nodes as indices of the nodes of `dst` with the same names; entries below 0 stay."""
    to = np.array([dst.node_index(nm) for nm in src.node_names] + [0], np.int32)
    placed = np.asarray(placed, np.int32)
    out = np.where(placed >= 0, to[np.where(placed >= 0, placed, len(src.node_names))], placed).astype(np.int32)
    if (out[placed >= 0] < 0).any():
        raise RuntimeError("PlanAddNodes: a placed pod's node is missing from the superset")
    return out


def feasible(res: Dict[str, int], max_cpu: int, max_mem: int, max_vg: int) -> bool:
    """No existing tail pod unschedulable, and satisfyResourceSetting's caps over the active nodes."""
    return res["n_unscheduled"] == 0 and capacity.occupancy_ok(res, max_cpu, max_mem, max_vg)


def plan(eng, gs: GrowSet, spec_names: Sequence[str], method: str = "sweep", max_cpu: Optional[int] = None,
         max_mem: Optional[int] = None, max_vg: Optional[int] = None) -> AddNodesPlan:
    """The search on `eng` (an Engine holding gs.compiled), then one batch of detail at each spec's K."""
    from .simulator import UnscheduledPod, format_fit_error
    if method not in METHODS:
        raise ValueError(f"PlanAddNodes: unknown method {method!r} (one of {', '.join(METHODS)})")
    if max_cpu is None or max_mem is None:
        ec, em = capacity.env_caps()
        max_cpu = ec if max_cpu is None else max_cpu
        max_mem = em if max_mem is None else max_mem
    local = gs.compiled.storage is not None
    if max_vg is None:
        max_vg = capacity.env_vg_cap() if local else 100
    keys = ("n_unscheduled", "n_scheduled", "req_mcpu", "alloc_mcpu", "req_mem", "alloc_mem") + (("vg_requested", "vg_capacity") if local else ())
    done: Dict[Tuple[int, int], Dict[str, int]] = {}
    eng.last_grow_batches = []

    def evaluate(pairs):
        todo = [pk for pk in dict.fromkeys(pairs) if pk not in done]
        if not todo:
            return
        raw = eng.grow_run(gs.placed, gs.n_prefix, [gs.scenario(s, k).nodes for s, k in todo], detail=False)
        eng.last_grow_batches.append(eng.last_grow)
        for pk, r in zip(todo, raw):
            done[pk] = {q: int(r[q]) for q in keys}

    def ok(s, k):
        return feasible(done[(s, k)], max_cpu, max_mem, max_vg)

    best_k, rounds = capacity.search_min_k(gs.n_specs, gs.kmax, method, evaluate, ok)
    key = capacity.INFEASIBLE_KEY
    for s, k in enumerate(best_k):
        if k >= 0:
            key = min(key, capacity.scenario_key(gs.scenario(s, k), done[(s, k)], max_cpu, max_mem, max_vg))
    best = capacity.decode_key(key)
    out = [SpecPlan(spec_names[s], k, {kk: dict(r) for (ss, kk), r in sorted(done.items()) if ss == s}, k if k >= 0 else gs.kmax)
           for s, k in enumerate(best_k)]
    # the detail at each spec's K, one batch
    c = gs.compiled
    if out:
        raw = eng.grow_run(gs.placed, gs.n_prefix, [gs.scenario(s, sp.K).nodes for s, sp in enumerate(out)], detail=True)
        eng.last_grow_batches.append(eng.last_grow)
        memo: dict = {}
        for s, (sp, r) in enumerate(zip(out, raw)):
            active = gs.scenario(s, sp.K).nodes.tolist()
            fails = {int(q): j for j, q in enumerate(r["fail_pod"].tolist())}
            for t, (g, w) in enumerate(zip(r["node"].tolist(), r["gpu_slots"].tolist())):
                if g == -3:
                    continue
                q = gs.n_prefix + t
                rec = c.pod_recs[q]
                sp.Pods.append(NewPod(rec, c.node_names[g] if g >= 0 else None, gpu_index(w) if g >= 0 else None))
                if g == -1:
                    j = fails.get(q)
                    counts = r["fail_counts"][j] if j is not None else np.zeros(abi.N_FAIL_CODES, np.uint32)
                    sp.UnscheduledPods.append(UnscheduledPod(rec, format_fit_error(c, rec, counts, active=active, static_memo=memo)))
    best_out = None if best is None else {"spec": gs.scenarios[best["scenario"]].spec,
                                          "Spec": spec_names[gs.scenarios[best["scenario"]].spec], "k": best["k"]}
    return AddNodesPlan(out, best_out, rounds, len(done))
