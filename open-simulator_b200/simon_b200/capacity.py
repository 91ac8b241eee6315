"""Capacity planning: the add-node search of `simon apply` (pkg/apply/apply.go:203-259) as a batch of what-if scenarios.

The reference re-runs a full Simulate() for every candidate node count k typed by the user, with k copies of ONE
node spec (utils.NewFakeNodes, pkg/utils/utils.go:885-901), and accepts a trial when no pod is unschedulable and
satisfyResourceSetting (apply.go:689-775: average CPU / memory occupancy <= MaxCPU / MaxMemory) holds.  Here every
(spec, k) pair is one independent scenario:
  * one compiled "superset" cluster holds the base nodes plus a pool of kmax copies of every candidate spec;
  * a scenario activates base + the first k copies of its spec, in ITS OWN nodeTree.list() order;
  * DaemonSet pods generated for pool nodes carry a guard node and exist only where that node is active;
  * scenarios are independent units: they are sharded round-robin over ranks (one process per GPU) and the global
    optimum is ONE all-reduce(MIN) of a packed int64 key  (k << 32 | scenario id)  — NCCL over NVLink when the
    ranks are GPUs.  There is no other data-path collective.
"""
from __future__ import annotations

import os
import re
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import objects as O
from .algo import order_app_pods
from .compiler import ClusterContext, Compiled, compile_cluster, node_tree_list
from .objects import AppResource, Obj, ResourceTypes, deep_copy
from .workloads import (PodRec, generate_valid_pods_from_app_resources, get_valid_pod_exclude_daemonset,
                        make_valid_node_by_node, make_valid_pods_by_daemonset)

INFEASIBLE_KEY = (1 << 62)


@dataclass
class Scenario:
    sid: int
    spec: int           # index of the candidate node spec
    k: int              # copies of that spec added
    nodes: np.ndarray   # active node indices (into the compiled snapshot) in this scenario's nodeTree.list() order


@dataclass
class ScenarioSet:
    compiled: Compiled
    scenarios: List[Scenario]
    pods: List[PodRec]
    n_base: int


def build_scenarios(cluster: ResourceTypes, apps: List[AppResource], specs: Sequence[Obj], ks: Sequence[int],
                    open_local: bool = False, local_devices: bool = False) -> ScenarioSet:
    """Superset cluster + one scenario per (spec, k in ks).

    open_local / local_devices: compile the superset with the Open-Local plugin (compile_cluster's switches), the StorageClasses
    taken from the cluster and the apps as Simulate() does.  The pool copies of a spec carry its simon/node-local-storage
    annotation (make_valid_node_by_node keeps annotations, like NewFakeNodes), so each copy adds the spec's VGs and devices."""
    kmax = max(ks) if len(ks) else 0
    base = list(cluster.Nodes)
    pool = pool_nodes(specs, kmax)
    nodes = base + [n for (_s, _i, n) in pool]
    # pod list over the superset (DaemonSet pods are generated per node and guarded by it)
    pods: List[PodRec] = get_valid_pod_exclude_daemonset(cluster)
    for ds in cluster.DaemonSets:
        pods.extend(make_valid_pods_by_daemonset(ds, nodes))
    for app in apps:
        app_pods = generate_valid_pods_from_app_resources(nodes, app.Name, app.Resource)
        order_app_pods(app_pods)
        pods.extend(app_pods)
    ctx = ClusterContext(services=list(cluster.Services), replicasets=list(cluster.ReplicaSets),
                         statefulsets=list(cluster.StatefulSets))
    storage_classes = list(cluster.StorageClasss) + [sc for a in apps for sc in a.Resource.StorageClasss] if open_local else None
    compiled = compile_cluster(nodes, pods, ctx, open_local=open_local, storage_classes=storage_classes, local_devices=local_devices)
    nb = len(base)
    scenarios = scenario_nodes(compiled, nodes, nb, kmax, len(specs), ks)
    return ScenarioSet(compiled, scenarios, pods, nb)


def pool_nodes(specs: Sequence[Obj], kmax: int) -> List[Tuple[int, int, Obj]]:
    """The candidate pool of a superset: (spec, ordinal, node) for kmax copies of every spec, spec by spec."""
    pool: List[Tuple[int, int, Obj]] = []
    for si, spec in enumerate(specs):
        work = deep_copy(spec)
        for i in range(kmax):
            # NewFakeNodes mutates its template across iterations (pkg/utils/utils.go:890-899); names are
            # simon-<rand5> in the reference, simon-<spec>-<ordinal> here
            n = make_valid_node_by_node(work, f"{O.NEW_NODE_NAME_PREFIX}-{si:02d}-{i:05d}")
            n["metadata"]["labels"][O.LABEL_NEW_NODE] = ""
            pool.append((si, i, deep_copy(n)))
    return pool


def scenario_nodes(compiled: Compiled, nodes: List[Obj], nb: int, kmax: int, n_specs: int, ks: Sequence[int]) -> List[Scenario]:
    """One Scenario per (spec, k in ks), spec by spec: the nb base nodes plus the first k pool copies of the spec (nodes = base +
    pool_nodes(specs, kmax), compiled as `compiled`), in the scenario's own nodeTree.list() order as compiled node indices."""
    orig_to_compiled = np.zeros(len(nodes), np.int64)
    for ci, oi in enumerate(compiled.node_orig_index):
        orig_to_compiled[oi] = ci
    scenarios: List[Scenario] = []
    for si in range(n_specs):
        for k in ks:
            members = list(range(nb)) + [nb + si * kmax + i for i in range(k)]
            sub = [nodes[m] for m in members]
            order = node_tree_list(sub)                      # positions within `members`
            act = np.array([orig_to_compiled[members[o]] for o in order], dtype=np.uint32)
            scenarios.append(Scenario(len(scenarios), si, k, act))
    return scenarios


def occupancy_ok(res: Dict[str, int], max_cpu: int = 100, max_mem: int = 100, max_vg: int = 100) -> bool:
    """satisfyResourceSetting (pkg/apply/apply.go:689-775): CPU, memory and, for results that carry the VG sums of a run with
    Open-Local storage (vg_requested / vg_capacity), the VG occupancy; a VG capacity of 0 skips that test (apply.go:766)."""
    if res["alloc_mcpu"] > 0:
        if int(float(res["req_mcpu"]) / float(res["alloc_mcpu"]) * 100) > max_cpu:
            return False
    if res["alloc_mem"] > 0:
        if int(float(res["req_mem"]) / float(res["alloc_mem"]) * 100) > max_mem:
            return False
    if res.get("vg_capacity"):
        if int(float(res["vg_requested"]) / float(res["vg_capacity"]) * 100) > max_vg:
            return False
    return True


def env_caps() -> Tuple[int, int]:
    """EnvMaxCPU / EnvMaxMemory (pkg/type/const.go:29-31; out-of-range values fall back to 100)."""
    def cap(name):
        v = os.environ.get(name, "")
        if not v:
            return 100
        x = int(v)
        return 100 if x > 100 or x < 0 else x
    return cap("MaxCPU"), cap("MaxMemory")


def env_vg_cap() -> int:
    """EnvMaxVG (pkg/type/const.go:31; apply.go:712-719): unset or empty gives 100, a value outside [0, 100] gives 100, and a
    value strconv.Atoi rejects is an error (ValueError)."""
    v = os.environ.get("MaxVG", "")
    if not v:
        return 100
    if not re.fullmatch(r"[+-]?[0-9]+", v):
        raise ValueError(f"failed to convert env MaxVG to int: {v!r}")
    x = int(v)
    return 100 if x > 100 or x < 0 else x


def scenario_key(sc: Scenario, res: Dict[str, int], max_cpu: int, max_mem: int, max_vg: int = 100) -> int:
    feasible = res["n_unscheduled"] == 0 and occupancy_ok(res, max_cpu, max_mem, max_vg)
    return ((sc.k << 32) | sc.sid) if feasible else INFEASIBLE_KEY


Runner = Callable[[ScenarioSet, List[Scenario]], List[Dict[str, int]]]


def gpu_runner(device: int = 0, engine=None) -> Runner:
    """Runs a shard of scenarios on one GPU through simon_scenarios_run (one thread-block cluster per scenario), or
    simon_scenarios_run_local when the superset was compiled with Open-Local storage (its results carry vg_requested /
    vg_capacity).  With `engine` (an Engine holding ss.compiled) the context, its uploaded snapshot and its pooled scenario
    buffers are reused across calls - the shape of a capacity search that tries several candidate sets on one cluster."""
    def go(eng, ss: ScenarioSet, shard: List[Scenario]):
        fn = eng.run_scenarios_local if ss.compiled.storage is not None else eng.run_scenarios
        return fn([sc.nodes for sc in shard])[0]

    def run(ss: ScenarioSet, shard: List[Scenario]) -> List[Dict[str, int]]:
        from .engine import Engine
        if not shard:
            return []
        if engine is not None:
            return go(engine, ss, shard)
        with Engine(ss.compiled, device=device) as eng:
            return go(eng, ss, shard)
    return run


def search(ss: ScenarioSet, runner: Runner, rank: int = 0, world: int = 1, all_reduce_min=None,
           max_cpu: Optional[int] = None, max_mem: Optional[int] = None, max_vg: Optional[int] = None):
    """Shard scenarios round-robin over `world` ranks, run the local shard, reduce the packed key with MIN.

    all_reduce_min: callable(int) -> int performing the collective (torch.distributed all_reduce MIN over NCCL/gloo);
    None for a single process.  max_vg applies to results with VG sums (an Open-Local superset).  Returns (best_key, local
    results keyed by scenario id)."""
    if max_cpu is None or max_mem is None:
        ec, em = env_caps()
        max_cpu = ec if max_cpu is None else max_cpu
        max_mem = em if max_mem is None else max_mem
    if max_vg is None:
        max_vg = env_vg_cap()
    shard = [sc for sc in ss.scenarios if sc.sid % world == rank]
    results = runner(ss, shard)
    local_best = INFEASIBLE_KEY
    by_sid = {}
    for sc, res in zip(shard, results):
        by_sid[sc.sid] = res
        local_best = min(local_best, scenario_key(sc, res, max_cpu, max_mem, max_vg))
    best = all_reduce_min(local_best) if all_reduce_min is not None else local_best
    return best, by_sid


def search_min_k(n_specs: int, kmax: int, method: str, evaluate: Callable[[List[Tuple[int, int]]], None],
                 ok: Callable[[int, int], bool]) -> Tuple[List[int], int]:
    """The add-node search over k in [0, kmax] for each of n_specs specs: evaluate(pairs) runs the (spec, k) pairs given (one batch per
    call), ok(spec, k) tells whether an evaluated pair is feasible.  "sweep": every pair in one batch.  Otherwise bisection, valid
    because feasibility is monotone in k for one spec: (s, 0) and (s, kmax) of every spec in one batch, then one batch per round with
    the midpoint of every spec still open.  Returns (per spec the minimal feasible k or -1, rounds)."""
    ks = range(kmax + 1)
    if method == "sweep":
        evaluate([(s, k) for s in range(n_specs) for k in ks])
        return [next((k for k in ks if ok(s, k)), -1) for s in range(n_specs)], 1
    evaluate([(s, k) for s in range(n_specs) for k in sorted({0, kmax})])
    rounds = 1
    best: List[Optional[int]] = []
    bounds: Dict[int, List[int]] = {}
    for s in range(n_specs):
        if ok(s, 0):
            best.append(0)
        elif not ok(s, kmax):
            best.append(-1)
        else:
            best.append(None)
            bounds[s] = [0, kmax]                   # invariant: lo infeasible, hi feasible
    while True:
        for s, (lo, hi) in list(bounds.items()):
            if hi - lo <= 1:
                best[s] = hi
                del bounds[s]
        if not bounds:
            break
        mids = {s: (lo + hi) // 2 for s, (lo, hi) in bounds.items()}
        evaluate(list(mids.items()))
        rounds += 1
        for s, mid in mids.items():
            bounds[s][1 if ok(s, mid) else 0] = mid
    return [int(b) for b in best], rounds


def decode_key(key: int):
    if key >= INFEASIBLE_KEY:
        return None
    return {"k": key >> 32, "scenario": key & 0xFFFFFFFF}


def torch_all_reduce_min(device: str):
    """The one collective of the capacity search: all_reduce(MIN) of an int64 over the default process group."""
    import torch
    import torch.distributed as dist

    def fn(v: int) -> int:
        t = torch.tensor([v], dtype=torch.int64, device=device)
        dist.all_reduce(t, op=dist.ReduceOp.MIN)
        return int(t.item())
    return fn
