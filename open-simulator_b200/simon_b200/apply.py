"""`simon apply -f <config>` on the engine, with the add-node loop made automatic (SURVEY 8f rank 2).

Reference flow (pkg/apply/apply.go:96-306): read the simon Config (cluster.customConfig | kubeConfig, appList[], newNode),
build ResourceTypes for the cluster and every app, then loop: Simulate(cluster + k fake nodes of the ONE newNode spec,
apps); if pods are left unscheduled the user is asked to type another k (apply.go:203-259); a run is accepted when nothing
is unscheduled and satisfyResourceSetting holds (apply.go:689-775).  There is no search in the reference.

Here the loop is a search over k carried out as batches of what-if scenarios (capacity.build_scenarios, one thread-block
cluster per scenario on the GPU):
    * "sweep": every k in 0..kmax in ONE batch - what the GPU is good at;
    * "bisect": feasibility is monotone in k for one spec (more nodes of the same kind never leave more pods
      unscheduled - tests/test_capacity.py), so log2(kmax) rounds of one scenario each find the minimum; used when kmax is
      large and the batch would not fit.
Charts (appList[].chart: true) need Helm rendering, which is outside the scheduling path: such entries are refused.

    python -m simon_b200.apply -f example/simon-config.yaml [--kmax 64] [--method sweep|bisect]
"""
from __future__ import annotations

import argparse
import json
import os
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional

import yaml

from . import capacity
from . import objects as O
from .objects import AppResource, ResourceTypes


@dataclass
class ApplyResult:
    new_node_num: int                      # minimal number of new nodes (0: the cluster already fits), -1: none up to kmax
    unscheduled_without_new_nodes: int
    scenarios_evaluated: int
    rounds: int
    per_k: Dict[int, Dict[str, int]] = field(default_factory=dict)


def load_config(path: str, base_dir: Optional[str] = None):
    """simon/v1alpha1 Config (pkg/api/v1alpha1/types.go; example/simon-config.yaml) -> (cluster, apps, new node spec or None).
    Relative paths are resolved against base_dir (the reference resolves them against the working directory)."""
    cfg = yaml.safe_load(open(path, "r", encoding="utf-8"))
    if not isinstance(cfg, dict) or cfg.get("kind") != "Config":
        raise ValueError(f"{path}: not a simon Config")
    spec = cfg.get("spec") or {}
    base = base_dir if base_dir is not None else os.getcwd()

    def rp(p):
        return p if os.path.isabs(p) else os.path.join(base, p)

    cl = spec.get("cluster") or {}
    if cl.get("kubeConfig") and not cl.get("customConfig"):
        raise NotImplementedError("cluster.kubeConfig: importing a live cluster needs an API server; use cluster.customConfig")
    if not cl.get("customConfig"):
        raise ValueError("spec.cluster.customConfig is required")
    cluster = O.create_cluster_resource_from_cluster_config(rp(cl["customConfig"]))
    apps: List[AppResource] = []
    for a in spec.get("appList") or []:
        if a.get("chart"):
            raise NotImplementedError(f"app {a.get('name')}: Helm charts are rendered outside the scheduling path; render it to YAML first")
        apps.append(AppResource(a.get("name", ""), O.get_object_from_yaml_content(O.get_yaml_content_from_directory(rp(a["path"])))))
    new_node = None
    if spec.get("newNode"):
        res = O.get_object_from_yaml_content(O.get_yaml_content_from_directory(rp(spec["newNode"])))
        O.match_and_set_local_storage_annotation_on_node(res.Nodes, rp(spec["newNode"]))
        if not res.Nodes:
            raise ValueError("spec.newNode holds no Node object")
        new_node = res.Nodes[0]                 # "only support temporarily adding a type of node at present" (apply.go:166-167)
    return cluster, apps, new_node


def auto_add_nodes(cluster: ResourceTypes, apps: List[AppResource], new_node, runner_factory: Callable, kmax: int = 64,
                   method: str = "sweep", max_cpu: Optional[int] = None, max_mem: Optional[int] = None,
                   open_local: bool = False, local_devices: bool = False, max_vg: Optional[int] = None) -> ApplyResult:
    """Minimal k in [0, kmax] such that cluster + k copies of new_node places every pod within the occupancy caps.

    runner_factory(ss) -> capacity.Runner for that scenario set (GPU: capacity.gpu_runner(device, engine=Engine(ss.compiled))).
    open_local / local_devices: place pods that request Open-Local storage (capacity.build_scenarios); per_k then also holds
    vg_requested / vg_capacity and the MaxVG cap (max_vg, default: the environment) applies.  Bisection stays valid: once every
    pod is placed, ΣVG requested is fixed, and ΣVG capacity can only grow with k."""
    if max_cpu is None or max_mem is None:
        ec, em = capacity.env_caps()
        max_cpu = ec if max_cpu is None else max_cpu
        max_mem = em if max_mem is None else max_mem
    if max_vg is None:
        max_vg = capacity.env_vg_cap() if open_local else 100
    specs = [new_node] if new_node is not None else []
    if not specs:
        kmax = 0
    ks = list(range(0, kmax + 1))
    ss = capacity.build_scenarios(cluster, apps, specs or [cluster.Nodes[0]], ks if specs else [0],
                                  open_local=open_local, local_devices=local_devices)
    runner = runner_factory(ss)
    by_k = {sc.k: sc for sc in ss.scenarios}
    per_k: Dict[int, Dict[str, int]] = {}
    keys = ("n_unscheduled", "n_scheduled", "req_mcpu", "alloc_mcpu", "req_mem", "alloc_mem")
    if open_local:
        keys += ("vg_requested", "vg_capacity")

    def evaluate(pairs):
        todo = [by_k[k] for _s, k in pairs if k not in per_k]
        for sc, res in zip(todo, runner(ss, todo)):
            per_k[sc.k] = {q: int(res[q]) for q in keys}

    def ok(_s, k):
        r = per_k[k]
        return r["n_unscheduled"] == 0 and capacity.occupancy_ok(r, max_cpu, max_mem, max_vg)

    (best,), rounds = capacity.search_min_k(1, kmax, method if specs else "sweep", evaluate, ok)
    return ApplyResult(best, per_k[0]["n_unscheduled"] if 0 in per_k else -1, len(per_k), rounds, per_k)


def main(argv=None):
    ap = argparse.ArgumentParser(description="simon apply on the GPU engine, add-node search automatic")
    ap.add_argument("-f", "--simon-config", required=True)
    ap.add_argument("--kmax", type=int, default=64)
    ap.add_argument("--method", default="sweep", choices=["sweep", "bisect"])
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--open-local", action="store_true",
                    help="place pods that request Open-Local storage (LVM volumes); the MaxVG cap applies")
    ap.add_argument("--open-local-devices", action="store_true",
                    help="also their exclusive SSD / HDD device volumes (implies --open-local)")
    a = ap.parse_args(argv)
    cluster, apps, new_node = load_config(a.simon_config)
    from .engine import Engine            # no CPU fallback: raises without the library / a CUDA device

    engines = []

    def factory(ss):
        eng = Engine(ss.compiled, device=a.device)
        engines.append(eng)
        return capacity.gpu_runner(a.device, engine=eng)

    res = auto_add_nodes(cluster, apps, new_node, factory, kmax=a.kmax, method=a.method,
                         open_local=a.open_local or a.open_local_devices, local_devices=a.open_local_devices)
    for e in engines:
        e.close()
    print(json.dumps({"new_node_num": res.new_node_num, "unscheduled_without_new_nodes": res.unscheduled_without_new_nodes,
                      "scenarios_evaluated": res.scenarios_evaluated, "rounds": res.rounds}))
    return 0 if res.new_node_num >= 0 else 1


if __name__ == "__main__":
    raise SystemExit(main())
