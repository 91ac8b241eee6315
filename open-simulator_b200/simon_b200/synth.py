"""Seeded synthetic clusters (SURVEY.md §8d): Kubernetes objects as dicts, so that synthetic inputs travel the
same path as YAML inputs (workload expansion -> snapshot compiler -> engine).

PRNG = SplitMix64, seed 0x51514D4F4E00 + config number.
  C2: N nodes (8 shapes), 16 zones, hostname label; Deployments x replicas with cpu/mem requests,
      5 % request nothing; one Service per workload (activates the system default spreading).
  C3: + regions, taints, 32 label keys x <=8 values, tolerations, nodeSelector, required node affinity,
      required hostname anti-affinity, preferred zone affinity, explicit topologySpreadConstraints,
      10 % of nodes pre-filled with ~20 running pods.
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import numpy as np

from .objects import AppResource, ResourceTypes

MASK = (1 << 64) - 1
SEED_BASE = 0x51514D4F4E00


class SplitMix64:
    def __init__(self, seed: int):
        self.s = seed & MASK

    def next(self) -> int:
        self.s = (self.s + 0x9E3779B97F4A7C15) & MASK
        z = self.s
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & MASK
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & MASK
        return z ^ (z >> 31)

    def below(self, n: int) -> int:
        return self.next() % n

    def chance(self, pct: int) -> bool:
        return self.below(100) < pct

    def pick(self, seq):
        return seq[self.below(len(seq))]


CPU_SHAPES = [8, 16, 32, 64, 96, 128, 192, 256]


def _node(name: str, cores: int, zone: str, region: str, eph_gi: int, labels=None, taints=None, pods=110) -> dict:
    lab = {"kubernetes.io/hostname": name, "topology.kubernetes.io/zone": zone}
    if region:
        lab["topology.kubernetes.io/region"] = region
    if labels:
        lab.update(labels)
    n = {"apiVersion": "v1", "kind": "Node", "metadata": {"name": name, "labels": lab},
         "spec": {},
         "status": {"allocatable": {"cpu": str(cores), "memory": f"{4 * cores}Gi", "ephemeral-storage": f"{eph_gi}Gi",
                                    "pods": str(pods)},
                    "capacity": {"cpu": str(cores), "memory": f"{4 * cores}Gi", "ephemeral-storage": f"{eph_gi}Gi",
                                 "pods": str(pods)}}}
    if taints:
        n["spec"]["taints"] = taints
    return n


def _log_uniform(rng: SplitMix64, lo: int, hi: int, step: int) -> int:
    """log-uniform integer in [lo, hi], rounded to a multiple of step."""
    import math
    u = rng.below(1 << 20) / float(1 << 20)
    v = math.exp(math.log(lo) + u * (math.log(hi) - math.log(lo)))
    q = max(step, int(round(v / step)) * step)
    return min(q, hi)


def _deployment(name: str, ns: str, replicas: int, labels: Dict[str, str], cpu_m: int, mem_mi: int, spec_extra=None) -> dict:
    c = {"name": "c", "image": f"registry.local/{name}:v1"}
    if cpu_m or mem_mi:
        req = {}
        if cpu_m:
            req["cpu"] = f"{cpu_m}m"
        if mem_mi:
            req["memory"] = f"{mem_mi}Mi"
        c["resources"] = {"requests": req}
    spec = {"containers": [c]}
    if spec_extra:
        spec.update(spec_extra)
    return {"apiVersion": "apps/v1", "kind": "Deployment", "metadata": {"name": name, "namespace": ns},
            "spec": {"replicas": replicas, "selector": {"matchLabels": dict(labels)},
                     "template": {"metadata": {"labels": dict(labels)}, "spec": spec}}}


def _service(name: str, ns: str, sel: Dict[str, str]) -> dict:
    return {"apiVersion": "v1", "kind": "Service", "metadata": {"name": name, "namespace": ns},
            "spec": {"selector": dict(sel), "ports": [{"port": 80}]}}


def make_c2(n_nodes: int = 1000, n_workloads: int = 100, replicas: int = 100, seed_no: int = 2,
            n_apps: int = 1) -> Tuple[ResourceTypes, List[AppResource]]:
    rng = SplitMix64(SEED_BASE + seed_no)
    cluster = ResourceTypes()
    for i in range(n_nodes):
        cores = rng.pick(CPU_SHAPES)
        eph = rng.pick([100, 200, 500, 1000, 2048])
        cluster.Nodes.append(_node(f"node-{i:05d}", cores, f"zone-{i % 16:02d}", "", eph))
    apps = [AppResource(f"app-{a}", ResourceTypes()) for a in range(n_apps)]
    for w in range(n_workloads):
        name = f"wl-{w:04d}"
        ns = "default"
        labels = {"app": name}
        if rng.chance(5):
            cpu, mem = 0, 0
        else:
            cpu = _log_uniform(rng, 100, 8000, 50)
            mem = _log_uniform(rng, 128, 32768, 64)
        apps[w % n_apps].Resource.Deployments.append(_deployment(name, ns, replicas, labels, cpu, mem))
        cluster.Services.append(_service(name, ns, labels))
    return cluster, apps


def make_c3(n_nodes: int = 10000, n_workloads: int = 1000, replicas: int = 100, seed_no: int = 3,
            n_apps: int = 10, prefill_pct: int = 10, prefill_pods: int = 20, gpu_pct: int = 0) -> Tuple[ResourceTypes, List[AppResource]]:
    """gpu_pct > 0: GPU-share devices on ~gpu_pct % of the nodes, GPU-share requests on ~15 % of the workloads and a DoNotSchedule
    zone spread on another ~10 % (placed by the scheduler, so they hold device memory).  These draws come from a second random
    stream: with gpu_pct = 0 the cluster is the same as without the keyword."""
    rng = SplitMix64(SEED_BASE + seed_no)
    grng = SplitMix64(SEED_BASE + 0x3000 + seed_no)
    cluster = ResourceTypes()
    hard_taints = [{"key": f"dedicated-{i}", "value": f"team-{i}", "effect": "NoSchedule"} for i in range(8)]
    soft_taints = [{"key": f"degraded-{i}", "value": "true", "effect": "PreferNoSchedule"} for i in range(4)]
    label_keys = [f"feature-{k:02d}" for k in range(32)]
    for i in range(n_nodes):
        cores = rng.pick(CPU_SHAPES)
        eph = rng.pick([100, 200, 500, 1000, 2048])
        region = f"region-{i % 3}"
        zone = f"{region}-zone-{(i // 3) % 16:02d}"
        labels = {}
        for k in label_keys:
            if rng.chance(50):
                labels[k] = f"v{rng.below(8)}"
        taints = []
        if rng.chance(10):
            taints.append(dict(rng.pick(hard_taints)))
        if rng.chance(5):
            taints.append(dict(rng.pick(soft_taints)))
        cluster.Nodes.append(_node(f"node-{i:05d}", cores, zone, region, eph, labels, taints or None))
        if gpu_pct and grng.chance(gpu_pct):
            cnt = grng.pick([1, 2, 4, 8])
            mem = f"{cnt * grng.pick([16, 32, 80])}Gi"
            for sect in ("allocatable", "capacity"):
                cluster.Nodes[-1]["status"][sect]["alibabacloud.com/gpu-count"] = str(cnt)
                cluster.Nodes[-1]["status"][sect]["alibabacloud.com/gpu-mem"] = mem
    # running pods on ~prefill_pct % of the nodes (pre-bound: spec.nodeName set)
    for i in range(n_nodes):
        if not rng.chance(prefill_pct):
            continue
        for j in range(prefill_pods):
            cluster.Pods.append({"apiVersion": "v1", "kind": "Pod",
                                 "metadata": {"name": f"running-{i:05d}-{j:02d}", "namespace": "kube-system",
                                              "labels": {"app": f"sys-{j % 4}"}},
                                 "spec": {"nodeName": f"node-{i:05d}",
                                          "containers": [{"name": "c", "image": "registry.local/sys:v1",
                                                          "resources": {"requests": {"cpu": "100m", "memory": "128Mi"}}}]}})
    apps = [AppResource(f"app-{a}", ResourceTypes()) for a in range(n_apps)]
    names = [f"wl-{w:04d}" for w in range(n_workloads)]
    for w in range(n_workloads):
        name = names[w]
        ns = f"ns-{w % 8}"
        labels = {"app": name, "tier": rng.pick(["web", "db", "cache", "batch"])}
        if rng.chance(5):
            cpu, mem = 0, 0
        else:
            cpu = _log_uniform(rng, 100, 8000, 50)
            mem = _log_uniform(rng, 128, 32768, 64)
        extra: dict = {}
        aff: dict = {}
        if rng.chance(30):
            t = rng.pick(hard_taints)
            tols = [{"key": t["key"], "operator": "Equal", "value": t["value"], "effect": "NoSchedule"}]
            if rng.chance(50):
                s = rng.pick(soft_taints)
                tols.append({"key": s["key"], "operator": "Exists"})
            extra["tolerations"] = tols
        if rng.chance(20):
            sel = {}
            for _ in range(1 + rng.below(2)):
                sel[rng.pick(label_keys)] = f"v{rng.below(8)}"
            extra["nodeSelector"] = sel
        if rng.chance(10):
            exprs = []
            kind = rng.below(3)
            k = rng.pick(label_keys)
            if kind == 0:
                exprs.append({"key": k, "operator": "In", "values": [f"v{rng.below(8)}", f"v{rng.below(8)}", f"v{rng.below(8)}"]})
            elif kind == 1:
                exprs.append({"key": k, "operator": "NotIn", "values": [f"v{rng.below(8)}"]})
            else:
                exprs.append({"key": k, "operator": "Exists"})
            aff["nodeAffinity"] = {"requiredDuringSchedulingIgnoredDuringExecution":
                                   {"nodeSelectorTerms": [{"matchExpressions": exprs}]}}
            if rng.chance(50):
                aff["nodeAffinity"]["preferredDuringSchedulingIgnoredDuringExecution"] = [
                    {"weight": 1 + rng.below(100),
                     "preference": {"matchExpressions": [{"key": rng.pick(label_keys), "operator": "In",
                                                          "values": [f"v{rng.below(8)}"]}]}}]
        if rng.chance(20):
            aff["podAntiAffinity"] = {"requiredDuringSchedulingIgnoredDuringExecution": [
                {"labelSelector": {"matchLabels": {"app": name}}, "topologyKey": "kubernetes.io/hostname"}]}
        if rng.chance(10):
            other = names[rng.below(n_workloads)]
            aff.setdefault("podAffinity", {})["preferredDuringSchedulingIgnoredDuringExecution"] = [
                {"weight": 1 + rng.below(100),
                 "podAffinityTerm": {"labelSelector": {"matchLabels": {"app": other}},
                                     "namespaces": [f"ns-{names.index(other) % 8}"],
                                     "topologyKey": "topology.kubernetes.io/zone"}}]
        if aff:
            extra["affinity"] = aff
        if rng.chance(10):
            extra["topologySpreadConstraints"] = [
                {"maxSkew": 1 + rng.below(5), "topologyKey": "topology.kubernetes.io/zone",
                 "whenUnsatisfiable": rng.pick(["DoNotSchedule", "ScheduleAnyway"]),
                 "labelSelector": {"matchLabels": {"app": name}}}]
        if gpu_pct and "topologySpreadConstraints" not in extra and grng.chance(10):
            extra["topologySpreadConstraints"] = [
                {"maxSkew": 1 + grng.below(3), "topologyKey": "topology.kubernetes.io/zone", "whenUnsatisfiable": "DoNotSchedule",
                 "labelSelector": {"matchLabels": {"app": name}}}]
        dep = _deployment(name, ns, replicas, labels, cpu, mem, extra)
        if gpu_pct and grng.chance(15):
            dep["spec"]["template"]["metadata"]["annotations"] = {"alibabacloud.com/gpu-mem": f"{grng.pick([4, 8, 16, 24])}Gi",
                                                                  "alibabacloud.com/gpu-count": str(grng.pick([1, 1, 1, 2]))}
        apps[w % n_apps].Resource.Deployments.append(dep)
        cluster.Services.append(_service(name, ns, {"app": name}))
    return cluster, apps


def make_c4(n_nodes: int = 2000, n_workloads: int = 50, replicas: int = 100, fill_pct: int = 85, seed_no: int = 4):
    """C4 (SURVEY.md §8d): base cluster ~fill_pct % full + pending pods that do not all fit; 8 candidate node specs.
    Returns (cluster, apps, specs)."""
    rng = SplitMix64(SEED_BASE + seed_no)
    cluster = ResourceTypes()
    for i in range(n_nodes):
        cores = rng.pick(CPU_SHAPES)
        eph = rng.pick([100, 200, 500, 1000, 2048])
        cluster.Nodes.append(_node(f"node-{i:05d}", cores, f"zone-{i % 16:02d}", "", eph))
        # one running "filler" pod per node occupying ~fill_pct % of cpu and memory
        cpu_m = cores * 10 * fill_pct
        mem_mi = cores * 4 * 1024 * fill_pct // 100
        cluster.Pods.append({"apiVersion": "v1", "kind": "Pod",
                             "metadata": {"name": f"filler-{i:05d}", "namespace": "kube-system", "labels": {"app": "filler"}},
                             "spec": {"nodeName": f"node-{i:05d}",
                                      "containers": [{"name": "c", "image": "registry.local/filler:v1",
                                                      "resources": {"requests": {"cpu": f"{cpu_m}m", "memory": f"{mem_mi}Mi"}}}]}})
    app = AppResource("pending", ResourceTypes())
    for w in range(n_workloads):
        name = f"pend-{w:03d}"
        cpu = _log_uniform(rng, 500, 8000, 50)
        mem = _log_uniform(rng, 512, 32768, 64)
        extra = {}
        if rng.chance(20):
            extra["affinity"] = {"podAntiAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": [
                {"labelSelector": {"matchLabels": {"app": name}}, "topologyKey": "kubernetes.io/hostname"}]}}
        app.Resource.Deployments.append(_deployment(name, "default", replicas, {"app": name}, cpu, mem, extra))
        cluster.Services.append(_service(name, "default", {"app": name}))
    specs = []
    for si, cores in enumerate(CPU_SHAPES):
        specs.append(_node(f"spec-{si}", cores, f"zone-{si % 16:02d}", "", 500))
    return cluster, [app], specs


def make_open_local(n_nodes: int = 10000, n_workloads: int = 200, replicas: int = 250, seed_no: int = 6
                    ) -> Tuple[ResourceTypes, List[AppResource]]:
    """Open-Local storage: ~60 % of the nodes carry the simon/node-local-storage annotation with 1-4 VGs and 0-8 SSD / HDD
    devices (~5 % of them allocated); the Deployments request no volume, LVM volumes only, devices only, or both, a quarter
    each.  The two device StorageClasses are in the cluster."""
    import json
    from .objects import ANNO_NODE_LOCAL_STORAGE, ANNO_POD_LOCAL_STORAGE
    gi = 1 << 30
    rng = SplitMix64(SEED_BASE + seed_no)
    cluster = ResourceTypes()
    for m in ("ssd", "hdd"):
        cluster.StorageClasss.append({"apiVersion": "storage.k8s.io/v1", "kind": "StorageClass",
                                      "metadata": {"name": f"open-local-device-{m}"}, "parameters": {"mediaType": m}})
    for i in range(n_nodes):
        n = _node(f"node-{i:05d}", rng.pick(CPU_SHAPES), f"zone-{i % 16:02d}", "", 1000)
        if rng.chance(60):
            vgs = [{"name": f"pool{v}", "capacity": str(rng.pick([100, 200, 500, 1000]) * gi),
                    "requested": str(rng.below(5) * 10 * gi)} for v in range(1 + rng.below(4))]
            devs = [{"name": f"/dev/vd{k}", "device": f"/dev/vd{k}", "capacity": str(rng.pick([100, 200, 400, 800, 1600]) * gi),
                     "mediaType": rng.pick(["ssd", "hdd"]), "isAllocated": "true" if rng.chance(5) else "false"}
                    for k in range(rng.below(9))]
            n["metadata"]["annotations"] = {ANNO_NODE_LOCAL_STORAGE: json.dumps({"vgs": vgs, "devices": devs})}
        cluster.Nodes.append(n)
    app = AppResource("open-local", ResourceTypes())
    for w in range(n_workloads):
        name = f"ol-{w:04d}"
        d = _deployment(name, "default", replicas, {"app": name}, _log_uniform(rng, 100, 2000, 50), _log_uniform(rng, 128, 4096, 64))
        kind = w % 4          # 0: no volume, 1: LVM, 2: devices, 3: both
        vols = []
        if kind in (1, 3):
            vols += [{"size": str(_log_uniform(rng, 5, 100, 5) * gi), "kind": "LVM", "scName": "open-local-lvm"}
                     for _ in range(1 + rng.below(3))]
        if kind in (2, 3):
            for _ in range(1 + rng.below(2)):
                m = rng.pick(["SSD", "HDD"])
                vols.append({"size": str(rng.pick([50, 100, 200, 400, 1000]) * gi), "kind": m,
                             "scName": f"open-local-device-{m.lower()}"})
        if vols:
            d["spec"]["template"]["metadata"]["annotations"] = {ANNO_POD_LOCAL_STORAGE: json.dumps({"volumes": vols})}
        app.Resource.Deployments.append(d)
    return cluster, [app]


def make_mix(seed_no: int = 100, n_nodes: int = 40, n_workloads: int = 30, max_replicas: int = 6, with_images: bool = False):
    """Small clusters that exercise EVERY predicate / score input the path knows, in random combinations: unschedulable
    nodes, NoSchedule / NoExecute / PreferNoSchedule taints and all toleration shapes, nodeSelector, required and
    preferred node affinity with In / NotIn / Exists / DoesNotExist / Gt / Lt and matchFields, host ports (with and
    without hostIP), extended (scalar) resources, ephemeral storage, init containers and overhead, required and
    preferred pod (anti-)affinity incl. self-affinity, hard and soft topology spread over hostname / zone / region with
    nodes that lack the zone label, GPU-share pods and nodes, pre-bound pods, DaemonSets, StatefulSets, Jobs and
    bare Pods.  Used by the parity tests (C oracle vs object-level restatement vs GPU)."""
    rng = SplitMix64(SEED_BASE + 0x1000 + seed_no)
    cluster = ResourceTypes()
    hard_taints = [{"key": f"dedicated-{i}", "value": f"team-{i}", "effect": "NoSchedule"} for i in range(3)]
    hard_taints.append({"key": "maintenance", "value": "true", "effect": "NoExecute"})
    soft_taints = [{"key": f"degraded-{i}", "value": "true", "effect": "PreferNoSchedule"} for i in range(3)]
    label_keys = [f"feature-{k}" for k in range(6)]
    node_names = []
    for i in range(n_nodes):
        cores = rng.pick([4, 8, 16, 32])
        region = f"region-{i % 2}"
        zone = f"{region}-zone-{(i // 2) % 4}"
        labels = {"rank": str(rng.below(100))}
        for k in label_keys:
            if rng.chance(50):
                labels[k] = f"v{rng.below(3)}"
        taints = []
        if rng.chance(15):
            taints.append(dict(rng.pick(hard_taints)))
        if rng.chance(15):
            taints.append(dict(rng.pick(soft_taints)))
        if rng.chance(5):
            t2 = dict(rng.pick(soft_taints))
            if all((t["key"], t["effect"]) != (t2["key"], t2["effect"]) for t in taints):   # the API server rejects duplicate (key, effect)
                taints.append(t2)
        name = f"node-{i:03d}"
        node_names.append(name)
        n = _node(name, cores, zone, region, rng.pick([50, 100, 200]), labels, taints or None, pods=rng.pick([8, 16, 110]))
        if rng.chance(10):
            del n["metadata"]["labels"]["topology.kubernetes.io/zone"]          # spreading / affinity over a missing key
        if rng.chance(5):
            n["spec"]["unschedulable"] = True
        if rng.chance(30):
            w = str(rng.pick([2, 4, 8]))
            n["status"]["allocatable"]["example.com/widget"] = w
            n["status"]["capacity"]["example.com/widget"] = w
        if rng.chance(25):
            cnt = rng.pick([1, 2, 4])
            mem = f"{cnt * rng.pick([8, 16])}Gi"
            for sect in ("allocatable", "capacity"):
                n["status"][sect]["alibabacloud.com/gpu-count"] = str(cnt)
                n["status"][sect]["alibabacloud.com/gpu-mem"] = mem
        cluster.Nodes.append(n)
    if with_images:
        # node images for ImageLocality: a few workload images of different sizes, each on a random subset of the nodes
        irng = SplitMix64(SEED_BASE + 0x2000 + seed_no)
        pool = [(f"registry.local/wl-{w:03d}:v1", (50 + irng.below(900)) * 1024 * 1024) for w in range(min(8, n_workloads))]
        for n in cluster.Nodes:
            imgs = [{"names": [nm, nm.replace("registry.local/", "mirror.local/")], "sizeBytes": sz} for (nm, sz) in pool if irng.chance(35)]
            if imgs:
                n["status"]["images"] = imgs
    # pre-bound pods (some carry labels that later selectors match, some hold host ports)
    for i in range(n_nodes):
        if not rng.chance(30):
            continue
        for j in range(1 + rng.below(3)):
            c = {"name": "c", "image": "registry.local/sys:v1",
                 "resources": {"requests": {"cpu": f"{rng.pick([100, 250, 500])}m", "memory": f"{rng.pick([128, 256, 1024])}Mi"}}}
            if rng.chance(20):
                c["ports"] = [{"containerPort": 8080, "hostPort": rng.pick([8080, 8081]), "protocol": "TCP"}]
            cluster.Pods.append({"apiVersion": "v1", "kind": "Pod",
                                 "metadata": {"name": f"running-{i:03d}-{j}", "namespace": rng.pick(["default", "kube-system"]),
                                              "labels": {"app": f"wl-{rng.below(n_workloads):03d}" if rng.chance(50) else f"sys-{j}"}},
                                 "spec": {"nodeName": node_names[i], "containers": [c]}})
    app = AppResource("mix", ResourceTypes())
    names = [f"wl-{w:03d}" for w in range(n_workloads)]
    zone_key, host_key, region_key = "topology.kubernetes.io/zone", "kubernetes.io/hostname", "topology.kubernetes.io/region"

    def pod_term(target: str, key: str, ns=None):
        t = {"labelSelector": {"matchLabels": {"app": target}}, "topologyKey": key}
        if ns is not None:
            t["namespaces"] = ns
        return t

    for w in range(n_workloads):
        name = names[w]
        ns = rng.pick(["default", "team-a"])
        labels = {"app": name, "tier": rng.pick(["web", "db"])}
        req = {}
        if not rng.chance(10):
            req["cpu"] = f"{_log_uniform(rng, 100, 4000, 50)}m"
            req["memory"] = f"{_log_uniform(rng, 128, 8192, 64)}Mi"
        if rng.chance(20):
            req["ephemeral-storage"] = f"{rng.pick([1, 5, 20])}Gi"
        if rng.chance(15):
            req["example.com/widget"] = str(1 + rng.below(2))
        cont = {"name": "c", "image": f"registry.local/{name}:v1"}
        if req:
            cont["resources"] = {"requests": req}
        if rng.chance(12):
            port = {"containerPort": 80, "hostPort": rng.pick([8080, 8081, 9090]), "protocol": rng.pick(["TCP", "UDP"])}
            if rng.chance(30):
                port["hostIP"] = rng.pick(["10.0.0.1", "0.0.0.0"])
            cont["ports"] = [port]
        spec: dict = {"containers": [cont]}
        if rng.chance(10):
            spec["initContainers"] = [{"name": "init", "image": "registry.local/init:v1",
                                       "resources": {"requests": {"cpu": f"{rng.pick([100, 2000, 6000])}m", "memory": "256Mi"}}}]
        if rng.chance(5):
            spec["overhead"] = {"cpu": "100m", "memory": "64Mi"}
        tols = []
        if rng.chance(30):
            t = rng.pick(hard_taints)
            tols.append({"key": t["key"], "operator": "Equal", "value": t["value"], "effect": t["effect"]})
        if rng.chance(15):
            tols.append({"key": rng.pick(soft_taints)["key"], "operator": "Exists"})
        if rng.chance(5):
            tols.append({"operator": "Exists"})                                   # tolerates everything
        if rng.chance(5):
            tols.append({"key": "node.kubernetes.io/unschedulable", "operator": "Exists", "effect": "NoSchedule"})
        if tols:
            spec["tolerations"] = tols
        if rng.chance(15):
            spec["nodeSelector"] = {rng.pick(label_keys): f"v{rng.below(3)}"}
        aff: dict = {}
        if rng.chance(25):
            terms = []
            for _ in range(1 + rng.below(2)):
                exprs = []
                for _ in range(1 + rng.below(2)):
                    kind = rng.below(6)
                    k = rng.pick(label_keys)
                    if kind == 0:
                        exprs.append({"key": k, "operator": "In", "values": [f"v{rng.below(3)}", f"v{rng.below(3)}"]})
                    elif kind == 1:
                        exprs.append({"key": k, "operator": "NotIn", "values": [f"v{rng.below(3)}"]})
                    elif kind == 2:
                        exprs.append({"key": k, "operator": "Exists"})
                    elif kind == 3:
                        exprs.append({"key": k, "operator": "DoesNotExist"})
                    elif kind == 4:
                        exprs.append({"key": "rank", "operator": "Gt", "values": [str(rng.below(60))]})
                    else:
                        exprs.append({"key": "rank", "operator": "Lt", "values": [str(40 + rng.below(60))]})
                term = {"matchExpressions": exprs}
                if rng.chance(10):
                    term = {"matchFields": [{"key": "metadata.name", "operator": rng.pick(["In", "NotIn"]), "values": [rng.pick(node_names)]}]}
                terms.append(term)
            na = {"requiredDuringSchedulingIgnoredDuringExecution": {"nodeSelectorTerms": terms}}
            aff["nodeAffinity"] = na
        if rng.chance(20):
            prefs = []
            for _ in range(1 + rng.below(2)):
                prefs.append({"weight": 1 + rng.below(100),
                              "preference": {"matchExpressions": [{"key": rng.pick(label_keys), "operator": rng.pick(["In", "Exists"]),
                                                                   "values": [f"v{rng.below(3)}"]}]}})
            for pr in prefs:
                if pr["preference"]["matchExpressions"][0]["operator"] == "Exists":
                    del pr["preference"]["matchExpressions"][0]["values"]
            aff.setdefault("nodeAffinity", {})["preferredDuringSchedulingIgnoredDuringExecution"] = prefs
        if rng.chance(12):
            target = name if rng.chance(40) else names[rng.below(n_workloads)]
            aff.setdefault("podAffinity", {})["requiredDuringSchedulingIgnoredDuringExecution"] = [
                pod_term(target, rng.pick([zone_key, host_key, region_key]), ns=["default", "team-a"] if rng.chance(50) else None)]
        if rng.chance(20):
            aff.setdefault("podAntiAffinity", {})["requiredDuringSchedulingIgnoredDuringExecution"] = [
                pod_term(name if rng.chance(70) else names[rng.below(n_workloads)], rng.pick([host_key, host_key, zone_key]))]
        if rng.chance(15):
            aff.setdefault("podAffinity", {})["preferredDuringSchedulingIgnoredDuringExecution"] = [
                {"weight": 1 + rng.below(100), "podAffinityTerm": pod_term(names[rng.below(n_workloads)], rng.pick([zone_key, host_key]),
                                                                           ns=["default", "team-a"])}]
        if rng.chance(15):
            aff.setdefault("podAntiAffinity", {})["preferredDuringSchedulingIgnoredDuringExecution"] = [
                {"weight": 1 + rng.below(100), "podAffinityTerm": pod_term(name, rng.pick([zone_key, host_key]))}]
        if aff:
            spec["affinity"] = aff
        if rng.chance(25):
            cons = []
            for key in ([host_key, zone_key] if rng.chance(40) else [rng.pick([host_key, zone_key, region_key])]):
                cons.append({"maxSkew": 1 + rng.below(3), "topologyKey": key,
                             "whenUnsatisfiable": rng.pick(["DoNotSchedule", "ScheduleAnyway"]),
                             "labelSelector": {"matchLabels": {"app": name}}})
            spec["topologySpreadConstraints"] = cons
        tmeta = {"labels": dict(labels)}
        if rng.chance(12):
            tmeta["annotations"] = {"alibabacloud.com/gpu-mem": f"{rng.pick([2, 4, 8])}Gi", "alibabacloud.com/gpu-count": str(rng.pick([1, 1, 2]))}
        replicas = 1 + rng.below(max_replicas)
        kind = rng.below(10)
        if kind < 6:
            app.Resource.Deployments.append({"apiVersion": "apps/v1", "kind": "Deployment", "metadata": {"name": name, "namespace": ns},
                                             "spec": {"replicas": replicas, "selector": {"matchLabels": {"app": name}},
                                                      "template": {"metadata": tmeta, "spec": spec}}})
        elif kind < 8:
            app.Resource.StatefulSets.append({"apiVersion": "apps/v1", "kind": "StatefulSet", "metadata": {"name": name, "namespace": ns},
                                              "spec": {"replicas": replicas, "serviceName": name, "selector": {"matchLabels": {"app": name}},
                                                       "template": {"metadata": tmeta, "spec": spec}}})
        elif kind == 8:
            app.Resource.Jobs.append({"apiVersion": "batch/v1", "kind": "Job", "metadata": {"name": name, "namespace": ns},
                                      "spec": {"completions": replicas, "template": {"metadata": tmeta, "spec": dict(spec, restartPolicy="Never")}}})
        else:
            app.Resource.Pods.append({"apiVersion": "v1", "kind": "Pod", "metadata": dict(tmeta, name=name, namespace=ns), "spec": spec})
        if rng.chance(70):
            cluster.Services.append(_service(name, ns, {"app": name}))
    # one DaemonSet in the cluster and one in the app
    ds_spec = {"containers": [{"name": "agent", "image": "registry.local/agent:v1",
                               "resources": {"requests": {"cpu": "50m", "memory": "64Mi"}}}],
               "tolerations": [{"operator": "Exists"}]}
    cluster.DaemonSets.append({"apiVersion": "apps/v1", "kind": "DaemonSet", "metadata": {"name": "node-agent", "namespace": "kube-system"},
                               "spec": {"selector": {"matchLabels": {"app": "node-agent"}},
                                        "template": {"metadata": {"labels": {"app": "node-agent"}}, "spec": ds_spec}}})
    app.Resource.DaemonSets.append({"apiVersion": "apps/v1", "kind": "DaemonSet", "metadata": {"name": "log-shipper", "namespace": "default"},
                                    "spec": {"selector": {"matchLabels": {"app": "log-shipper"}},
                                             "template": {"metadata": {"labels": {"app": "log-shipper"}},
                                                          "spec": {"containers": [{"name": "ship", "image": "registry.local/ship:v1",
                                                                                   "resources": {"requests": {"cpu": "100m", "memory": "128Mi"}}}],
                                                                   "nodeSelector": {label_keys[0]: "v0"}}}}})
    return cluster, [app]


SAME_KEY_SELECTORS = [{"matchLabels": {"a": "x"}}, {"matchLabels": {"b": "y"}}, {"matchLabels": {"a": "x", "b": "y"}},
                      {"matchExpressions": [{"key": "a", "operator": "In", "values": ["x", "y"]}]},
                      {"matchExpressions": [{"key": "b", "operator": "Exists"}]}]


def make_same_key(seed_no: int = 1, n_nodes: int = 24, n_workloads: int = 14, max_replicas: int = 6):
    """Clusters whose workloads carry 2-4 PodTopologySpread constraints on ONE topology key (hostname, zone or a custom rack
    key): all DoNotSchedule, all ScheduleAnyway, or both kinds on the key.  The selectors are disjoint, overlapping (a pod labelled
    a=x, b=y matches two or three of them) or identical with another maxSkew.  The reference sums the counts of such constraints per
    topology pair.  Around them: nodes without the zone or rack label, a nodeSelector that restricts eligibility, a constraint on a
    second key, pre-bound pods labelled for the selectors, bare pods, and a DaemonSet with two zone constraints."""
    rng = SplitMix64(SEED_BASE + 0x3000 + seed_no)
    cluster = ResourceTypes()
    zone_key, host_key, rack_key = "topology.kubernetes.io/zone", "kubernetes.io/hostname", "example.com/rack"
    node_names = []
    for i in range(n_nodes):
        name = f"node-{i:03d}"
        node_names.append(name)
        labels = {"pool": rng.pick(["a", "b"])}
        if not rng.chance(15):
            labels[rack_key] = f"rack-{rng.below(4)}"
        n = _node(name, 64 if i % 7 == 3 else rng.pick([4, 8, 16]), f"zone-{i % 3}", "", 100, labels, pods=rng.pick([8, 16, 110]))
        if rng.chance(10):
            del n["metadata"]["labels"][zone_key]
        cluster.Nodes.append(n)

    def labelled():
        return {"a": rng.pick(["x", "y"]), "b": rng.pick(["y", "z"])}

    for i in range(n_nodes):
        if rng.chance(25):
            cluster.Pods.append({"apiVersion": "v1", "kind": "Pod",
                                 "metadata": {"name": f"running-{i:03d}", "namespace": "default", "labels": labelled()},
                                 "spec": {"nodeName": node_names[i],
                                          "containers": [{"name": "c", "image": "registry.local/sys:v1",
                                                          "resources": {"requests": {"cpu": "250m", "memory": "256Mi"}}}]}})
    app = AppResource("same-key", ResourceTypes())
    for w in range(n_workloads):
        name = f"wl-{w:03d}"
        key = rng.pick([host_key, zone_key, zone_key, rack_key])
        mode = rng.below(3)          # 0: DoNotSchedule, 1: ScheduleAnyway, 2: both kinds on the key
        cons = []
        for j in range(2 + rng.below(3)):
            when = ("DoNotSchedule", "ScheduleAnyway")[j % 2] if mode == 2 else ("DoNotSchedule", "ScheduleAnyway")[mode]
            same = [x for x in cons if x["whenUnsatisfiable"] == when]
            sel = dict(same[-1]["labelSelector"]) if same and rng.chance(25) else rng.pick(SAME_KEY_SELECTORS)
            # a DoNotSchedule maxSkew of 0 is a valid filter that no domain at or above the minimum passes
            skew = 0 if when == "DoNotSchedule" and rng.chance(8) else 1 + rng.below(3)
            cons.append({"maxSkew": skew, "topologyKey": key, "whenUnsatisfiable": when, "labelSelector": sel})
        if rng.chance(20):
            cons.append({"maxSkew": 2, "topologyKey": rng.pick([k for k in (host_key, zone_key, rack_key) if k != key]),
                         "whenUnsatisfiable": rng.pick(["DoNotSchedule", "ScheduleAnyway"]), "labelSelector": rng.pick(SAME_KEY_SELECTORS)})
        cont = {"name": "c", "image": f"registry.local/{name}:v1",
                "resources": {"requests": {"cpu": f"{_log_uniform(rng, 100, 3000, 50)}m", "memory": f"{_log_uniform(rng, 128, 4096, 64)}Mi"}}}
        spec = {"containers": [cont], "topologySpreadConstraints": cons}
        if rng.chance(20):
            spec["nodeSelector"] = {"pool": "a"}
        labels = dict(labelled(), app=name)
        if rng.chance(25):
            app.Resource.Pods.append({"apiVersion": "v1", "kind": "Pod", "metadata": {"name": name, "namespace": "default", "labels": labels},
                                      "spec": spec})
        else:
            app.Resource.Deployments.append({"apiVersion": "apps/v1", "kind": "Deployment", "metadata": {"name": name, "namespace": "default"},
                                             "spec": {"replicas": 1 + rng.below(max_replicas), "selector": {"matchLabels": {"app": name}},
                                                      "template": {"metadata": {"labels": labels}, "spec": spec}}})
    ds_cons = [{"maxSkew": 3, "topologyKey": zone_key, "whenUnsatisfiable": "DoNotSchedule", "labelSelector": sel}
               for sel in SAME_KEY_SELECTORS[:2]]
    app.Resource.DaemonSets.append({"apiVersion": "apps/v1", "kind": "DaemonSet", "metadata": {"name": "agent", "namespace": "default"},
                                    "spec": {"selector": {"matchLabels": {"app": "agent"}},
                                             "template": {"metadata": {"labels": {"app": "agent", "a": "x", "b": "y"}},
                                                          "spec": {"containers": [{"name": "a", "image": "registry.local/agent:v1",
                                                                                   "resources": {"requests": {"cpu": "50m", "memory": "64Mi"}}}],
                                                                   "topologySpreadConstraints": ds_cons}}}})
    return cluster, [app]


class LiveSnapshot:
    """A compiled cluster whose pod list is a set of RUNNING pods (spec.nodeName set): what importing a live cluster yields.
    Same arrays as compiler.Compiled as far as Engine / Oracle are concerned."""

    def __init__(self, base, pod_class, pod_fixed):
        self.snap, self.snap_dims = base.snap, dict(base.snap_dims)
        self.pods = dict(base.pods)
        self.pods["pod_class"] = np.ascontiguousarray(pod_class, dtype=np.int32)
        self.pods["pod_fixed_node"] = np.ascontiguousarray(pod_fixed, dtype=np.int32)
        self.pods["pod_pin_node"] = np.full(len(pod_class), -1, dtype=np.int32)
        self.pods_dims = dict(base.pods_dims)
        self.pods_dims["n_pods"] = len(pod_class)
        self.n_nodes = base.n_nodes
        self.node_names = base.node_names


def make_c5(compiled, n_running: int = 300000, seed_no: int = 5) -> LiveSnapshot:
    """C5 (SURVEY 8d): a live snapshot with ~n_running pods already bound.  The pods are instances of the classes of
    `compiled` (a C3-shaped cluster), each bound to a uniformly drawn node that still has room for it (CPU, memory, pod
    count); pods for which 8 draws find no room are dropped.  Pre-bound pods bypass the filters (simulator.go:326-329), so the
    snapshot may violate soft rules - as live clusters do."""
    rng = np.random.RandomState(0x5151 + seed_no)
    blob, off = compiled.pods["class_blob"], compiled.pods["class_off"]
    C = int(compiled.pods_dims["n_classes"])
    N = compiled.n_nodes
    hdr = np.array([[int(blob[int(off[k]) + w]) for w in (0, 1, 7, 10, 13)] for k in range(C)], dtype=np.int64)   # mcpu, mem, gpu, nodeName, guard
    usable = np.nonzero((hdr[:, 2] == 0) & (hdr[:, 3] == -1) & (hdr[:, 4] == -1))[0]      # no GPU share, not pinned, not a DaemonSet pod
    cap_c, cap_m, cap_p = compiled.snap["alloc_mcpu"].astype(np.int64), compiled.snap["alloc_mem"].astype(np.int64), compiled.snap["alloc_pods"].astype(np.int64)
    use_c, use_m, use_p = np.zeros(N, np.int64), np.zeros(N, np.int64), np.zeros(N, np.int64)
    cls_draw = usable[rng.randint(0, len(usable), n_running)]
    node_draw = rng.randint(0, max(N, 1), (n_running, 8))
    pc, pf = [], []
    for i in range(n_running):
        k = int(cls_draw[i])
        rc, rm = int(hdr[k, 0]), int(hdr[k, 1])
        for g in node_draw[i]:
            g = int(g)
            if use_p[g] + 1 <= cap_p[g] and use_c[g] + rc <= cap_c[g] and use_m[g] + rm <= cap_m[g]:
                use_p[g] += 1; use_c[g] += rc; use_m[g] += rm
                pc.append(k); pf.append(g)
                break
    return LiveSnapshot(compiled, np.array(pc, np.int32), np.array(pf, np.int32))
