"""The C4 capacity search with Open-Local storage: synth.make_c4 (2,000 base nodes ~85 % full, 50 Deployments x 100 pending pods,
8 candidate node specs x k = 1..32 -> 256 scenarios) with the simon/node-local-storage annotation (1-3 VGs, 0-4 SSD / HDD devices)
on ~60 % of the base nodes and on every other spec, and a quarter of the Deployments each asking for LVM volumes, a device volume,
or both.  Prints one JSON line:
  * seconds per search through simon_scenarios_run_local (best of --steps after --warmup; wall clock of capacity.search: the
    scenario lists, the launch, the reductions and the result download);
  * the same scenario set with every storage annotation stripped, through simon_scenarios_run, so the cost of storage shows;
  * whether --check sampled scenarios of the storage batch equal independent single-scenario runs of the same nodes and pods
    (placements by node name, VG requested per node and VG, device masks).
Writes nothing."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "open-simulator_b200"), ROOT):
    sys.path.insert(0, p)
import numpy as np
import torch
from simon_b200 import capacity, synth
from simon_b200 import objects as O
from simon_b200.compiler import ClusterContext, compile_cluster
from simon_b200.engine import Engine

GI = 1 << 30
ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=3)
ap.add_argument("--warmup", type=int, default=1)
ap.add_argument("--check", type=int, default=4, help="scenarios compared with single-scenario runs")
a = ap.parse_args()
if not torch.cuda.is_available():
    raise SystemExit("open_local_capacity_bench.py needs a CUDA device (there is no CPU fallback)")

rng = np.random.default_rng(8)
cluster, apps, specs = synth.make_c4(n_nodes=2000, n_workloads=50, replicas=100)
for m in ("ssd", "hdd"):
    cluster.StorageClasss.append({"apiVersion": "storage.k8s.io/v1", "kind": "StorageClass",
                                  "metadata": {"name": f"open-local-device-{m}"}, "parameters": {"mediaType": m}})


def annotate(node):
    vgs = [{"name": f"pool{v}", "capacity": str(int(rng.choice([200, 500, 1000])) * GI), "requested": str(int(rng.integers(0, 5)) * 10 * GI)}
           for v in range(int(rng.integers(1, 4)))]
    devs = [{"name": f"/dev/vd{k}", "device": f"/dev/vd{k}", "capacity": str(int(rng.choice([200, 400, 800])) * GI),
             "mediaType": str(rng.choice(["ssd", "hdd"])), "isAllocated": "true" if rng.random() < 0.05 else "false"}
            for k in range(int(rng.integers(0, 5)))]
    O.meta(node).setdefault("annotations", {})[O.ANNO_NODE_LOCAL_STORAGE] = json.dumps({"vgs": vgs, "devices": devs})


for n in cluster.Nodes:
    if rng.random() < 0.6:
        annotate(n)
for si, s in enumerate(specs):
    if si % 2 == 0:
        annotate(s)
for w, d in enumerate(apps[0].Resource.Deployments):
    kind = w % 4            # 0: no volume, 1: LVM, 2: a device, 3: both
    vols = []
    if kind in (1, 3):
        vols += [{"size": str(int(rng.choice([5, 10, 20])) * GI), "kind": "LVM", "scName": "open-local-lvm"}]
    if kind in (2, 3):
        m = str(rng.choice(["SSD", "HDD"]))
        vols.append({"size": str(int(rng.choice([50, 100])) * GI), "kind": m, "scName": f"open-local-device-{m.lower()}"})
    if vols:
        d["spec"]["template"].setdefault("metadata", {}).setdefault("annotations", {})[O.ANNO_POD_LOCAL_STORAGE] = json.dumps({"volumes": vols})

ks = list(range(1, 33))
t0 = time.perf_counter()
ss = capacity.build_scenarios(cluster, apps, specs, ks, open_local=True, local_devices=True)
build_s = time.perf_counter() - t0


def strip(objs):
    out = []
    for o in objs:
        o = O.deep_copy(o)
        for m in (O.meta(o), (o.get("spec", {}).get("template") or {}).get("metadata") or {}):
            (m.get("annotations") or {}).pop(O.ANNO_NODE_LOCAL_STORAGE, None)
            (m.get("annotations") or {}).pop(O.ANNO_POD_LOCAL_STORAGE, None)
        out.append(o)
    return out


bare_cluster = O.ResourceTypes(Nodes=strip(cluster.Nodes), Pods=list(cluster.Pods), Services=list(cluster.Services))
bare_apps = [O.AppResource(apps[0].Name, O.ResourceTypes(Deployments=strip(apps[0].Resource.Deployments)))]
ss_bare = capacity.build_scenarios(bare_cluster, bare_apps, strip(specs), ks)


def timed(s):
    with Engine(s.compiled, device=0) as eng:
        run = capacity.gpu_runner(0, engine=eng)
        for _ in range(a.warmup):
            capacity.search(s, run, max_cpu=100, max_mem=100, max_vg=100)
        times = []
        for _ in range(a.steps):
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            best, res = capacity.search(s, run, max_cpu=100, max_mem=100, max_vg=100)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t1)
        states = {}
        if s is ss:
            picks = sorted(np.random.default_rng(1).choice(len(s.scenarios), size=min(a.check, len(s.scenarios)), replace=False).tolist())
            out, nodes = eng.run_scenarios_local([sc.nodes for sc in s.scenarios], want_nodes=True)
            states = {i: (nodes[i], eng.scenario_storage_state(i)) for i in picks}
        return times, best, res, eng.last_kernel_ms(), states


t_local, best_local, res_local, ms_local, states = timed(ss)
t_bare, best_bare, _res_bare, ms_bare, _ = timed(ss_bare)

# sampled scenarios against their own single-scenario runs
c = ss.compiled
scs = list(cluster.StorageClasss)
ctx = ClusterContext(services=list(cluster.Services), replicasets=list(cluster.ReplicaSets), statefulsets=list(cluster.StatefulSets))
same = True
for i, (bnodes, (bvg, bdev)) in states.items():
    sc = ss.scenarios[i]
    act = sorted(int(g) for g in sc.nodes)
    names = {c.node_names[g] for g in act}
    keep = [q for q, p in enumerate(ss.pods) if not p.tmpl.guard_node_name or p.tmpl.guard_node_name in names]
    solo = compile_cluster([c.node_objs[g] for g in sorted(act, key=lambda g: c.node_orig_index[g])], [ss.pods[q] for q in keep], ctx,
                           open_local=True, storage_classes=scs, local_devices=True)
    with Engine(solo, device=0) as eng:
        out = eng.schedule()[0]
        vg, dev = eng.storage_state(), eng.device_state()
    got = [c.node_names[g] if g >= 0 else int(g) for g in bnodes[keep].tolist()]
    want = [solo.node_names[g] if g >= 0 else int(g) for g in out.tolist()]
    same &= got == want
    for g2, nm in enumerate(solo.node_names):
        g, nv = c.node_index(nm), int(solo.storage.node_n_vg[g2])
        same &= bvg[:nv, g].tolist() == vg[:nv, g2].tolist() and int(bdev[g]) == int(dev[g2])

gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                     capture_output=True, text=True).stdout.strip()
dec = capacity.decode_key(best_local)
print(json.dumps({
    "workload": "C4 + Open-Local: 2000-node base (~60 % with VGs / devices), 5000 pending pods (3/4 with volumes), "
                "8 specs (4 with storage) x k = 1..32 -> 256 scenarios",
    "scenarios": len(ss.scenarios), "gpu": gpu,
    "search_s_local": min(t_local), "search_s_local_all": t_local, "kernel_ms_local": ms_local,
    "search_s_without_storage": min(t_bare), "search_s_without_storage_all": t_bare, "kernel_ms_without_storage": ms_bare,
    "best_local": dec, "best_local_vg": (None if dec is None else {k: res_local[dec["scenario"]][k] for k in ("vg_requested", "vg_capacity")}),
    "best_without_storage": capacity.decode_key(best_bare),
    "solo_check": {"scenarios": sorted(states), "identical": bool(same)},
    "host_build_s": build_s,
    "timing": "wall clock of capacity.search (lists, launch, reductions, download), best of --steps"}))
