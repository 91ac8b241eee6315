"""Nodes to add to the live cluster (Simulator.PlanAddNodes, simon_grow_run) on a seeded C3 session.

The C3 session of tools/session_bench.py (synth.make_c3: --nodes nodes, GPU share on ~25 % of them): RunCluster(PrepareCluster(cluster))
and ScheduleApp of its workloads.  The app PlanAddNodes plans for is --last-workloads C2 workloads (synth.make_c2's Deployments of CPU
and memory requests, --replicas each: 1,000 pods at the defaults) that select the node pool `node-pool: new` by nodeSelector.  The
running cluster has no such node, so the app needs new nodes: the --specs candidate specs are C2 shapes (the first nodes of
synth.make_c2: 64, 8, 128 and 128 cores at the defaults) labelled with that pool, k up to --kmax, with the sweep and the bisection.
Per method: the wall clock of PlanAddNodes split into the superset's compile and the plan (device batches and host work), the device
setup and placement ms of every batch, and the number of chunks.  For comparison, the recompile-plus-resume loop the call replaces
(compile the session's nodes + k copies with the pods that exist there, simon_schedule_resume from the session's placements) is timed
on --check sampled (spec, k), and each sample must place what the grow batch placed: the same tail nodes and GPU slots.
Prints one JSON line with the GPU's name and power limit, read in the same run.  Writes nothing."""
import argparse
import copy
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
from simon_b200 import grow, objects as O, synth
from simon_b200.compiler import compile_cluster
from simon_b200.engine import Engine
from simon_b200.scaledown import pod_guard
from simon_b200.simulator import NewSimulator, PrepareCluster

ap = argparse.ArgumentParser()
ap.add_argument("--nodes", type=int, default=10000)
ap.add_argument("--workloads", type=int, default=1000)
ap.add_argument("--gpu-pct", type=int, default=25)
ap.add_argument("--last-workloads", type=int, default=10)
ap.add_argument("--replicas", type=int, default=100)
ap.add_argument("--specs", type=int, default=4)
ap.add_argument("--kmax", type=int, default=64)
ap.add_argument("--check", type=int, default=3)
a = ap.parse_args()
if not torch.cuda.is_available():
    raise SystemExit("grow_bench.py needs a CUDA device (there is no CPU fallback)")
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()

cluster, apps = synth.make_c3(n_nodes=a.nodes, n_workloads=a.workloads, n_apps=1, gpu_pct=a.gpu_pct)
first = apps[0]
c2, c2_apps = synth.make_c2(n_nodes=a.specs, n_workloads=a.last_workloads, replicas=a.replicas)
POOL = {"node-pool": "new"}
last_deps = copy.deepcopy(c2_apps[0].Resource.Deployments)
for d in last_deps:
    d["metadata"]["name"] = "last-" + d["metadata"]["name"]
    labels = {"app": d["metadata"]["name"]}          # not the C3 workload's labels of the same name
    d["spec"]["selector"]["matchLabels"] = dict(labels)
    d["spec"]["template"]["metadata"]["labels"] = dict(labels)
    d["spec"]["template"]["spec"]["nodeSelector"] = dict(POOL)
last = O.AppResource("last", O.ResourceTypes(Deployments=last_deps))
specs = [copy.deepcopy(n) for n in c2.Nodes]
for i, s in enumerate(specs):
    s["metadata"]["name"] = f"c2-spec-{i}"
    s["metadata"]["labels"].update(POOL)

sim = NewSimulator()
t0 = time.perf_counter()
sim.RunCluster(PrepareCluster(cluster))
sim.ScheduleApp(first)
session_s = time.perf_counter() - t0
out = dict(gpu=gpu, nodes=a.nodes, session_pods=int(len(sim.placements)), session_s=round(session_s, 2), specs=a.specs, kmax=a.kmax)
for method in ("sweep", "bisect"):
    t0 = time.perf_counter()
    res = sim.PlanAddNodes([last], specs, kmax=a.kmax, method=method)
    wall = time.perf_counter() - t0
    batches = sim.last_grow
    out[method] = dict(wall_s=round(wall, 3), compile_s=round(sim.last_grow_timing["compile_s"], 3),
                       plan_s=round(sim.last_grow_timing["plan_s"], 3), batches=len(batches),
                       chunks=sum(b["chunks"] for b in batches),
                       setup_ms=[round(b["setup_ms"], 2) for b in batches], place_ms=[round(b["place_ms"], 2) for b in batches],
                       kernel=batches[0]["launches"][0]["kernel"] if batches and batches[0]["launches"] else "",
                       new_node_num=[s.NewNodeNum for s in res.Specs], best=res.Best, scenarios=res.ScenariosEvaluated,
                       rounds=res.Rounds)

# the recompile-plus-resume loop on sampled (spec, k), each checked against the grow batch
gs = grow.build(sim, [last], specs, a.kmax)
rng = np.random.default_rng(7)
picks = [(int(rng.integers(0, a.specs)), int(k)) for k in [0, a.kmax] + list(rng.integers(1, a.kmax, max(0, a.check - 2)))][:a.check]
with Engine(gs.compiled, device=0) as eng:
    raw = eng.grow_run(gs.placed, gs.n_prefix, [gs.scenario(s, k).nodes for s, k in picks])
guard = pod_guard(gs.compiled)
loop = []
for (s, k), r in zip(picks, raw):
    t0 = time.perf_counter()
    c = gs.compiled
    active = set(gs.scenario(s, k).nodes.tolist())
    keep = [q for q in range(c.pods_dims["n_pods"]) if not (guard[q] >= 0 and guard[q] not in active)]
    nodes = [c.node_objs[g] for g in sorted(active, key=lambda g: c.node_orig_index[g])]
    cc = compile_cluster(nodes, [c.pod_recs[q] for q in keep], sim._plan().ctx)
    t1 = time.perf_counter()
    with Engine(cc, device=0) as e2:
        o, _s, _fc, _fp = e2.schedule_resume(grow.remap(sim.compiled, cc, sim.placements))
        sl = e2.gpu_slot_words()
    t2 = time.perf_counter()
    to_super = np.array([c.node_index(nm) for nm in cc.node_names], np.int32)
    tail = np.array(keep[gs.n_prefix:], np.int64) - gs.n_prefix
    want = np.where(o[gs.n_prefix:] >= 0, to_super[np.maximum(o[gs.n_prefix:], 0)], o[gs.n_prefix:])
    same = bool(np.array_equal(r["node"][tail], want) and np.array_equal(r["gpu_slots"][tail], sl[gs.n_prefix:]))
    loop.append(dict(spec=s, k=k, compile_s=round(t1 - t0, 3), resume_s=round(t2 - t1, 3), same=same))
out["recompile_resume"] = loop
sim.Close()
print(json.dumps(out))
if not all(x["same"] for x in loop):
    raise SystemExit("a sampled scenario differs from its recompile-and-resume run")
