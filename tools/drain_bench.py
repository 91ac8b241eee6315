"""Node drains at production size: every single-node drain of a seeded C3 cluster, the scale-down planner, and sampled drains
against the recompile + resume path they are defined by.

A seeded C3 cluster (synth.make_c3: --nodes nodes, GPU-share on ~--gpu-pct % of them) is placed once (simon_schedule: the live state).
Then, on that context:
  * the sweep: one drain per node (the node alone removed), as batches sized from simon_drain_budget; device time of the setup
    (rebuild of the live state, clearing of the scenarios' per-class caches, copies into the scenario slots, counter removal) and of
    the placement, the evicted-pod decisions, the batches and the per-scenario pool bytes; --rounds sweeps after --warmup, median
    reported;
  * the planner (scaledown.plan_scale_down: sweep, order, prefixes up to --max-remove), wall clock end to end;
  * --samples drains of one node each through the recompile + simon_schedule_resume path (the cluster without the node, pod list
    [pods not on it] + [evicted pods], resumed): the evicted pods' nodes and GPU-share slots must equal the drain's; wall clock per
    drain of that path.
Prints one JSON line with the GPU's name and power limit.  Writes nothing."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "open-simulator_b200"), ROOT):
    sys.path.insert(0, p)
import numpy as np
import torch
from simon_b200 import objects as O, scaledown, simulator, synth
from simon_b200.compiler import compile_cluster
from simon_b200.engine import Engine

ap = argparse.ArgumentParser()
ap.add_argument("--nodes", type=int, default=10000)
ap.add_argument("--workloads", type=int, default=1000)
ap.add_argument("--gpu-pct", type=int, default=25)
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--warmup", type=int, default=1)
ap.add_argument("--max-remove", type=int, default=256)
ap.add_argument("--samples", type=int, default=8)
a = ap.parse_args()
if not torch.cuda.is_available():
    raise SystemExit("drain_bench.py needs a CUDA device (there is no CPU fallback)")

gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
t0 = time.perf_counter()
cluster, apps = synth.make_c3(n_nodes=a.nodes, n_workloads=a.workloads, n_apps=1, gpu_pct=a.gpu_pct)
p = simulator.plan(cluster, apps)
c = compile_cluster(p.nodes, p.pods, p.ctx)
setup_s = time.perf_counter() - t0
out = dict(bench="drain_sweep", gpu=gpu, nodes=c.n_nodes, pods=len(p.pods), classes=int(c.pods_dims["n_classes"]), setup_s=round(setup_s, 2))

with Engine(c) as eng:
    placed = eng.schedule()[0]
    out["live_unscheduled"] = int((placed == -1).sum())
    order = scaledown.NodeOrder(c)
    t0 = time.perf_counter()
    remain = [order.remaining([g]) for g in range(c.n_nodes)]
    out["orders_s"] = round(time.perf_counter() - t0, 2)
    sweeps = []
    for r in range(a.warmup + a.rounds):
        t0 = time.perf_counter()
        res = eng.drain_run(placed, remain, detail=False)
        wall = time.perf_counter() - t0
        if r >= a.warmup:
            info = eng.last_drain
            sweeps.append(dict(wall_s=wall, setup_ms=info["setup_ms"], place_ms=info["place_ms"], chunks=info["chunks"]))
    info = eng.last_drain
    out.update(scenario_bytes=info["scenario_bytes"], chunk=info["chunk"], chunks=info["chunks"], kernel=info["launches"][0]["kernel"],
               geometry=[info["launches"][0][k] for k in ("cluster_ctas", "threads_per_cta", "node_slots")])
    out["evicted_decisions"] = int(sum(r["n_evicted"] for r in res))
    out["drainable_nodes"] = int(sum(1 for r in res if r["n_blocked"] == 0 and r["n_unscheduled"] == 0))
    for k in ("wall_s", "setup_ms", "place_ms"):
        out[f"sweep_{k}_median"] = round(statistics.median(s[k] for s in sweeps), 3)
    out["sweep_device_ms_median"] = round(statistics.median(s["setup_ms"] + s["place_ms"] for s in sweeps), 3)
    out["sweeps"] = sweeps

    t0 = time.perf_counter()
    plan = scaledown.plan_scale_down(c, placed, lambda rl: eng.drain_run(placed, rl, detail=False), max_remove=a.max_remove)
    out.update(plan_s=round(time.perf_counter() - t0, 2), plan_removed=len(plan.RemovedNodes), plan_prefixes=len(plan.Prefixes))

    rng = np.random.default_rng(1)
    gpu_nodes = np.nonzero(c.snap["gpu_count"] > 0)[0]
    picks = [int(g) for g in rng.choice(gpu_nodes, a.samples // 2, replace=False)] + \
            [int(g) for g in rng.choice(c.n_nodes, a.samples - a.samples // 2, replace=False)]
    got = eng.drain_run(placed, [order.remaining([g]) for g in picks])

names = c.node_names
same = True
resume_s = []
for g, d in zip(picks, got):
    t0 = time.perf_counter()
    ev, bl, va = scaledown.classify(c, placed, [g])
    gone = set(ev) | {q for q, _ in bl} | set(va)
    first = [q for q in range(len(p.pods)) if q not in gone]
    nodes = [n for n in p.nodes if O.name_of(n) != names[g]]
    c2 = compile_cluster(nodes, [p.pods[q] for q in first] + [p.pods[q] for q in ev], p.ctx)
    prefix = np.array([c2.node_index(names[placed[q]]) if placed[q] >= 0 else placed[q] for q in first], np.int32)
    with Engine(c2) as e2:
        o2 = e2.schedule_resume(prefix)[0]
        s2 = e2.gpu_slot_words()
    resume_s.append(time.perf_counter() - t0)
    nf = len(first)
    same &= [c2.node_names[x] if x >= 0 else None for x in o2[nf:]] == [names[x] if x >= 0 else None for x in d["node"]]
    same &= bool(np.array_equal(s2[nf:], d["gpu_slots"])) and d["evicted"].tolist() == ev
out.update(samples=len(picks), samples_identical=bool(same), recompile_resume_s_median=round(statistics.median(resume_s), 2))
print(json.dumps(out))
