"""Node drains on a cluster with Open-Local storage, with and without moving the pods that have local volumes.

A seeded Open-Local cluster (synth.make_open_local: --nodes nodes, ~60 % of them with VGs and SSD / HDD devices, 200 Deployments x 250
pods mixing no volume, LVM only, devices only and both), compiled with storage and devices, is placed once (the live state).  Then,
on that context:
  * the sweep of every single-node drain, with local volumes off (Engine.drain_run: pods with volumes block) and on
    (Engine.drain_run(..., local=True): they are evicted and provisioned again), alternated --rounds times after --warmup: per mode
    the medians of the setup and placement device time (simon_drain_times, summed over the batches) and of the wall clock, the
    batches, the evicted pods and how many of them carry volumes, and the drainable nodes;
  * the planner with local volumes (scaledown.plan_scale_down over drain_run(..., local=True), capped at --max-remove nodes) with
    MaxVG unset and with MaxVG one point below the VG occupancy of the unset plan's last accepted prefix, which binds;
  * --samples single-node drains with local volumes against the recompile + simon_schedule_resume path (the cluster without the
    node compiled with storage and devices, pod list [pods not on it] + [evicted pods], resumed): the evicted pods' nodes and GPU
    slots, and the final VG requested and device masks of every remaining node, must be identical.
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
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--warmup", type=int, default=1)
ap.add_argument("--max-remove", type=int, default=256)
ap.add_argument("--samples", type=int, default=8)
a = ap.parse_args()
if not torch.cuda.is_available():
    raise SystemExit("drain_local_bench.py needs a CUDA device (there is no CPU fallback)")

gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
t0 = time.perf_counter()
cluster, apps = synth.make_open_local(n_nodes=a.nodes)
scs = list(cluster.StorageClasss)
p = simulator.plan(cluster, apps)
c = compile_cluster(p.nodes, p.pods, p.ctx, open_local=True, storage_classes=scs, local_devices=True)
setup_s = time.perf_counter() - t0
local_cls = c.storage.class_local[c.pods["pod_class"]].astype(bool)
out = dict(bench="drain_local_sweep", gpu=gpu, nodes=c.n_nodes, pods=len(p.pods), pods_with_volumes=int(local_cls.sum()),
           classes=int(c.pods_dims["n_classes"]), setup_s=round(setup_s, 2))


def sweep_stats(res, eng):
    info = eng.last_drain
    ev = [q for r in res for q in r["evicted"].tolist()]
    return dict(setup_ms=info["setup_ms"], place_ms=info["place_ms"], chunks=info["chunks"], evicted=len(ev),
                evicted_with_volumes=int(local_cls[np.asarray(ev, dtype=np.int64)].sum()) if ev else 0,
                blocked=int(sum(r["n_blocked"] for r in res)), drainable=int(sum(1 for r in res if scaledown.drainable(r))),
                kernel=info["launches"][0]["kernel"])


with Engine(c) as eng:
    placed = eng.schedule()[0]
    out["live_unscheduled"] = int((placed == -1).sum())
    order = scaledown.NodeOrder(c)
    remain = [order.remaining([g]) for g in range(c.n_nodes)]
    runs = {False: [], True: []}
    for r in range(a.warmup + a.rounds):
        for local in (False, True):
            t0 = time.perf_counter()
            res = eng.drain_run(placed, remain, detail=True, local=local)
            wall = time.perf_counter() - t0
            if r >= a.warmup:
                runs[local].append(dict(sweep_stats(res, eng), wall_s=wall))
    for local, rs in runs.items():
        key = "local" if local else "plain"
        last = rs[-1]
        out[key] = dict(kernel=last["kernel"], chunks=last["chunks"], evicted=last["evicted"],
                        evicted_with_volumes=last["evicted_with_volumes"], blocked=last["blocked"], drainable=last["drainable"],
                        **{f"{k}_median": round(statistics.median(x[k] for x in rs), 3) for k in ("setup_ms", "place_ms", "wall_s")},
                        rounds=[{k: round(x[k], 3) for k in ("setup_ms", "place_ms", "wall_s")} for x in rs])
    out["scenario_bytes"] = eng.last_drain["scenario_bytes"]

    def runner(rl):
        return eng.drain_run(placed, rl, detail=False, local=True)
    t0 = time.perf_counter()
    plan = scaledown.plan_scale_down(c, placed, runner, max_remove=a.max_remove, max_vg=100)
    out["plan_unset"] = dict(s=round(time.perf_counter() - t0, 2), removed=len(plan.RemovedNodes), prefixes=len(plan.Prefixes))
    ok = [q for q in plan.Prefixes if q["ok"]]
    if ok and ok[-1]["vg_capacity"]:
        occ = int(float(ok[-1]["vg_requested"]) / float(ok[-1]["vg_capacity"]) * 100)
        cap = max(0, occ - 1)
        t0 = time.perf_counter()
        plan2 = scaledown.plan_scale_down(c, placed, runner, max_remove=a.max_remove, max_vg=cap)
        out["plan_capped"] = dict(max_vg=cap, s=round(time.perf_counter() - t0, 2), removed=len(plan2.RemovedNodes),
                                  prefixes=len(plan2.Prefixes))

    rng = np.random.default_rng(1)
    vol_nodes = sorted({int(placed[q]) for q in np.nonzero(local_cls & (placed >= 0))[0].tolist()})
    picks = [int(g) for g in rng.choice(vol_nodes, a.samples, replace=False)]
    got = eng.drain_run(placed, [order.remaining([g]) for g in picks], local=True)
    states = [eng.scenario_storage_state(i) for i in range(len(picks))]

names = c.node_names
same = True
resume_s = []
for g, d, (vg, dev) in zip(picks, got, states):
    t0 = time.perf_counter()
    ev, bl, va = scaledown.classify(c, placed, [g], local_volumes=True)
    gone = set(ev) | {q for q, _ in bl} | set(va)
    first = [q for q in range(len(p.pods)) if q not in gone]
    nodes = [n for n in p.nodes if O.name_of(n) != names[g]]
    c2 = compile_cluster(nodes, [p.pods[q] for q in first] + [p.pods[q] for q in ev], p.ctx, open_local=True, storage_classes=scs,
                         local_devices=True)
    prefix = np.array([c2.node_index(names[placed[q]]) if placed[q] >= 0 else placed[q] for q in first], np.int32)
    with Engine(c2) as e2:
        o2 = e2.schedule_resume(prefix)[0]
        s2 = e2.gpu_slot_words()
        vg2, dev2 = e2.storage_state(), e2.device_state()
    resume_s.append(time.perf_counter() - t0)
    nf = len(first)
    same &= [c2.node_names[x] if x >= 0 else None for x in o2[nf:]] == [names[x] if x >= 0 else None for x in d["node"]]
    same &= bool(np.array_equal(s2[nf:], d["gpu_slots"])) and d["evicted"].tolist() == ev
    for g2, nm in enumerate(c2.node_names):
        x = c.node_index(nm)
        nv = max(int(c2.storage.node_n_vg[g2]), 0)
        same &= vg[:nv, x].tolist() == vg2[:nv, g2].tolist() and int(dev[x]) == int(dev2[g2])
out.update(samples=len(picks), samples_evicted_with_volumes=int(sum(local_cls[d["evicted"].astype(np.int64)].sum() for d in got)),
           samples_identical=bool(same), recompile_resume_s_median=round(statistics.median(resume_s), 2))
print(json.dumps(out))
