"""Node-pool replacement at production size: every node of one node shape of a seeded C3 session replaced by a spec of twice its cores
and memory.

A seeded C3 session (synth.make_c3: --nodes nodes, GPU share on ~--gpu-pct % of them) runs once (RunCluster and ScheduleApp).  The
pool is every node of the synth's most common (cpu, memory) shape.  Simulator.PlanNodeReplacement sizes the replacement (one batch
of k = 0 .. kmax) and plans it at MinNodes with --max-surge and --max-unavailable.  Reports batches, waves, skipped nodes, moved pods,
device time split into setup (copies of the base into the slots, counter removal), placement and commit, the superset's compile time
and the wall clock of the call.

Then the same cluster without GPU share (its GPU-share node capacities removed), where the wave base and a rebuild per wave agree: the
plan by waves (replace.plan_replacement on Engine.wave_*) and the same plan by rebuilding the state for every wave batch from the host
placement (simon_wave_begin_pool, the drains' rebuild of the live state, before each batch; the committed moves applied on the host),
one after the other on one context.  The two must give the same sizing, waves, skipped nodes and final placement.
Prints one JSON line with the GPU's name and power limit.  Writes nothing."""
import argparse
import copy
import json
import os
import subprocess
import sys
import time
from collections import Counter

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "open-simulator_b200"), ROOT):
    sys.path.insert(0, p)
import numpy as np
import torch
from simon_b200 import objects as O, replace, rolling, simulator, synth
from simon_b200.engine import Engine
from simon_b200.quantity import Quantity

ap = argparse.ArgumentParser()
ap.add_argument("--nodes", type=int, default=10000)
ap.add_argument("--workloads", type=int, default=1000)
ap.add_argument("--gpu-pct", type=int, default=25)
ap.add_argument("--max-surge", type=int, default=10)
ap.add_argument("--max-unavailable", type=int, default=0)
a = ap.parse_args()
if not torch.cuda.is_available():
    raise SystemExit("replace_bench.py needs a CUDA device (there is no CPU fallback)")


def shape(n):
    al = n["status"]["allocatable"]
    return Quantity.parse(al["cpu"]).milli_value(), Quantity.parse(al["memory"]).int_value()


def doubled(n):
    n = copy.deepcopy(n)
    n["metadata"]["name"] = "replacement"
    for part in ("allocatable", "capacity"):
        al = n["status"].get(part)
        if al:
            c, m = Quantity.parse(al["cpu"]).milli_value(), Quantity.parse(al["memory"]).int_value()
            al["cpu"], al["memory"] = f"{2 * c}m", str(2 * m)
    return n


class RebuildRunner(rolling.WaveRunner):
    """The waves with the state rebuilt from a host placement for every batch: simon_wave_begin_pool from it (the pods of retired
    nodes' DaemonSets as pending, retired nodes as absent, which no remain list names), then the batch; a commit applies the moves
    on the host."""

    def __init__(self, eng, guard):
        self.eng, self.guard = eng, guard
        self.setup_ms = self.place_ms = 0.0

    def begin(self, placed, present=None):
        self.placed = np.array(placed, np.int32)
        self.state = np.asarray(present, bool).astype(np.int8)

    def run(self, remain_lists, joins=None):
        self.eng.wave_begin(np.where(self.placed == -3, -1, self.placed), self.state == 1)
        self.last, self.last_remain = self.eng.wave_run(remain_lists, joins, detail=True), remain_lists
        self.last_joins = joins
        self.setup_ms += self.eng.last_wave["setup_ms"]
        self.place_ms += self.eng.last_wave["place_ms"]
        return self.last

    def commit(self, i, retire=False):
        r = self.last[i]
        self.placed[r["evicted"]] = r["node"]
        self.placed[r["join_pods"]] = r["join_node"]
        self.state[np.asarray(self.last_joins[i], np.int64)] = 1
        keep = np.zeros(len(self.state), bool)
        keep[np.asarray(self.last_remain[i], np.int64)] = True
        gone = (self.state == 1) & ~keep
        self.state[gone] = 2
        g = self.guard
        self.placed[(g >= 0) & gone[np.maximum(g, 0)]] = -3

    def placement(self):
        return self.placed.copy(), np.zeros(len(self.placed), np.uint32)


def session(cl, apps):
    sim = simulator.NewSimulator()
    sim.RunCluster(cl)
    for app in apps:
        sim.ScheduleApp(app)
    return sim


def outline(plan):
    return (plan.Sizing, [(w.Joined, w.Nodes, [(e.Pod.name, e.To) for e in w.Evicted], [(j.Pod.name, j.Node) for j in w.JoinPods])
                          for w in plan.Waves], [(s.Node, s.Reasons) for s in plan.Skipped], plan.FinalPlacement)


gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
cl, apps = synth.make_c3(n_nodes=a.nodes, n_workloads=a.workloads, n_apps=1, gpu_pct=a.gpu_pct)
sim = session(cl, apps)
shapes = Counter(shape(n) for n in cl.Nodes)
top = shapes.most_common(1)[0][0]
pool = [O.name_of(n) for n in cl.Nodes if shape(n) == top]
spec = doubled(next(n for n in cl.Nodes if shape(n) == top))
t0 = time.perf_counter()
plan = sim.PlanNodeReplacement(pool, spec, max_surge=a.max_surge, max_unavailable=a.max_unavailable)
wall = time.perf_counter() - t0
info = sim.last_replace
out = dict(bench="node_replacement", gpu=gpu, nodes=len(cl.Nodes), pods=len(sim.placements), pool=len(pool),
           shape_mcpu=top[0], shape_mem=top[1], max_surge=a.max_surge, max_unavailable=a.max_unavailable,
           min_nodes=plan.Sizing.MinNodes, count=plan.Count, batches=info["batches"], waves=plan.TotalWaves, skipped=len(plan.Skipped),
           joined=plan.JoinedNodes, retired=plan.RetiredNodes, never_joined=len(plan.NeverJoined), moved_pods=plan.MovedPods,
           setup_ms=round(info["setup_ms"], 1), place_ms=round(info["place_ms"], 1), commit_ms=round(info["commit_ms"], 1),
           compile_s=round(sim.last_replace_timing["compile_s"], 2), wall_s=round(wall, 2), kernel=info["launches"][0]["kernel"])
print(f"gpu-share plan: {wall:.1f} s", file=sys.stderr, flush=True)
sim.Close()

cl, apps = synth.make_c3(n_nodes=a.nodes, n_workloads=a.workloads, n_apps=1, gpu_pct=0)
sim = session(cl, apps)
pool = [O.name_of(n) for n in cl.Nodes if shape(n) == top]
c, placed, present, pidx, copies, _ = replace.superset(sim, pool, doubled(next(n for n in cl.Nodes if shape(n) == top)), len(pool))
from simon_b200.scaledown import pod_guard
res = out["no_gpu_share"] = dict(pool=len(pool))
with Engine(c) as eng:
    kw = dict(max_surge=a.max_surge, max_unavailable=a.max_unavailable)
    t0 = time.perf_counter()
    pw = replace.plan_replacement(c, placed, rolling.EngineRunner(eng), present, pidx, copies, **kw)
    res["wave_wall_s"] = round(time.perf_counter() - t0, 2)
    i = eng.last_wave
    res["wave_device_ms"] = round(i["setup_ms"] + i["place_ms"] + i["commit_ms"], 1)
    rr = RebuildRunner(eng, np.asarray(pod_guard(c)))
    t0 = time.perf_counter()
    pr = replace.plan_replacement(c, placed, rr, present, pidx, copies, **kw)
    res["rebuild_wall_s"] = round(time.perf_counter() - t0, 2)
    res["rebuild_device_ms"] = round(rr.setup_ms + rr.place_ms, 1)
res.update(min_nodes=pw.Sizing.MinNodes, waves=pw.TotalWaves, skipped=len(pw.Skipped), moved_pods=pw.MovedPods,
           identical=outline(pw) == outline(pr))
print(json.dumps(out))
if not res["identical"]:
    raise SystemExit("the plan by waves and the plan rebuilt per wave differ")
