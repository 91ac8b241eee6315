"""Rolling maintenance at production size: a plan over every node of a seeded C3 cluster, waves of --max-unavailable.

A seeded C3 cluster (synth.make_c3: --nodes nodes, GPU share on ~--gpu-pct % of them) is placed once (simon_schedule: the live state).
Then rolling.plan_rolling over all nodes on the device (Engine.wave_*): waves, skipped nodes, wall clock of the call, and device time
split into setup (copies of the base into the slots, counter removal), placement and commit.

Then the same cluster without GPU share (its GPU-share node capacities removed), where the wave definition and a rebuild per wave agree:
the plan by waves and the same plan by rebuilding per wave (Engine.drain_run from the host placement; the evicted pods' moves applied
on the host), alternated --rounds times on one context.  The two must give the same waves and final placement.
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
from simon_b200 import rolling, simulator, synth
from simon_b200.compiler import compile_cluster
from simon_b200.engine import Engine

ap = argparse.ArgumentParser()
ap.add_argument("--nodes", type=int, default=10000)
ap.add_argument("--workloads", type=int, default=1000)
ap.add_argument("--gpu-pct", type=int, default=25)
ap.add_argument("--max-unavailable", type=int, default=100)
ap.add_argument("--rounds", type=int, default=2)
a = ap.parse_args()
if not torch.cuda.is_available():
    raise SystemExit("rolling_bench.py needs a CUDA device (there is no CPU fallback)")


class RebuildRunner(rolling.WaveRunner):
    """The waves as drains from a host placement: every batch rebuilds the live state from it (simon_drain_run)."""

    def __init__(self, eng):
        self.eng = eng
        self.setup_ms = self.place_ms = 0.0

    def begin(self, placed):
        self.placed = np.array(placed, np.int32)

    def run(self, remain_lists):
        self.last = self.eng.drain_run(self.placed, remain_lists, detail=True)
        self.setup_ms += self.eng.last_drain["setup_ms"]
        self.place_ms += self.eng.last_drain["place_ms"]
        return self.last

    def commit(self, i):
        r = self.last[i]
        self.placed[r["evicted"]] = r["node"]

    def placement(self):
        return self.placed.copy(), np.zeros(len(self.placed), np.uint32)


def cluster(gpu_pct):
    cl, apps = synth.make_c3(n_nodes=a.nodes, n_workloads=a.workloads, n_apps=1, gpu_pct=gpu_pct)
    p = simulator.plan(cl, apps)
    return p, compile_cluster(p.nodes, p.pods, p.ctx)


def waves(plan):
    return [w.Nodes for w in plan.Waves], [s.Node for s in plan.Skipped]


gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
out = dict(bench="rolling_maintenance", gpu=gpu, max_unavailable=a.max_unavailable)
p, c = cluster(a.gpu_pct)
out.update(nodes=c.n_nodes, pods=len(p.pods), gpu_share_nodes=int((np.asarray(c.snap["gpu_count"]) > 0).sum()))
with Engine(c) as eng:
    placed = eng.schedule()[0]
    t0 = time.perf_counter()
    plan = rolling.plan_rolling(c, placed, rolling.EngineRunner(eng), max_unavailable=a.max_unavailable)
    wall = time.perf_counter() - t0
    info = eng.last_wave
    print(f"gpu-share plan: {wall:.1f} s", file=sys.stderr, flush=True)
    out.update(waves=plan.TotalWaves, skipped=len(plan.Skipped), moved_pods=plan.MovedPods, batches=info["batches"],
               wall_s=round(wall, 2), setup_ms=round(info["setup_ms"], 1), place_ms=round(info["place_ms"], 1),
               commit_ms=round(info["commit_ms"], 1), kernel=info["launches"][0]["kernel"])

p, c = cluster(0)
out["no_gpu_share"] = res = dict(nodes=c.n_nodes, pods=len(p.pods), wave_wall_s=[], rebuild_wall_s=[], wave_device_ms=[],
                                 rebuild_device_ms=[])
with Engine(c) as eng:
    placed = eng.schedule()[0]
    plans = []
    for _ in range(a.rounds):
        t0 = time.perf_counter()
        pw = rolling.plan_rolling(c, placed, rolling.EngineRunner(eng), max_unavailable=a.max_unavailable)
        res["wave_wall_s"].append(round(time.perf_counter() - t0, 2))
        i = eng.last_wave
        res["wave_device_ms"].append(round(i["setup_ms"] + i["place_ms"] + i["commit_ms"], 1))
        rr = RebuildRunner(eng)
        t0 = time.perf_counter()
        pr = rolling.plan_rolling(c, placed, rr, max_unavailable=a.max_unavailable)
        res["rebuild_wall_s"].append(round(time.perf_counter() - t0, 2))
        res["rebuild_device_ms"].append(round(rr.setup_ms + rr.place_ms, 1))
        plans.append((waves(pw), waves(pr), pw.FinalPlacement == pr.FinalPlacement))
        print(f"no-gpu-share round: waves {res['wave_wall_s'][-1]} s, rebuild {res['rebuild_wall_s'][-1]} s", file=sys.stderr, flush=True)
    res.update(waves=pw.TotalWaves, skipped=len(pw.Skipped), identical=all(x == y and f for x, y, f in plans),
               wave_wall_s_median=statistics.median(res["wave_wall_s"]), rebuild_wall_s_median=statistics.median(res["rebuild_wall_s"]))
print(json.dumps(out))
