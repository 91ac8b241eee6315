"""Cost of explained placement decisions (simon_explain_set) on the C3 headline pod list of bench.py.

The C3 cluster and pod list of bench.py's headline (synth.make_c3: --nodes nodes, --workloads workloads x --replicas replicas, 10 apps,
seed 3, the list of bench.py's first GPU) is placed on one context from the empty state in these modes, alternated round by round so that each mode sees the same
machine conditions: no pod explained, 1 % of the pods that reach the scheduler explained (every 100th) at top_k 3, and every pod
explained at top_k 1, 3 and 8.  Per mode: the median and spread of the device time of the whole list (simon_last_kernel_ms), the
kernel launched, the records' bytes on the device, and whether the placements equal those of the unexplained run.
Prints one JSON line with the GPU's name and power limit, read in the same run.  Writes nothing."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "open-simulator_b200"), ROOT):
    sys.path.insert(0, p)
import numpy as np
import torch
from simon_b200 import abi, simulator, synth
from simon_b200.compiler import compile_cluster
from simon_b200.engine import Engine

ap = argparse.ArgumentParser()
ap.add_argument("--nodes", type=int, default=10000)
ap.add_argument("--workloads", type=int, default=1000)
ap.add_argument("--replicas", type=int, default=100)
ap.add_argument("--rounds", type=int, default=5)
a = ap.parse_args()
if not torch.cuda.is_available():
    raise SystemExit("explain_bench.py needs a CUDA device (there is no CPU fallback)")
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()

cluster, apps = synth.make_c3(n_nodes=a.nodes, n_workloads=a.workloads, replicas=a.replicas, n_apps=10, seed_no=3)
p = simulator.plan(cluster, apps)
c = compile_cluster(p.nodes, p.pods, p.ctx)
P = c.pods_dims["n_pods"]
reached = np.nonzero(c.pods["pod_fixed_node"] == -1)[0].astype(np.uint32)
every = np.arange(P, dtype=np.uint32)
MODES = {"none": (None, 0), "1pct_top3": (reached[::100], 3), "all_top1": (every, 1), "all_top3": (every, 3), "all_top8": (every, 8)}

res = {m: dict(ms=[], kernel=None, record_bytes=0, same_placements=True) for m in MODES}
with Engine(c, device=0) as eng:
    ref = None
    for r in range(a.rounds + 1):                 # round 0 warms every mode up and is not counted
        for m, (pods, k) in MODES.items():
            eng.explain_set([] if pods is None else pods, max(k, 1))
            eng.reset()
            eng.schedule(download=False)
            ms = eng.last_kernel_ms()
            out = eng.results()
            if ref is None:
                ref = out
            res[m]["same_placements"] &= bool(np.array_equal(out, ref))
            res[m]["kernel"] = eng.last_launch()["kernel"]
            n = 0 if pods is None else len(pods)
            res[m]["record_bytes"] = n * (abi.EXPLAIN_RECORD_DTYPE.itemsize + k * abi.EXPLAIN_NODE_DTYPE.itemsize)
            res[m]["explained"] = n
            if r:
                res[m]["ms"].append(ms)
for m in res:
    v = np.array(res[m].pop("ms"))
    res[m].update(median_ms=float(np.median(v)), min_ms=float(v.min()), max_ms=float(v.max()))
base = res["none"]["median_ms"]
for m in res:
    res[m]["vs_none"] = res[m]["median_ms"] / base
print(json.dumps(dict(gpu=gpu, nodes=a.nodes, pods=P, reach_scheduler=int(len(reached)), rounds=a.rounds, modes=res)))
