"""Open-Local volumes (LVM and exclusive SSD / HDD devices) at scale: a seeded cluster (synth.make_open_local: --nodes nodes, ~60 %
of them with storage, 200 Deployments x 250 pods mixing no volume, LVM only, devices only and both).  Prints one JSON line: the
device time of a full pass (CUDA events, mean of --steps passes after warm-up, L2 flushed before each) as decisions/s, and whether
the engine's final VG state and device masks equal the host's replay of Bind in placement order (one lvm_place / device_place per
placed pod).  Writes nothing."""
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
from simon_b200 import simulator, synth
from simon_b200.compiler import compile_cluster
from simon_b200.engine import Engine
from simon_b200.storage import StorageReplay

ap = argparse.ArgumentParser()
ap.add_argument("--nodes", type=int, default=10000)
ap.add_argument("--steps", type=int, default=3)
ap.add_argument("--warmup", type=int, default=2)
a = ap.parse_args()
if not torch.cuda.is_available():
    raise SystemExit("open_local_bench.py needs a CUDA device (there is no CPU fallback)")
cluster, apps = synth.make_open_local(n_nodes=a.nodes)
t0 = time.perf_counter()
p = simulator.plan(cluster, apps)
c = compile_cluster(p.nodes, p.pods, p.ctx, open_local=True, storage_classes=list(cluster.StorageClasss), local_devices=True)
host_s = time.perf_counter() - t0
D = int((c.pods["pod_fixed_node"] == -1).sum())
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda:0")
with Engine(c, device=0) as eng:
    for _ in range(a.warmup):
        eng.replay(1)
    ms = 0.0
    for _ in range(a.steps):
        flush.zero_()
        torch.cuda.synchronize()
        ms += eng.replay(1)
    eng.reset()
    out = eng.schedule()[0]
    vg, dev = eng.storage_state(), eng.device_state()
rep = StorageReplay(c.storage, c.node_names)
pod_class = c.pods["pod_class"]
try:
    for i, n in enumerate(out.tolist()):
        if n >= 0:
            rep.bind(int(pod_class[i]), n)
    same = bool(np.array_equal(vg, rep.requested()) and np.array_equal(dev, rep.alloc_masks()))
except AssertionError:          # a placement the restated Filter rejects
    same = False
st = c.storage
local_cls = st.class_local[pod_class].astype(bool)
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                     capture_output=True, text=True).stdout.strip()
print(json.dumps({
    "workload": f"Open-Local: {c.n_nodes} nodes ({int((st.node_n_vg >= 0).sum())} with storage, "
                f"{int(st.node_n_ssd.sum()) + int(st.node_n_hdd.sum())} SSD / HDD devices) x {D} pods ({int(local_cls.sum())} with volumes)",
    "value": D * a.steps / (ms * 1e-3), "unit": "decisions/s", "ms_per_step": ms / a.steps, "host_compile_s": host_s,
    "placed": int((out >= 0).sum()), "placed_with_volumes": int(((out >= 0) & local_cls).sum()),
    "unschedulable": int((out == -1).sum()), "replay_identical": same, "gpu": gpu}), flush=True)
