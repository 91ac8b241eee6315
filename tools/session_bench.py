"""The incremental session against a whole new Simulate() for "and what if I also deploy this app?".

A seeded C3 cluster (synth.make_c3: --nodes nodes, GPU-share on ~25 % of them) with its workloads split into a large first app and a
last app of --last-workloads Deployments (100 pods each).  Each round builds a session (RunCluster(PrepareCluster(cluster)), then
ScheduleApp(first), untimed) and then, alternating the order from round to round, times
  * ScheduleApp(last) end to end (plan + compile of cluster + both apps, context + uploads, rebuild of the earlier pods' state and
    placement of the last app's, result), and
  * Simulate(cluster, [first, last]) end to end;
and, on the context the session's last call left (the same compiled pod list), the device time of the rebuild + placement of the last
app (simon_schedule_resume) against the placement of every pod (simon_schedule from the empty state), alternated --steps times.
Checks in the same run that the two give identical results: NodeStatus pod lists and node objects, the last app's UnscheduledPods
(pod and reason text), and the session's placements and GPU-share slots against simon_schedule's.  Prints one JSON line with the GPU's
name and power limit.  Writes nothing."""
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
from simon_b200 import objects as O, synth
from simon_b200.simulator import NewSimulator, PrepareCluster, Simulate

ap = argparse.ArgumentParser()
ap.add_argument("--nodes", type=int, default=10000)
ap.add_argument("--workloads", type=int, default=1000)
ap.add_argument("--last-workloads", type=int, default=10)
ap.add_argument("--gpu-pct", type=int, default=25)
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--warmup", type=int, default=1)
ap.add_argument("--steps", type=int, default=5)
a = ap.parse_args()
if not torch.cuda.is_available():
    raise SystemExit("session_bench.py needs a CUDA device (there is no CPU fallback)")

cluster, apps = synth.make_c3(n_nodes=a.nodes, n_workloads=a.workloads, n_apps=1, gpu_pct=a.gpu_pct)
deps = apps[0].Resource.Deployments
first = O.AppResource("first", O.ResourceTypes(Deployments=deps[:-a.last_workloads]))
last = O.AppResource("last", O.ResourceTypes(Deployments=deps[-a.last_workloads:]))


def pod_id(r):
    return (r.app_name,) + r.key()


def same_result(x, y, app_name):
    if len(x.NodeStatus) != len(y.NodeStatus):
        return False
    for s, t in zip(x.NodeStatus, y.NodeStatus):
        if s.Node != t.Node or [pod_id(r) for r in s.Pods] != [pod_id(r) for r in t.Pods]:
            return False
    mine = [(pod_id(u.Pod), u.Reason) for u in x.UnscheduledPods]
    ref = [(pod_id(u.Pod), u.Reason) for u in y.UnscheduledPods if u.Pod.app_name == app_name]
    return mine == ref


session_s, simulate_s, timings, sim_timings, identical = [], [], [], [], True
resume_ms, full_ms = [], []
n_prefix = n_pods = 0
for rnd in range(a.warmup + a.rounds):
    sim = NewSimulator()
    sim.RunCluster(PrepareCluster(cluster))
    sim.ScheduleApp(first)
    prefix = sim.placements.copy()
    res_s = res_r = None
    for which in ((0, 1) if rnd % 2 == 0 else (1, 0)):
        t0 = time.perf_counter()
        if which == 0:
            res_s = sim.ScheduleApp(last)
            dt_s = time.perf_counter() - t0
        else:
            res_r = Simulate(cluster, [first, last])
            dt_r = time.perf_counter() - t0
            sim_timing = dict(Simulate.last_timing)
    identical &= same_result(res_s, res_r, "last")
    eng = sim.engine
    n_prefix, n_pods = len(prefix), len(sim.placements)
    placements, slots = sim.placements.copy(), sim.gpu_slots.copy()
    for step in range(a.steps):
        for which in ((0, 1) if step % 2 == 0 else (1, 0)):
            if which == 0:
                out = eng.schedule_resume(prefix)[0]
                ms = eng.last_kernel_ms()
                if rnd >= a.warmup:
                    resume_ms.append(ms)
                identical &= bool(np.array_equal(out, placements) and np.array_equal(eng.gpu_slot_words(), slots))
            else:
                eng.reset()
                out = eng.schedule()[0]
                ms = eng.last_kernel_ms()
                if rnd >= a.warmup:
                    full_ms.append(ms)
                identical &= bool(np.array_equal(out, placements) and np.array_equal(eng.gpu_slot_words(), slots))
    if rnd >= a.warmup:
        session_s.append(dt_s)
        simulate_s.append(dt_r)
        timings.append(dict(sim.last_timing))
        sim_timings.append(sim_timing)
    sim.Close()

gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                     capture_output=True, text=True).stdout.strip()
med = statistics.median
print(json.dumps({
    "gpu": gpu or torch.cuda.get_device_name(0), "nodes": a.nodes, "pods": n_pods, "prefix_pods": n_prefix, "last_app_pods": n_pods - n_prefix,
    "schedule_app_s": round(med(session_s), 4), "simulate_s": round(med(simulate_s), 4),
    "schedule_app_s_all": [round(x, 4) for x in session_s], "simulate_s_all": [round(x, 4) for x in simulate_s],
    "schedule_app_phases": {k: round(med(t[k] for t in timings), 4) for k in timings[0]},
    "simulate_phases_s": {k: round(med(t[k] for t in sim_timings), 4) for k in sim_timings[0]},
    "device_ms_resume": round(med(resume_ms), 3), "device_ms_full_placement": round(med(full_ms), 3),
    "identical": bool(identical)}))
