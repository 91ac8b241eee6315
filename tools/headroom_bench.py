"""Scheduling headroom (Simulator.Headroom, simon_probe_run) on a seeded C3 session and an Open-Local cluster.

The C3 session of tools/session_bench.py (synth.make_c3: --nodes nodes, GPU share on ~25 % of them, RunCluster(PrepareCluster(cluster))
then ScheduleApp of its workloads), timed for
  (a) one workload probe per workload of the cluster and apps, capped at --workload-cap replicas (the live context, no recompile);
  (b) --templates template probes of C2 shapes (the pod templates of synth.make_c2's Deployments that request CPU and memory) with
      the default cap, the cluster's free pod slots (one compile of the session's pods + the templates, on a context of its own);
  (c) workload probes of the Deployments with volumes on synth.make_open_local (a session WithOpenLocal(devices=True)), capped at
      --workload-cap.
Per case: device setup and placement ms (summed over the batches), batches, replicas placed, replica decisions per second of device
time (placed replicas + the failed decision of each Unschedulable probe, over setup + placement), and the wall clock of the call.  8
sampled probes per case (among those with fewer than --check-max replicas) are checked against the
equivalence that defines them: the pod list with the probe's replicas appended, resumed with the live placements as the prefix
(simon_schedule_resume), gives the same nodes and GPU slots, and the copy after them fails.
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
from simon_b200 import headroom, synth
from simon_b200.compiler import compile_cluster
from simon_b200.engine import Engine
from simon_b200.simulator import NewSimulator, PrepareCluster, WithOpenLocal
from simon_b200.workloads import make_valid_pod_by_pod

ap = argparse.ArgumentParser()
ap.add_argument("--nodes", type=int, default=10000)
ap.add_argument("--workloads", type=int, default=1000)
ap.add_argument("--gpu-pct", type=int, default=25)
ap.add_argument("--templates", type=int, default=64)
ap.add_argument("--workload-cap", type=int, default=64)
ap.add_argument("--check", type=int, default=8)
ap.add_argument("--check-max", type=int, default=10 ** 7)
a = ap.parse_args()
if not torch.cuda.is_available():
    raise SystemExit("headroom_bench.py needs a CUDA device (there is no CPU fallback)")
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()


def workload_refs(compiled, want=None):
    """Kind/namespace/name of every workload whose pods reach the scheduler (want: a predicate on the first pod index)."""
    guard = headroom.pod_guard(compiled)
    seen = {}
    for q, r in enumerate(compiled.pod_recs):
        if compiled.pods["pod_fixed_node"][q] != -1 or guard[q] != -1:
            continue
        k = (r.tmpl.workload_kind, r.tmpl.workload_namespace, r.workload_name)
        if k not in seen:
            seen[k] = q
    return [f"{k}/{ns}/{n}" for (k, ns, n), q in seen.items() if want is None or want(q)]


def timed(sim, probes, cap):
    t0 = time.perf_counter()
    res = sim.Headroom(probes, max_replicas=cap)
    wall = time.perf_counter() - t0
    info = sim.last_headroom
    setup = sum(x["setup_ms"] for x in info)
    place = sum(x["place_ms"] for x in info)
    placed = sum(r.Replicas for r in res)
    decisions = placed + sum(r.Stopped == "Unschedulable" for r in res)
    return res, dict(probes=len(res), setup_ms=round(setup, 2), place_ms=round(place, 2), batches=sum(x["chunks"] for x in info),
                     replicas=placed, unschedulable=sum(r.Stopped == "Unschedulable" for r in res),
                     decisions_per_s=round(decisions / max((setup + place) * 1e-3, 1e-9)), wall_s=round(wall, 3))


def sample(res):
    pool = [i for i, r in enumerate(res) if r.Replicas < a.check_max]
    return sorted(rng.choice(pool, size=min(a.check, len(pool)), replace=False).tolist()) if pool else []


def check(sim, res, idx, extra_recs, open_local=False, scs=None):
    """res[i] for i in idx against the recompile + resume equivalence; extra_recs: the template PodRecs appended after the session's
    pods (probe i of a template case is extra_recs[i])."""
    p = sim._plan()
    base = list(p.pods) + list(extra_recs)
    placed = np.concatenate([sim.placements, np.full(len(extra_recs), -1, np.int32)])
    ok = 0
    for i in idx:
        r = res[i]
        if extra_recs:
            q = len(p.pods) + i
        else:
            q = headroom.workload_pod(sim.compiled, r.Probe)
        n = r.Replicas + (r.Stopped == "Unschedulable")
        pods = base + [copy.copy(base[q]) for _ in range(n)]
        c2 = compile_cluster(p.nodes, pods, p.ctx, open_local=open_local, storage_classes=scs, local_devices=open_local)
        with Engine(c2) as eng:
            out, _s, fc, _fp = eng.schedule_resume(placed)
            slots = eng.gpu_slot_words()
        tail = out[len(base):]
        names = [c2.node_names[g] for g in tail[:r.Replicas]]
        good = names == r.Nodes and [headroom.gpu_index(int(w)) for w in slots[len(base):len(base) + r.Replicas]] == r.GpuIndex
        if r.Stopped == "Unschedulable":
            good = good and tail[r.Replicas] == -1 and len(fc) >= 1
        ok += bool(good)
    return ok


out = dict(bench="headroom", gpu=gpu, nodes=a.nodes)
rng = np.random.default_rng(7)
cluster, apps = synth.make_c3(n_nodes=a.nodes, n_workloads=a.workloads, n_apps=1, gpu_pct=a.gpu_pct)
with NewSimulator() as sim:
    sim.RunCluster(PrepareCluster(cluster))
    sim.ScheduleApp(apps[0])
    out["pods"] = int(len(sim.placements))
    out["free_pod_slots"] = headroom.free_pod_slots(sim.compiled, sim.placements)
    refs = workload_refs(sim.compiled)
    sim.Headroom(refs[:2], max_replicas=4)                        # warm-up: module load, first launches
    res, out["a_workloads"] = timed(sim, refs, a.workload_cap)
    idx = sample(res)
    out["a_workloads"]["checked"], out["a_workloads"]["equal"] = len(idx), check(sim, res, idx, [])
    print(json.dumps(out["a_workloads"]), file=sys.stderr, flush=True)        # progress: each case as it completes
    _c2, c2_apps = synth.make_c2(n_nodes=100, n_workloads=2 * a.templates, replicas=1)
    shapes = [d for d in c2_apps[0].Resource.Deployments
              if d["spec"]["template"]["spec"]["containers"][0].get("resources", {}).get("requests", {}).get("cpu") not in (None, "0", "0m", 0)]
    tmpls = []
    for j, d in enumerate(shapes[:a.templates]):
        t = d["spec"]["template"]
        tmpls.append({"apiVersion": "v1", "kind": "Pod", "metadata": dict(t.get("metadata") or {}, name=f"probe-{j}", namespace="default"),
                      "spec": copy.deepcopy(t["spec"])})
    res, out["b_templates"] = timed(sim, tmpls, None)
    out["b_templates"]["max_replicas"] = out["free_pod_slots"]
    idx = sample(res)
    out["b_templates"]["checked"] = len(idx)
    out["b_templates"]["equal"] = check(sim, res, idx, [make_valid_pod_by_pod(x) for x in tmpls])
    print(json.dumps(out["b_templates"]), file=sys.stderr, flush=True)
del sim

cluster, apps = synth.make_open_local(n_nodes=a.nodes)
scs = list(cluster.StorageClasss)
with NewSimulator(WithOpenLocal(devices=True)) as sim:
    sim.RunCluster(PrepareCluster(cluster))
    for app in apps:
        sim.ScheduleApp(app)
    st = sim.compiled.storage
    refs = workload_refs(sim.compiled, lambda q: bool(st.class_local[int(sim.compiled.pods["pod_class"][q])]))
    sim.Headroom(refs[:2], max_replicas=4)
    res, out["c_open_local"] = timed(sim, refs, a.workload_cap)
    out["c_open_local"]["kernel"] = sim.last_headroom[0]["launches"][0]["kernel"]
    idx = sample(res)
    out["c_open_local"]["checked"] = len(idx)
    out["c_open_local"]["equal"] = check(sim, res, idx, [], open_local=True, scs=scs + [sc for x in apps for sc in x.Resource.StorageClasss])
print(json.dumps(out))
