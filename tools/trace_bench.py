"""Trace replay on a C3-sized session: one replay on the session's nodes and one sweep over k added nodes, with the per-run cost.

The session is synth.make_c3 (GPU share on about --gpu-pct % of the nodes) after RunCluster and ScheduleApp of its app.  The trace draws --creates pods from the
session's own pod shapes (bare copies of its non-DaemonSet pods' templates), arriving as a Poisson process with exponential lifetimes,
and also deletes --session-deletes of the session's placed pods at uniform times.  Prints one JSON line: the card and its power limit,
compile time, and per batch the runs, launches, device time (setup, runs), wall clock, decisions/s and device time per run; the first
--check events are checked against the CPU trace checker (tests/checkers.c).

  python tools/trace_bench.py [--nodes 10000] [--creates 50000] [--kmax 8]"""
from __future__ import annotations

import argparse
import copy
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "open-simulator_b200"), ROOT, os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)

import numpy as np  # noqa: E402

from simon_b200 import simulator, synth, trace  # noqa: E402
from simon_b200.engine import Engine  # noqa: E402
from simon_b200.scaledown import pod_guard  # noqa: E402


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True, timeout=30)
        return out.strip().splitlines()[0]
    except Exception as e:         # the numbers below still come from the device; say where the card name could not be read
        return f"unknown ({e})"


def make_trace(sim, n_creates, n_session_deletes, rate, mean_life, seed):
    rng = np.random.default_rng(seed)
    c = sim.compiled
    guard = pod_guard(c)
    shapes = [q for q in range(len(c.pod_recs)) if guard[q] < 0 and c.pods["pod_fixed_node"][q] == -1]
    t = np.cumsum(rng.exponential(1.0 / rate, n_creates))
    items = []
    for i in range(n_creates):
        rec = c.pod_recs[int(shapes[int(rng.integers(len(shapes)))])]
        pod = copy.deepcopy(rec.tmpl.pod)
        pod["metadata"]["name"] = f"trace-{i}"
        pod["metadata"].pop("ownerReferences", None)
        pod["spec"].pop("nodeName", None)
        items.append((pod, float(t[i]), float(t[i] + rng.exponential(mean_life))))
    events = trace.from_lifetimes(items)
    horizon = float(t[-1]) if n_creates else 1.0
    placed = [q for q in range(len(sim.placements)) if sim.placements[q] >= 0 and guard[q] < 0]
    gone = rng.choice(len(placed), size=min(n_session_deletes, len(placed)), replace=False)
    dels = sorted((float(rng.uniform(0, horizon)), trace.pod_key(c.pod_recs[placed[int(j)]])) for j in gone)
    merged = [(e.time, 1 if e.op == trace.CREATE else 0, k, e) for k, e in enumerate(events)]
    merged += [(tm, 0, -1, trace.Event(tm, trace.DELETE, key)) for tm, key in dels]
    merged.sort(key=lambda x: x[:3])
    return [m[3] for m in merged]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=10000)
    ap.add_argument("--workloads", type=int, default=1000)
    ap.add_argument("--replicas", type=int, default=100)
    ap.add_argument("--gpu-pct", type=int, default=25)
    ap.add_argument("--creates", type=int, default=50000)
    ap.add_argument("--session-deletes", type=int, default=20000)
    ap.add_argument("--rate", type=float, default=10.0)          # arrivals per time unit
    ap.add_argument("--life", type=float, default=300.0)         # mean lifetime
    ap.add_argument("--kmax", type=int, default=8)
    ap.add_argument("--check", type=int, default=2000)
    ap.add_argument("--seed", type=int, default=11)
    a = ap.parse_args()
    out = dict(card=card())
    cluster, apps = synth.make_c3(n_nodes=a.nodes, n_workloads=a.workloads, replicas=a.replicas, n_apps=1, gpu_pct=a.gpu_pct, seed_no=3)
    sim = simulator.NewSimulator()
    t0 = time.perf_counter()
    sim.RunCluster(cluster)
    sim.ScheduleApp(apps[0])
    out["session_s"] = time.perf_counter() - t0
    events = make_trace(sim, a.creates, a.session_deletes, a.rate, a.life, a.seed)
    spec = copy.deepcopy(cluster.Nodes[0])
    t0 = time.perf_counter()
    ts = trace.build(sim, events, spec, a.kmax)
    out["compile_s"] = time.perf_counter() - t0
    n_ev = len(ts.events)
    out.update(n_nodes=a.nodes, n_session_pods=int(ts.n_prefix), n_events=n_ev, n_creates=int((ts.events[:, 0] == 1).sum()),
               n_deletes=int((ts.events[:, 0] == 2).sum()))
    samples = trace.sample_events(n_ev, 100)
    with Engine(ts.compiled, record_scores=False) as eng:
        for name, scen in (("replay", [ts.scenarios[0].nodes]), ("sweep", [s.nodes for s in ts.scenarios])):
            eng.trace_run(ts.placed, ts.n_prefix, ts.events, scen[:1], samples=samples, detail=False)      # warm-up: module load, pools
            t0 = time.perf_counter()
            raw = eng.trace_run(ts.placed, ts.n_prefix, ts.events, scen, samples=samples, detail=name == "replay")
            wall = time.perf_counter() - t0
            lt = eng.last_trace
            creates = out["n_creates"] * len(scen)
            out[name] = dict(scenarios=len(scen), chunks=lt["chunks"], runs=lt["runs"], launches=lt["run_launches"],
                             setup_ms=round(lt["setup_ms"], 3), run_ms=round(lt["place_ms"], 3), wall_s=round(wall, 3),
                             decisions_per_s=round(creates / max(lt["place_ms"] * 1e-3, 1e-9)),
                             us_per_run=round(lt["place_ms"] * 1e3 / max(lt["runs"], 1), 2),
                             failed=[int(r["n_unscheduled"]) for r in raw], removed=[int(r["n_removed"]) for r in raw],
                             kernel=lt["launches"][-1]["kernel"] if lt["launches"] else "")
            if name == "replay":
                first = raw[0]
    if a.check:
        import checkers
        from oracle.binding import Oracle
        ev = ts.events[:a.check]
        o = Oracle(ts.compiled)
        w = checkers.trace(o, ts.placed, ts.n_prefix, ts.scenarios[0].nodes, ev)
        created = ev[ev[:, 0] == 1][:, 1].astype(np.int64) - ts.n_prefix
        bad = int((first["node"][created] != w["node"][created]).sum() + (first["gpu_slots"][created] != w["gpu_slots"][created]).sum())
        out["check"] = dict(events=int(len(ev)), creates=int(len(created)), mismatches=bad)
        o.close()
    print(json.dumps(out))
    if out.get("check", {}).get("mismatches"):
        sys.exit(1)


if __name__ == "__main__":
    main()
