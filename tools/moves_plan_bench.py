"""Migration-plan timing (simon_moves_plan).

C5: 1M sampled candidate moves on a 10k-node live snapshot with 300k running pods, a plan of up to 1,000 steps; the device time per
step next to simon_moves_replay's time per scoring pass on the same list (the difference is the apply kernel and the step loop), and
the first steps against the CPU checker (its time per step is the CPU baseline).  C3 session: candidates from the 200 most-utilised
nodes of a placed C3 cluster onto every node."""
import argparse
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "open-simulator_b200"), ROOT, os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import numpy as np
from simon_b200 import moves as M, rebalance, scaledown, simulator, synth
from simon_b200.compiler import compile_cluster
from simon_b200.engine import Engine

ap = argparse.ArgumentParser()
ap.add_argument("--nodes", type=int, default=10000)
ap.add_argument("--running", type=int, default=300000)
ap.add_argument("--moves", type=int, default=1000000)
ap.add_argument("--max-moves", type=int, default=1000)
ap.add_argument("--check", type=int, default=20, help="plan steps compared with the CPU checker")
ap.add_argument("--c3-nodes", type=int, default=10000)
ap.add_argument("--c3-sources", type=int, default=200)
a = ap.parse_args()


def steps_of(r):
    s = r["steps"]
    return np.stack([s["move"], s["pod"], s["from"], s["to"], s["gain"], s["gpu_slots"]], 1).astype(np.int64)


t0 = time.time()
cluster, apps = synth.make_c3(n_nodes=a.nodes, n_workloads=max(10, a.nodes // 10), replicas=10, n_apps=10, seed_no=3)
p = simulator.plan(cluster, apps)
c = compile_cluster(p.nodes, p.pods, p.ctx)
live = synth.make_c5(c, a.running)
print(f"C5 snapshot: {live.n_nodes} nodes, {live.pods_dims['n_pods']} running pods, built in {time.time() - t0:.1f} s", flush=True)
with Engine(live, device=0) as eng:
    out = eng.schedule()[0]
    mv = M.sample_moves(len(out), live.n_nodes, a.moves, seed=11, placement=out)
    eng.moves_upload(mv, 0)
    eng.moves_replay(3)
    pass_ms = eng.moves_replay(20) / 20
    eng.moves_plan(10, 1)                   # warm-up
    t1 = time.perf_counter()
    r = eng.moves_plan(a.max_moves, 1)
    wall = time.perf_counter() - t1
    n = len(r["steps"])
    print(f"C5 plan: {n} steps (stop {rebalance.STOP_REASONS[r['stop_reason']]}), device {r['kernel_ms']:.1f} ms = "
          f"{r['kernel_ms'] / max(n, 1) * 1e3:.1f} us per step, wall {wall * 1e3:.1f} ms; one scoring pass (simon_moves_replay) "
          f"{pass_ms * 1e3:.1f} us -> apply + loop {(r['kernel_ms'] / max(n, 1) - pass_ms) * 1e3:.1f} us per step; "
          f"gains {int(r['steps']['gain'][0]) if n else None} .. {int(r['steps']['gain'][-1]) if n else None}", flush=True)
    if a.check:
        import checkers
        from oracle.binding import Oracle
        o = Oracle(live)
        o.schedule()
        t2 = time.perf_counter()
        ref = checkers.plan(o, mv, out, o.gpu_slot_words(), a.check)
        cpu = time.perf_counter() - t2
        same = np.array_equal(ref["steps"], steps_of(r)[:a.check])
        print(f"C5 checker: first {a.check} steps identical: {same}; CPU checker {cpu / a.check * 1e3:.0f} ms per step", flush=True)
        o.close()

t0 = time.time()
cluster, apps = synth.make_c3(n_nodes=a.c3_nodes, n_workloads=max(10, a.c3_nodes // 10), replicas=100, n_apps=2, seed_no=3)
with simulator.NewSimulator() as sim:
    sim.RunCluster(simulator.PrepareCluster(cluster))
    for app in apps:
        sim.ScheduleApp(app)
    eng, c3 = sim._live()
    util = scaledown.node_utilisation(c3, sim.placements)
    busy = np.argsort(-util, kind="stable")[:a.c3_sources]
    mv = rebalance.candidates(c3, sim.placements, sources=busy.tolist())
    print(f"C3 session: {c3.n_nodes} nodes, {int((sim.placements >= 0).sum())} placed pods, {len(mv)} candidates from the "
          f"{a.c3_sources} most-utilised nodes, set up in {time.time() - t0:.1f} s", flush=True)
    eng.moves_upload(mv, 0)
    pass_ms = eng.moves_replay(5) / 5
    t1 = time.perf_counter()
    mp = sim.PlanMigrations(sources=[c3.node_names[g] for g in busy], max_moves=a.max_moves)
    wall = time.perf_counter() - t1
    n = len(mp.Migrations)
    print(f"C3 plan: {n} migrations (stop {mp.StopReason}), device {mp.KernelMs:.1f} ms = {mp.KernelMs / max(n, 1) * 1e3:.1f} us per "
          f"step, one scoring pass {pass_ms * 1e3:.1f} us; PlanMigrations wall {wall * 1e3:.0f} ms (candidates + upload + plan)", flush=True)
