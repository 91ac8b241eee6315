"""PodDisruptionBudget cost in migration plans and drain sweeps (simon_pdbs_upload).

C5 plan: 1M sampled candidate moves on a 10k-node live snapshot with 300k running pods, a plan of up to 1,000 steps with no table and
with one PDB per workload (here: per pod class, maxUnavailable 1, and a "25%" variant), alternated on the same list; per-step device
time, stop reason, blocked and exhausted counts, and the first steps against the CPU checker.  C3 sweep: every single-node drain of a
placed 10k-node C3 cluster with and without the same kind of PDBs (per workload: app label); setup, placement and host time, and how
many drains the PDBs make non-drainable.  Prints one JSON line per measurement; writes nothing."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "open-simulator_b200"), ROOT, os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import numpy as np
from simon_b200 import disruption, moves as M, rebalance, scaledown, simulator, synth
from simon_b200.compiler import compile_cluster
from simon_b200.disruption import PdbTables
from simon_b200.engine import Engine

ap = argparse.ArgumentParser()
ap.add_argument("--nodes", type=int, default=10000)
ap.add_argument("--running", type=int, default=300000)
ap.add_argument("--moves", type=int, default=1000000)
ap.add_argument("--max-moves", type=int, default=1000)
ap.add_argument("--check", type=int, default=20, help="plan steps compared with the CPU checker")
ap.add_argument("--repeats", type=int, default=3)
ap.add_argument("--sweep-nodes", type=int, default=10000)
a = ap.parse_args()


def per_class_table(cls, form):
    """One PDB per pod class of a live snapshot: maxUnavailable 1 or "25%"."""
    n = int(cls.max()) + 1
    cnt = np.bincount(cls, minlength=n)
    spec = {"maxUnavailable": 1} if form == "1" else {"maxUnavailable": "25%"}
    desired = np.array([disruption.desired_of(spec, int(k)) for k in cnt], np.int32)
    return PdbTables(names=[f"class-{k}" for k in range(n)], pod_off=np.arange(len(cls) + 1, dtype=np.uint32),
                     pod_pdb=np.asarray(cls, np.uint32), desired=desired)


t0 = time.time()
cluster, apps = synth.make_c3(n_nodes=a.nodes, n_workloads=max(10, a.nodes // 10), replicas=10, n_apps=10, seed_no=3)
p = simulator.plan(cluster, apps)
c = compile_cluster(p.nodes, p.pods, p.ctx)
live = synth.make_c5(c, a.running)
cls = live.pods["pod_class"]
tables = {"none": None, "max1": per_class_table(cls, "1"), "max25pct": per_class_table(cls, "25%")}
with Engine(live, device=0) as eng:
    out = eng.schedule()[0]
    mv = M.sample_moves(len(out), live.n_nodes, a.moves, seed=11, placement=out)
    eng.moves_upload(mv, 0)
    eng.moves_plan(10, 1)                   # warm-up
    res = {k: [] for k in tables}
    for _ in range(a.repeats):
        for k, t in tables.items():
            eng.pdbs_upload(t)
            allowed = eng.pdbs_allowed() if t is not None else None
            r = eng.moves_plan(a.max_moves, 1)
            n = len(r["steps"])
            res[k].append(dict(steps=n, us_per_step=r["kernel_ms"] / max(n, 1) * 1e3, stop=rebalance.STOP_REASONS[r["stop_reason"]],
                               blocked=r["pdb_blocked"],
                               exhausted=len(disruption.exhausted(t, allowed, r["steps"]["pod"])) if t is not None else 0))
            if k != "none" and a.check and _ == 0:
                import checkers
                from oracle.binding import Oracle
                o = Oracle(live)
                o.schedule()
                ref = checkers.plan_pdb(o, mv, out, o.gpu_slot_words(), a.check, 1, 0, t.pod_off, t.pod_pdb, allowed)
                o.close()
                s = r["steps"][:a.check]
                got = np.stack([s["move"], s["pod"], s["from"], s["to"], s["gain"], s["gpu_slots"]], 1).astype(np.int64)
                res[k][-1]["checked_steps"] = int(len(ref["steps"]))
                res[k][-1]["checker_equal"] = bool(np.array_equal(got, ref["steps"][:len(got)]))
    for k, v in res.items():
        print(json.dumps(dict(what="c5_plan", table=k, nodes=live.n_nodes, pods=int(live.pods_dims["n_pods"]), moves=len(mv),
                              us_per_step=[round(x["us_per_step"], 1) for x in v], **{q: v[0][q] for q in v[0] if q != "us_per_step"})),
              flush=True)

# ---- C3 sweep of every single-node drain ----
cluster, apps = synth.make_c3(n_nodes=a.sweep_nodes, n_workloads=max(10, a.sweep_nodes // 10), replicas=10, n_apps=10, seed_no=3)
p = simulator.plan(cluster, apps)
c = compile_cluster(p.nodes, p.pods, p.ctx)
wl = sorted({(r.tmpl.namespace or "default", r.tmpl.labels.get("app")) for r in c.pod_recs if r.tmpl.labels.get("app")})
for form in ("1", "25%"):
    objs = [{"metadata": {"name": f"pdb-{a_}", "namespace": ns}, "spec": {"selector": {"matchLabels": {"app": a_}}, "maxUnavailable": form if form.endswith("%") else 1}}
            for ns, a_ in wl]
    t = disruption.compile_pdbs(objs, c)
    order = scaledown.NodeOrder(c)
    remain = [order.remaining([g]) for g in range(c.n_nodes)]
    with Engine(c, device=0) as eng:
        out = eng.schedule()[0]
        for k, tab in (("none", None), (f"max{form}", t)):
            eng.pdbs_upload(tab)
            h0 = time.perf_counter()
            r = eng.drain_run(out, remain, detail=False)
            host = time.perf_counter() - h0
            info = eng.last_drain
            print(json.dumps(dict(what="c3_sweep", table=k, nodes=c.n_nodes, drains=len(remain), setup_ms=round(info["setup_ms"], 2),
                                  place_ms=round(info["place_ms"], 2), wall_s=round(host, 3),
                                  drainable=sum(scaledown.drainable(x) for x in r),
                                  pdb_violating=sum(x["n_pdb_violated"] > 0 for x in r))), flush=True)
