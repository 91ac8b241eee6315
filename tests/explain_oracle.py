"""Expected explained-decision records (simon_explain_set) from the CPU oracle's per-pod detail (TEST INFRASTRUCTURE ONLY).

record(...) builds one record from one pod's detail: the feasible count F, the histogram of the per-node reason bits over the active
nodes, and the best min(top_k, F) feasible nodes by (total descending, node order) with their ten words; with F == 1 the one node and
all words 0.  expected(...) runs the oracle pod by pod and calls it for every explained pod; assert_records_equal compares the
engine's records (Engine.explanations) with them."""
from __future__ import annotations

import numpy as np

import checkers
from simon_b200 import abi


def record(node: int, reached: bool, reasons, detail, top_k: int, order=None) -> dict:
    """One pod's record.  node: its out_node; reached: it went through the scheduler (else nothing else is recorded); reasons [N]: the
    filter verdict bitmask of every node (0 feasible); detail [N][10]: the oracle's score words of the feasible nodes; order: the active
    nodes in scenario order (None: every node in index order)."""
    rejected = np.zeros(abi.N_FAIL_CODES, np.uint32)
    if not reached:
        return dict(node=int(node), feasible=0, rejected=rejected, top=[])
    reasons = np.asarray(reasons, np.uint32)
    order = np.arange(len(reasons)) if order is None else np.asarray(order)
    for b in range(abi.N_FAIL_CODES):
        rejected[b] = int(((reasons[order] >> b) & 1).sum())
    feas = [int(n) for n in order if reasons[n] == 0]
    F = len(feas)
    if F == 1:
        top = [(feas[0], [0] * abi.EXPLAIN_WORDS)]
    else:
        rank = {n: r for r, n in enumerate(feas)}
        best = sorted(feas, key=lambda n: (-int(detail[n][8]), rank[n]))[:top_k]
        top = [(n, [int(x) for x in detail[n]]) for n in best]
    return dict(node=int(node), feasible=F, rejected=rejected, top=top)


def expected(c, pods, top_k: int, open_local: bool = False, threads: int = 1) -> list:
    """The records of a full run of compiled cluster c from the empty state in which the ascending pod indices `pods` are explained."""
    from oracle.binding import Oracle
    o = Oracle(c, threads=threads, open_local=open_local)
    o.enable_dump()
    fixed = c.pods["pod_fixed_node"]
    out, pos = [], 0
    for q in pods:
        q = int(q)
        if q > pos:
            o.schedule(pos, q - pos)
        node = int(o.schedule(q, 1)[0][0])
        reached = fixed[q] == -1 and node != -3
        reasons = detail = None
        if reached:
            reasons = checkers.last_reasons(o)
            _code, detail = o.last_detail()
        out.append(record(node, reached, reasons, detail, top_k))
        pos = q + 1
    o.close()
    return out


def assert_records_equal(rec, nodes, want, pods, what=""):
    """Engine.explanations() (rec, nodes) against expected(...) for the same pods."""
    assert len(rec) == len(want), what
    for i, (r, w) in enumerate(zip(rec, want)):
        at = f"{what} record {i} (pod {pods[i]})"
        assert (int(r["node"]), int(r["feasible"])) == (w["node"], w["feasible"]), f"{at}: {r['node'], r['feasible']} != {w['node'], w['feasible']}"
        np.testing.assert_array_equal(r["rejected"], w["rejected"], err_msg=at)
        assert int(r["n_top"]) == len(w["top"]), at
        got = [(int(x["node"]), [int(v) for v in x["words"]]) for x in nodes[i][:len(w["top"])]]
        assert got == w["top"], f"{at}: {got} != {w['top']}"


def static_mix(seed_no: int = 104, n_nodes: int = 80, n_workloads: int = 40):
    """make_mix with container images, preferAvoidPods annotations on every third node naming the controllers of two of its
    ReplicaSets, and one host-side extra score plugin: every part of the static row (word 7) varies across nodes.  -> (plan, compiled,
    plugins)."""
    import json

    from simon_b200 import objects as O
    from simon_b200 import simulator, synth
    from simon_b200.compiler import ExtraScorePlugin, compile_cluster
    cluster, apps = synth.make_mix(seed_no=seed_no, n_nodes=n_nodes, n_workloads=n_workloads, max_replicas=6, with_images=True)
    # pods controlled by a ReplicaSet with a uid, which the annotations name (the generated workloads' ReplicaSets carry none)
    for j in range(8):
        apps[0].Resource.Pods.append({"kind": "Pod", "metadata": {"name": f"avoided-{j}", "namespace": "default", "ownerReferences": [
            {"kind": "ReplicaSet", "name": "avoided", "uid": "rs-avoided", "controller": True}]},
            "spec": {"containers": [{"name": "c", "image": "nginx", "resources": {"requests": {"cpu": "100m", "memory": "128Mi"}}}]}})
    p = simulator.plan(cluster, apps)
    ann = json.dumps({"preferAvoidPods": [{"podSignature": {"podController": {"kind": "ReplicaSet", "uid": "rs-avoided", "name": "avoided"}}}]})
    for i, n in enumerate(p.nodes):
        if i % 3 == 0:
            n.setdefault("metadata", {}).setdefault("annotations", {})["scheduler.alpha.kubernetes.io/preferAvoidPods"] = ann
    plugins = [ExtraScorePlugin("NameParity", 2, lambda pod, node: 100 if sum(map(ord, O.name_of(node))) % 2 == 0 else 30)]
    c = compile_cluster(p.nodes, p.pods, p.ctx, extra_plugins=plugins)
    return p, c, plugins
