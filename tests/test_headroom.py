"""Scheduling headroom probes (simon_probe_run, Engine.probe_run, simon_b200.headroom, Simulator.Headroom).

CPU: the probe checker (tests/checkers.c) on hand-derived answers with their exact FitError texts, the host's refusals through a
fake runner, the compiler's per-class pod limit against its own guards, and the variant tables.  GPU: every probe kernel variant against
the checker, probes against the recompile + simon_schedule_resume equivalence that pins the definition, the context state a probe batch
leaves, chunking, the C-entry refusals and the session end to end."""
import copy

import pytest

from simon_b200 import abi, compiler, headroom, objects as O, simulator
from simon_b200.compiler import compile_cluster
from util import compiled_kernels


def _node(name, mcpu="4000m", pods="110", zone=None, gpu=None):
    labels = {"kubernetes.io/hostname": name}
    if zone:
        labels["topology.kubernetes.io/zone"] = zone
    al = {"cpu": mcpu, "memory": "16Gi", "pods": pods}
    if gpu:
        al.update({"alibabacloud.com/gpu-count": str(gpu[0]), "alibabacloud.com/gpu-mem": gpu[1]})
    return {"apiVersion": "v1", "kind": "Node", "metadata": {"name": name, "labels": labels},
            "status": {"allocatable": dict(al), "capacity": dict(al)}}


def _dep(name, n, cpu="1000m", extra=None, ann=None):
    spec = {"containers": [{"name": "c", "image": "nginx", "resources": {"requests": {"cpu": cpu, "memory": "1Gi"}}}]}
    spec.update(extra or {})
    meta = {"labels": {"app": name}}
    if ann:
        meta["annotations"] = ann
    return {"apiVersion": "apps/v1", "kind": "Deployment", "metadata": {"name": name, "namespace": "default"},
            "spec": {"replicas": n, "selector": {"matchLabels": {"app": name}}, "template": {"metadata": meta, "spec": spec}}}


ANTI = {"affinity": {"podAntiAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": [
    {"labelSelector": {"matchLabels": {"app": "anti"}}, "topologyKey": "kubernetes.io/hostname"}]}}}
SPREAD = {"topologySpreadConstraints": [{"maxSkew": 1, "topologyKey": "topology.kubernetes.io/zone", "whenUnsatisfiable": "DoNotSchedule",
                                         "labelSelector": {"matchLabels": {"app": "sp"}}}]}
GPU_ANN = {"alibabacloud.com/gpu-mem": "8Gi", "alibabacloud.com/gpu-count": "1"}

# name -> (nodes, deployments, probed workload, max_replicas, replicas placed, FitError text after "nodes are available: " or None)
KNOWN = {
    # 4 x 4000m holding eight 1000m pods: 8 more fit, two per node
    "cpu": ([_node(f"node-{i}") for i in range(4)], [_dep("web", 8)], "Deployment/default/web", 20, 8, "4 Insufficient cpu."),
    # required hostname anti-affinity on its own label: the 2 live replicas occupy 2 of the 4 nodes
    "anti": ([_node(f"node-{i}") for i in range(4)], [_dep("anti", 2, extra=ANTI)], "Deployment/default/anti", 20, 2,
             "4 node(s) didn't match pod affinity/anti-affinity, 4 node(s) didn't match pod anti-affinity rules."),
    # hard zone spread, maxSkew 1: zone a (2 nodes, 8 pods of cpu) may hold at most zone b's count + 1 = 5, zone b (1 node) 4;
    # the live replica is in zone a: (5 - 1) + 4 = 8
    "spread": ([_node("node-0", zone="a"), _node("node-1", zone="a"), _node("node-2", zone="b")], [_dep("sp", 1, extra=SPREAD)],
               "Deployment/default/sp", 40, 8, "1 Insufficient cpu, 2 node(s) didn't match pod topology spread constraints."),
    # GPU share: 2 devices of 16Gi on node-0, 8Gi per replica, one live: 3 more
    "gpu": ([_node("node-0", gpu=(2, "32Gi")), _node("node-1")], [_dep("g", 1, cpu="100m", ann=GPU_ANN)], "Deployment/default/g", 20, 3,
            "2 Node:<2 nodes rejected by Open-Gpu-Share>."),
    # the pod-count limit: 2 nodes of 3 pods, one live
    "pods": ([_node(f"node-{i}", pods="3") for i in range(2)], [_dep("small", 1, cpu="10m")], "Deployment/default/small", 20, 5,
             "2 Too many pods."),
    # a cap reached
    "cap": ([_node(f"node-{i}") for i in range(4)], [_dep("web", 8)], "Deployment/default/web", 3, 3, None),
}


def _case(name):
    nodes, deps, ref, R, want_k, want_text = KNOWN[name]
    cluster = O.ResourceTypes(Nodes=nodes)
    apps = [O.AppResource("a", O.ResourceTypes(Deployments=deps))]
    return cluster, apps, ref, R, want_k, want_text


class CheckerEngine:
    """Engine.probe_run on the CPU: the probe checker from an oracle's live placement, plus the occupancy sums of its end state."""

    def __init__(self, c):
        from oracle.binding import Oracle
        self.c = c
        self.o = Oracle(c)
        self.calls = []

    def probe_run(self, placed, probes, detail=True):
        import checkers
        self.calls.append(list(probes))
        out = []
        for q, r in probes:
            d = checkers.probe(self.o, placed, q, r)
            st = self.o.state()
            d.update(req_mcpu=int(st["req_mcpu"].sum()), alloc_mcpu=int(self.c.snap["alloc_mcpu"].sum()),
                     req_mem=int(st["req_mem"].sum()), alloc_mem=int(self.c.snap["alloc_mem"].sum()))
            out.append(d)
        return out


def _live(cluster, apps):
    from oracle.binding import Oracle
    p = simulator.plan(cluster, apps)
    c = compile_cluster(p.nodes, p.pods, p.ctx)
    return p, c, Oracle(c).schedule()[0]


# ---- CPU --------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", sorted(KNOWN))
def test_known_answer_through_the_checker(name):
    cluster, apps, ref, R, want_k, want_text = _case(name)
    _p, c, placed = _live(cluster, apps)
    eng = CheckerEngine(c)
    q = headroom.workload_pod(c, ref)
    res = headroom.run(eng, c, placed, [(ref, q, R)])[0]
    assert res.Replicas == want_k and len(res.Nodes) == want_k
    if want_text is None:
        assert res.Stopped == "MaxReplicas" and res.Reason is None
    else:
        assert res.Stopped == "Unschedulable"
        assert res.Reason == f"failed to schedule pod ({c.pod_recs[q].tmpl.namespace}/{c.pod_recs[q].name}): Unschedulable: " \
                             f"0/{c.n_nodes} nodes are available: {want_text}"


def test_known_answer_nodes_and_gpu_index():
    for name, nodes, idx in (("cpu", ["node-0", "node-1", "node-2", "node-3"] * 2, [None] * 8),
                             ("anti", ["node-2", "node-3"], [None, None]),
                             ("gpu", ["node-0"] * 3, ["0", "1", "1"])):
        cluster, apps, ref, R, _k, _t = _case(name)
        _p, c, placed = _live(cluster, apps)
        res = headroom.run(CheckerEngine(c), c, placed, [(ref, headroom.workload_pod(c, ref), R)])[0]
        assert (res.Nodes, res.GpuIndex) == (nodes, idx), name
    cluster, apps, ref, R, _k, _t = _case("cpu")
    _p, c, placed = _live(cluster, apps)
    res = headroom.run(CheckerEngine(c), c, placed, [(ref, 0, R)])[0]
    assert res.Occupancy == dict(req_mcpu=16000, alloc_mcpu=16000, req_mem=16 << 30, alloc_mem=64 << 30)


def test_free_pod_slots_default_cap():
    cluster, apps, *_ = _case("pods")
    _p, c, placed = _live(cluster, apps)
    assert headroom.free_pod_slots(c, placed) == 5            # 2 x 3 slots, one taken


def test_workload_references():
    cluster, apps, *_ = _case("anti")
    _p, c, _placed = _live(cluster, apps)
    assert headroom.workload_pod(c, "Deployment/default/anti") == headroom.workload_pod(c, "ReplicaSet/default/anti") == 0
    with pytest.raises(ValueError, match="no workload"):
        headroom.workload_pod(c, "Deployment/default/nope")
    with pytest.raises(ValueError, match="not a workload reference"):
        headroom.workload_pod(c, "anti")


def _mixed_cluster():
    """A DaemonSet, a pod bound by spec.nodeName and a Deployment on 3 nodes."""
    cluster = O.ResourceTypes(Nodes=[_node(f"node-{i}") for i in range(3)])
    ds = {"apiVersion": "apps/v1", "kind": "DaemonSet", "metadata": {"name": "agent", "namespace": "kube-system"},
          "spec": {"selector": {"matchLabels": {"app": "agent"}}, "template": {"metadata": {"labels": {"app": "agent"}},
                   "spec": {"containers": [{"name": "c", "image": "x", "resources": {"requests": {"cpu": "100m"}}}]}}}}
    bound = {"apiVersion": "v1", "kind": "Pod", "metadata": {"name": "static", "namespace": "default"},
             "spec": {"nodeName": "node-1", "containers": [{"name": "c", "image": "x", "resources": {"requests": {"cpu": "100m"}}}]}}
    cluster.DaemonSets.append(ds)
    cluster.Pods.append(bound)
    return cluster, [O.AppResource("a", O.ResourceTypes(Deployments=[_dep("web", 2)]))]


def test_host_refusals_before_the_runner():
    cluster, apps = _mixed_cluster()
    p, c, placed = _live(cluster, apps)
    eng = CheckerEngine(c)
    fixed = c.pods["pod_fixed_node"]
    ds = next(q for q, r in enumerate(c.pod_recs) if r.tmpl.workload_kind == "DaemonSet")
    bound = next(q for q in range(len(fixed)) if fixed[q] >= 0)
    web = headroom.workload_pod(c, "Deployment/default/web")
    with pytest.raises(ValueError, match="DaemonSet"):
        headroom.run(eng, c, placed, [("ds", ds, 3)])
    with pytest.raises(ValueError, match="spec.nodeName"):
        headroom.run(eng, c, placed, [("bound", bound, 3)])
    with pytest.raises(ValueError, match="at least 1"):
        headroom.run(eng, c, placed, [("web", web, 0)])
    c.class_pod_limit = list(c.class_pod_limit)
    c.class_pod_limit[int(c.pods["pod_class"][web])] = len(p.pods) + 4
    with pytest.raises(ValueError, match="int32 bounds"):
        headroom.run(eng, c, placed, [("web", web, 3), ("web", web, 5)])
    assert eng.calls == []                                    # every refusal came before the runner
    assert headroom.run(eng, c, placed, [("web", web, 4)])[0].Replicas == 4


def test_session_refusals_without_a_device():
    sim = simulator.NewSimulator()
    with pytest.raises(RuntimeError, match="RunCluster"):
        sim.Headroom(["Deployment/default/web"])


SOFT = {"topologySpreadConstraints": [{"maxSkew": 1, "topologyKey": "kubernetes.io/hostname", "whenUnsatisfiable": "ScheduleAnyway",
                                       "labelSelector": {"matchLabels": {"app": "soft"}}}]}


def _pods_of_length(p, n):
    """p's pod list cut or extended (copies of its last pod) to n pods."""
    pods = list(p.pods[:n])
    while len(pods) < n:
        pods.append(copy.copy(p.pods[-1]))
    return pods


def test_class_pod_limit_is_the_spread_guard(monkeypatch):
    # the ScheduleAnyway bound pods x multiplicity x ln(N + 2 + ...) < PTS_COUNTS_MAX, lowered so that a few hundred pods reach it
    monkeypatch.setattr(compiler, "PTS_COUNTS_MAX", 1000)
    cluster = O.ResourceTypes(Nodes=[_node(f"node-{i}") for i in range(6)])
    p = simulator.plan(cluster, [O.AppResource("a", O.ResourceTypes(Deployments=[_dep("soft", 4, cpu="10m", extra=SOFT)]))])
    c = compile_cluster(p.nodes, p.pods, p.ctx)
    lim = c.class_pod_limit[int(c.pods["pod_class"][0])]
    assert len(p.pods) <= lim < 1000
    c2 = compile_cluster(p.nodes, _pods_of_length(p, lim), p.ctx)
    assert c2.class_pod_limit[int(c2.pods["pod_class"][0])] == lim
    with pytest.raises(compiler.CompileError, match="topology spread"):
        compile_cluster(p.nodes, _pods_of_length(p, lim + 1), p.ctx)


def test_class_pod_limit_is_the_affinity_guard():
    w = 77
    pref = {"affinity": {"podAffinity": {"preferredDuringSchedulingIgnoredDuringExecution": [
        {"weight": w, "podAffinityTerm": {"labelSelector": {"matchLabels": {"app": "aff"}}, "topologyKey": "kubernetes.io/hostname"}}]}}}
    cluster = O.ResourceTypes(Nodes=[_node(f"node-{i}") for i in range(3)])
    p = simulator.plan(cluster, [O.AppResource("a", O.ResourceTypes(Deployments=[_dep("aff", 3, cpu="10m", extra=pref)]))])
    c = compile_cluster(p.nodes, p.pods, p.ctx)
    lim = c.class_pod_limit[int(c.pods["pod_class"][0])]
    # the class scores its own preferred term and, matching its own selector, the same term of its existing pods: weight 2w
    assert lim == ((1 << 31) - 1) // (2 * w)
    assert compiler._ipa_bound_ok(lim, 2 * w) and not compiler._ipa_bound_ok(lim + 1, 2 * w)
    _p, plain, _placed = _live(*_case("cpu")[:2])
    assert set(plain.class_pod_limit) == {compiler.POD_LIMIT_NONE}     # no bound applies without those tables


PROBE_VARIANTS = {
    # kernel -> (CTAs per scenario, threads per CTA, force_large)
    "simon_probe_kernel_256": (2, 128, False),
    "simon_probe_kernel_320": (2, 288, False),
    "simon_probe_kernel_384": (1, 352, False),
    "simon_probe_kernel_big": (4, 64, True),
}
PROBE_LOCAL_VARIANTS = {
    "simon_probe_local_kernel_256": (2, 128, False),
    "simon_probe_local_kernel_320": (2, 288, False),
    "simon_probe_local_kernel_384": (1, 352, False),
    "simon_probe_local_kernel_big": (4, 64, True),
}


def test_probe_variant_tables_name_every_probe_kernel():
    assert set(PROBE_VARIANTS) == compiled_kernels("simon_probe_kernel_")
    assert set(PROBE_LOCAL_VARIANTS) == compiled_kernels("simon_probe_local_kernel_")


def test_abi_restates_the_probe_entry_points():
    assert abi.PROBE_STOP_UNSCHEDULABLE == 1 and abi.PROBE_STOP_MAX_REPLICAS == 2
    assert {"simon_probe_run", "simon_probe_download", "simon_probe_times"} <= set(abi.SIGNATURES)
