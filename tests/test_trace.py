"""Trace replay (simon_trace_run, Engine.trace_run, simon_b200.trace, Simulator.ReplayTrace) on the CPU.

The replay (trace.build + trace.replay) runs here on the trace checker (tests/checkers.c), which applies one event at a time with the
oracle's own primitives, on hand-derived cases: a delete that frees room for a later create, required anti-affinity unblocked by
deleting the peer, spread skew falling after deletes, a GPU-share device freed and reused, a host port freed, extended resources, a
deleted pre-bound pod; the host refusals; and the ordering rule of trace.from_lifetimes."""
import numpy as np
import pytest

from simon_b200 import abi, objects as O, trace
from simon_b200.objects import ResourceTypes

from test_grow import session


def _node(name, mcpu="4000m", zone=None, gpu=None, extra=None):
    labels = {"kubernetes.io/hostname": name}
    if zone:
        labels["topology.kubernetes.io/zone"] = zone
    al = {"cpu": mcpu, "memory": "16Gi", "pods": "110"}
    if gpu:
        al.update({"alibabacloud.com/gpu-count": str(gpu[0]), "alibabacloud.com/gpu-mem": gpu[1]})
    al.update(extra or {})
    return {"apiVersion": "v1", "kind": "Node", "metadata": {"name": name, "labels": labels},
            "status": {"allocatable": dict(al), "capacity": dict(al)}}


def _pod(name, cpu="1000m", labels=None, ann=None, extra=None, node=None, limits=None):
    res = {"requests": {"cpu": cpu, "memory": "1Gi"}}
    if limits:
        res["requests"].update(limits)
        res["limits"] = dict(limits)
    spec = {"containers": [{"name": "c", "image": "nginx", "resources": res}]}
    spec.update(extra or {})
    if node:
        spec["nodeName"] = node
    meta = {"name": name, "namespace": "default", "labels": dict(labels or {"app": name})}
    if ann:
        meta["annotations"] = dict(ann)
    return {"apiVersion": "v1", "kind": "Pod", "metadata": meta, "spec": spec}


class CheckerEngine:
    """Engine.trace_run on the CPU: the trace checker per scenario, with the samples it records after every event."""

    def __init__(self, c):
        from oracle.binding import Oracle
        self.c = c
        self.o = Oracle(c)

    def trace_run(self, placed, n_prefix, events, scenarios=None, samples=None, detail=True, chunk=None):
        import checkers
        out = []
        for nodes in scenarios:
            r = checkers.trace(self.o, placed, n_prefix, nodes, events)
            idx = np.asarray([] if samples is None else samples, np.int64)
            pts = np.zeros(len(idx), abi.TRACE_POINT_DTYPE)
            pts["event"] = idx
            for f, v in r.pop("samples").items():
                pts[f] = v[idx]
            r["samples"] = pts
            out.append(r)
        return out


def replay(cluster, events, new_node=None, kmax=0, samples=100):
    sim = session(cluster)
    ts = trace.build(sim, events, new_node, kmax)
    return ts, trace.replay(CheckerEngine(ts.compiled), ts, samples)


def ev(*items):
    """(time, op, pod) triples -> Events."""
    return [trace.Event(t, op, p) for t, op, p in items]


C, D = trace.CREATE, trace.DELETE


def test_delete_frees_room_for_a_later_create():
    cluster = ResourceTypes(Nodes=[_node("n0")], Pods=[_pod("old", "3000m")])
    ts, r = replay(cluster, ev((1, C, _pod("a", "2000m")), (2, D, "default/old"), (3, C, _pod("b", "2000m"))))
    k0 = r.PerK[0]
    assert [u.Pod.name for u in k0.Failures] == ["a"] and k0.FirstFailureTime == 1
    assert "Insufficient cpu" in k0.Failures[0].Reason
    assert k0.Deletes == 1 and k0.Creates == 2
    assert [(p.Pod.name, p.Node) for p in r.Pods] == [("a", None), ("b", "n0")]
    assert r.MinNodes == -1
    # the samples: running pods and requested cpu after each event
    s = k0.Samples
    assert s["n_running"].tolist() == [1, 0, 1] and s["n_failed"].tolist() == [1, 1, 1]
    assert s["req_mcpu"].tolist() == [3000, 0, 2000] and s["time"].tolist() == [1, 2, 3]


def test_required_anti_affinity_unblocked_by_deleting_the_peer():
    anti = {"affinity": {"podAntiAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": [
        {"labelSelector": {"matchLabels": {"app": "anti"}}, "topologyKey": "kubernetes.io/hostname"}]}}}
    cluster = ResourceTypes(Nodes=[_node("n0")], Pods=[_pod("peer", "100m", labels={"app": "anti"}, extra=anti)])
    _, r = replay(cluster, ev((1, C, _pod("x1", "100m", labels={"app": "anti"}, extra=anti)), (2, D, "default/peer"),
                              (3, C, _pod("x2", "100m", labels={"app": "anti"}, extra=anti))))
    assert [u.Pod.name for u in r.PerK[0].Failures] == ["x1"]
    assert "anti-affinity" in r.PerK[0].Failures[0].Reason
    assert [(p.Pod.name, p.Node) for p in r.Pods] == [("x1", None), ("x2", "n0")]


def test_spread_skew_falls_after_deletes():
    spread = {"topologySpreadConstraints": [{"maxSkew": 1, "topologyKey": "topology.kubernetes.io/zone", "whenUnsatisfiable": "DoNotSchedule",
                                             "labelSelector": {"matchLabels": {"app": "sp"}}}]}
    nodes = [_node("a0", zone="a"), _node("b0", zone="b", mcpu="1000m")]
    # zone b is full of another pod and holds no sp pod; zone a holds sp-0: one more sp pod in a would be skew 2
    pods = [_pod("sp-0", "100m", labels={"app": "sp"}, extra=spread, node="a0"), _pod("fill", "1000m", node="b0")]
    cluster = ResourceTypes(Nodes=nodes, Pods=pods)
    mk = lambda n: _pod(n, "100m", labels={"app": "sp"}, extra=spread)
    _, r = replay(cluster, ev((1, C, mk("sp-1")), (2, D, "default/sp-0"), (3, C, mk("sp-2")), (4, C, mk("sp-3")),
                              (5, D, "default/sp-2"), (6, C, mk("sp-4"))))
    # sp-1 fails on skew; deleting sp-0 takes zone a's count to 0, so sp-2 fits there and sp-3 fails again; deleting sp-2 lets sp-4 in
    got = [(p.Pod.name, p.Node) for p in r.Pods]
    assert got == [("sp-1", None), ("sp-2", "a0"), ("sp-3", None), ("sp-4", "a0")]
    assert all("topology spread" in u.Reason for u in r.PerK[0].Failures)


def test_gpu_share_device_freed_and_reused():
    ann = {"alibabacloud.com/gpu-mem": "12Gi", "alibabacloud.com/gpu-count": "1"}
    cluster = ResourceTypes(Nodes=[_node("g0", gpu=(2, "32Gi"))],
                            Pods=[_pod("g-a", "100m", ann=ann), _pod("g-b", "100m", ann=ann)])
    sim = session(cluster)
    assert sorted(sim.gpu_slots.tolist()) == [0x1, 0x10]
    first = sim.compiled.pod_recs[int(np.nonzero(sim.gpu_slots == 0x1)[0][0])].name
    ann8 = {"alibabacloud.com/gpu-mem": "8Gi", "alibabacloud.com/gpu-count": "1"}
    ts = trace.build(sim, ev((1, C, _pod("big", "100m", ann=ann)), (2, D, f"default/{first}"), (3, C, _pod("big2", "100m", ann=ann)),
                             (4, C, _pod("small", "100m", ann=ann8))), None, 0)
    r = trace.replay(CheckerEngine(ts.compiled), ts, 10)
    got = [(p.Pod.name, p.Node, p.GpuIndex) for p in r.Pods]
    # big: each device has 4Gi free -> fails; device 0 freed -> big2 takes it; small: 4Gi free on each -> fails
    assert got == [("big", None, None), ("big2", "g0", "0"), ("small", None, None)]
    s = r.PerK[0].Samples
    assert s["gpu_total"].tolist() == [32 << 30] * 4
    assert s["gpu_used"].tolist() == [24 << 30, 12 << 30, 24 << 30, 24 << 30]
    assert s["idle_devices"].tolist() == [0, 1, 0, 0] and s["partial_devices"].tolist() == [2, 1, 2, 2]


def test_host_port_freed():
    port = {"containers": [{"name": "c", "image": "nginx", "ports": [{"containerPort": 80, "hostPort": 8080}],
                            "resources": {"requests": {"cpu": "100m", "memory": "1Gi"}}}]}
    cluster = ResourceTypes(Nodes=[_node("n0")], Pods=[_pod("p0", extra=port)])
    _, r = replay(cluster, ev((1, C, _pod("p1", extra=port)), (2, D, "default/p0"), (3, C, _pod("p2", extra=port))))
    assert [(p.Pod.name, p.Node) for p in r.Pods] == [("p1", None), ("p2", "n0")]
    assert "free ports" in r.PerK[0].Failures[0].Reason


def test_extended_resources():
    ext = {"example.com/fpga": "1"}
    cluster = ResourceTypes(Nodes=[_node("n0", extra={"example.com/fpga": "1"})], Pods=[_pod("f0", "100m", limits=ext)])
    _, r = replay(cluster, ev((1, C, _pod("f1", "100m", limits=ext)), (2, D, "default/f0"), (3, C, _pod("f2", "100m", limits=ext))))
    assert [(p.Pod.name, p.Node) for p in r.Pods] == [("f1", None), ("f2", "n0")]
    assert "example.com/fpga" in r.PerK[0].Failures[0].Reason


def test_deleted_prebound_pod():
    cluster = ResourceTypes(Nodes=[_node("n0")], Pods=[_pod("bound", "3500m", node="n0")])
    _, r = replay(cluster, ev((1, D, "default/bound"), (2, C, _pod("a", "3500m"))))
    assert [(p.Pod.name, p.Node) for p in r.Pods] == [("a", "n0")]
    assert r.MinNodes == 0 and r.AllFromMinNodes and r.PerK[0].Deletes == 1


def test_sweep_over_new_nodes():
    cluster = ResourceTypes(Nodes=[_node("n0")], Pods=[_pod("old", "3000m")])
    events = ev((1, C, _pod("a", "2000m")), (2, C, _pod("b", "2000m")), (3, D, "default/a"), (4, C, _pod("c", "2000m")))
    ts, r = replay(cluster, events, new_node=_node("spec"), kmax=2)
    # k = 0: n0 has 1000m free, every create fails; k = 1: a and b fill the new node, the delete of a makes room for c
    assert [len(t.Failures) for t in r.PerK] == [3, 0, 0]
    assert r.MinNodes == 1 and r.AllFromMinNodes and r.K == 1
    assert all(p.Node is not None for p in r.Pods)


def test_host_refusals():
    cluster = ResourceTypes(Nodes=[_node("n0")], Pods=[_pod("old")])
    sim = session(cluster)
    with pytest.raises(ValueError, match="no pod holds"):
        trace.build(sim, ev((1, D, "default/nope")))
    with pytest.raises(ValueError, match="no pod holds"):
        trace.build(sim, ev((1, D, "default/old"), (2, D, "default/old")))
    with pytest.raises(ValueError, match="exists already"):
        trace.build(sim, ev((1, C, _pod("old"))))
    with pytest.raises(ValueError, match="spec.nodeName"):
        trace.build(sim, ev((1, C, _pod("x", node="n0"))))
    with pytest.raises(ValueError, match="not a Pod"):
        trace.build(sim, ev((1, C, _node("n1"))))
    with pytest.raises(ValueError, match="op"):
        trace.build(sim, ev((1, "evict", "default/old")))
    ds = {"apiVersion": "apps/v1", "kind": "DaemonSet", "metadata": {"name": "agent", "namespace": "kube-system"},
          "spec": {"selector": {"matchLabels": {"app": "agent"}}, "template": {"metadata": {"labels": {"app": "agent"}}, "spec": {
              "containers": [{"name": "c", "image": "a", "resources": {"requests": {"cpu": "10m"}}}]}}}}
    sim2 = session(ResourceTypes(Nodes=[_node("n0")], DaemonSets=[ds]))
    dpod = trace.pod_key(sim2.compiled.pod_recs[0])
    with pytest.raises(ValueError, match="DaemonSet pod"):
        trace.build(sim2, ev((1, D, dpod)))


def test_from_lifetimes_orders_deletes_first_and_is_stable():
    a, b, c = _pod("a"), _pod("b"), _pod("c")
    evs = trace.from_lifetimes([(a, 0, 5), (b, 5, None), (c, 5, 7)])
    assert [(e.time, e.op, e.pod if e.op == D else O.name_of(e.pod)) for e in evs] == [
        (0, C, "a"), (5, D, "default/a"), (5, C, "b"), (5, C, "c"), (7, D, "default/c")]
    with pytest.raises(ValueError, match="not after its start"):
        trace.from_lifetimes([(a, 3, 3)])
    assert trace.sample_events(10, 4) == [1, 4, 6, 9] and trace.sample_events(3, 100) == [0, 1, 2] and trace.sample_events(0, 5) == []


def test_class_pod_limit_refused(monkeypatch):
    """A superset whose pod count passes a class's int32 bound (Compiled.class_pod_limit) is refused before any device work."""
    real = trace.compile_cluster

    def tight(*a, **kw):
        c = real(*a, **kw)
        c.class_pod_limit = [2] * len(c.class_pod_limit)
        return c
    monkeypatch.setattr(trace, "compile_cluster", tight)
    sim = session(ResourceTypes(Nodes=[_node("n0")], Pods=[_pod("old")]))
    with pytest.raises(ValueError, match="int32 bounds"):
        trace.build(sim, ev((1, C, _pod("a")), (2, C, _pod("b"))))
