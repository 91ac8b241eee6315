"""DaemonSet pods (utils.MakeValidPodsByDaemonset, pkg/utils/utils.go:337-351; SetDaemonSetPodNodeNameByNodeAffinity :770-815):
one pod per node, pinned by a required matchFields metadata.name term.  The snapshot compiler gives the pods of one DaemonSet ONE
class whose programs say "the pod's pin" (REQ_NODE_IS payload -3) and a per-pod pin column (simon_podset.pod_pin_node), instead of
one class per node.  CPU: C oracle (pin-aware classes) == object-level restatement (which sees the real per-pod affinity).
GPU: engine == oracle, incl. failure histograms, scenarios in which the pin node does not exist, and a DaemonSet-heavy cluster."""
import numpy as np
import pytest

from simon_b200 import objects as O, simulator, synth
from simon_b200.compiler import CLS_PINNED, SCW_FLAGS, SCW_GUARD_NODE, compile_cluster
from util import assert_ext_equal, run_oracle, run_oracle_ext, run_pyref


def _node(name, cpu="4", zone=None, taints=None, unschedulable=False, labels=None):
    lab = {"kubernetes.io/hostname": name, "kubernetes.io/os": "linux"}
    if zone:
        lab["topology.kubernetes.io/zone"] = zone
    lab.update(labels or {})
    n = {"apiVersion": "v1", "kind": "Node", "metadata": {"name": name, "labels": lab}, "spec": {},
         "status": {"allocatable": {"cpu": cpu, "memory": "8Gi", "pods": "20"}, "capacity": {"cpu": cpu, "memory": "8Gi", "pods": "20"}}}
    if taints:
        n["spec"]["taints"] = taints
    if unschedulable:
        n["spec"]["unschedulable"] = True
    return n


def _ds(name, cpu="500m", port=None, tolerations=None, node_selector=None, affinity=None, labels=None, tsc=None):
    c = {"name": "c", "image": f"{name}:v1", "resources": {"requests": {"cpu": cpu, "memory": "64Mi"}}}
    if port:
        c["ports"] = [{"containerPort": port, "hostPort": port}]
    spec = {"containers": [c]}
    if tolerations is not None:
        spec["tolerations"] = tolerations
    if node_selector:
        spec["nodeSelector"] = node_selector
    if affinity:
        spec["affinity"] = affinity
    if tsc:
        spec["topologySpreadConstraints"] = tsc
    lab = dict(labels or {"ds": name})
    return {"apiVersion": "apps/v1", "kind": "DaemonSet", "metadata": {"name": name, "namespace": "kube-system"},
            "spec": {"selector": {"matchLabels": lab}, "template": {"metadata": {"labels": lab}, "spec": spec}}}


def _deploy(name, replicas, cpu="1", labels=None, anti_to=None):
    lab = dict(labels or {"app": name})
    spec = {"containers": [{"name": "c", "image": "app:v1", "resources": {"requests": {"cpu": cpu, "memory": "128Mi"}}}]}
    if anti_to:
        spec["affinity"] = {"podAntiAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": [
            {"labelSelector": {"matchLabels": anti_to}, "topologyKey": "kubernetes.io/hostname"}]}}
    return {"apiVersion": "apps/v1", "kind": "Deployment", "metadata": {"name": name, "namespace": "default"},
            "spec": {"replicas": replicas, "selector": {"matchLabels": lab}, "template": {"metadata": {"labels": lab}, "spec": spec}}}


def _cluster():
    nodes = [_node("n0", zone="a"), _node("n1", zone="a", cpu="1"), _node("n2", zone="b", taints=[{"key": "gpu", "value": "y", "effect": "NoSchedule"}]),
             _node("n3", zone="b", unschedulable=True), _node("n4", labels={"role": "edge"}), _node("n5", zone="c", labels={"role": "edge"})]
    two_terms = {"nodeAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": {"nodeSelectorTerms": [
        {"matchExpressions": [{"key": "role", "operator": "In", "values": ["edge"]}]},
        {"matchExpressions": [{"key": "topology.kubernetes.io/zone", "operator": "In", "values": ["a"]}]}]}}}
    dss = [
        _ds("plain"),                                                               # fails on the tainted node
        _ds("tolerant", tolerations=[{"operator": "Exists"}], port=9100),           # runs everywhere, incl. the unschedulable node
        _ds("selected", node_selector={"role": "edge"}),                            # nodeSelector AND pin
        _ds("twoterm", affinity=two_terms, cpu="600m"),                             # every term gets the pin
        _ds("hungry", cpu="900m", tolerations=[{"operator": "Exists"}]),            # does not fit n1 after the others
        _ds("spread", tsc=[{"maxSkew": 1, "topologyKey": "topology.kubernetes.io/zone", "whenUnsatisfiable": "DoNotSchedule",
                            "labelSelector": {"matchLabels": {"ds": "spread"}}}]),   # hard constraint: needs the zone label
    ]
    cluster = O.ResourceTypes(Nodes=nodes, DaemonSets=dss)
    app = O.ResourceTypes(Deployments=[_deploy("web", 5), _deploy("shy", 3, anti_to={"ds": "tolerant"})],
                          DaemonSets=[_ds("late", cpu="300m", port=9100)])         # port clash with "tolerant" on every node
    return cluster, [O.AppResource("app", app)]


def _compiled():
    cluster, apps = _cluster()
    p = simulator.plan(cluster, apps)
    return p, compile_cluster(p.nodes, p.pods, p.ctx)


def test_one_class_per_daemonset_with_per_pod_pins():
    p, c = _compiled()
    off, blob, pc, pin = c.pods["class_off"], c.pods["class_blob"], c.pods["pod_class"], c.pods["pod_pin_node"]
    ds_pods = [i for i, r in enumerate(p.pods) if r.tmpl.workload_kind == "DaemonSet"]
    by_ds = {}
    for i in ds_pods:
        by_ds.setdefault(p.pods[i].tmpl.workload_name, set()).add(int(pc[i]))
        assert c.node_names[pin[i]] == p.pods[i].tmpl.guard_node_name
        w = blob[off[pc[i]]:]
        assert w[SCW_GUARD_NODE] == -3 and (w[SCW_FLAGS] & CLS_PINNED)
    assert all(len(v) == 1 for v in by_ds.values()) and len(by_ds) == 7
    assert all(pin[i] == -1 for i in range(len(p.pods)) if i not in ds_pods)
    # eligibility of utils.NodeShouldRunPod (selector + taints; spec.unschedulable is left to the NodeUnschedulable filter)
    count = lambda name: sum(1 for i in ds_pods if p.pods[i].tmpl.workload_name == name)
    assert count("plain") == 5 and count("tolerant") == 6 and count("selected") == 2 and count("twoterm") == 4


def test_oracle_with_pinned_classes_matches_the_object_level_restatement():
    p, c = _compiled()
    (out, _score, fc, fp), _st = run_oracle(c)
    np.testing.assert_array_equal(out, run_pyref(p, c))
    # every placed DaemonSet pod sits on its pin
    for i, r in enumerate(p.pods):
        if r.tmpl.workload_kind == "DaemonSet" and out[i] >= 0:
            assert c.node_names[out[i]] == r.tmpl.guard_node_name
    # "late" asks for the host port "tolerant" already holds on every node: all of its pods fail, on the pin with NodePorts,
    # on every other node with NodeAffinity (the pin) - unless an earlier static filter rejects that node first
    late = [i for i, r in enumerate(p.pods) if r.tmpl.workload_name == "late"]
    assert late and all(out[i] == -1 for i in late)
    row = {int(pod): fc[j] for j, pod in enumerate(fp)}
    for i in late:
        on_unschedulable = p.pods[i].tmpl.guard_node_name == "n3"      # NodeUnschedulable rejects the pin itself before NodePorts runs
        assert row[i][1] == (0 if on_unschedulable else 1) and row[i][0] + row[i][1] == c.n_nodes and row[i].sum() == c.n_nodes
    msg = simulator.format_fit_error(c, p.pods[late[0]], row[late[0]])
    assert "1 node(s) didn't have free ports for the requested pod ports" in msg and "node(s) didn't match Pod's node affinity" in msg


@pytest.mark.parametrize("seed", [3, 4, 5, 6])
def test_mixed_clusters_with_daemonsets_cpu(seed):
    cluster, apps = synth.make_mix(seed_no=seed, n_nodes=30, n_workloads=25, max_replicas=5)
    for k in range(3):
        cluster.DaemonSets.append(_ds(f"extra-{k}", cpu="50m", port=9200 + k, tolerations=[{"operator": "Exists"}] if k else None))
    p = simulator.plan(cluster, apps)
    c = compile_cluster(p.nodes, p.pods, p.ctx)
    (out, _s, _fc, _fp), _st = run_oracle(c)
    np.testing.assert_array_equal(out, run_pyref(p, c))
    assert c.pods_dims["n_classes"] < len({id(r.tmpl) for r in p.pods})


def _gpu_cmp(c):
    """Both device paths of pinned pods - the run-at-once fast path and the general decision path - against the oracle."""
    from simon_b200.engine import Engine
    (ref, rscore, rfc, rfp), rstate, rext, rslots = run_oracle_ext(c)
    for pin_fast in (True, False):
        with Engine(c, device=0, record_scores=True, pin_fast=pin_fast) as eng:
            out, score, fc, fp = eng.schedule()
            st = eng.state()
            assert_ext_equal(eng, rext, rslots, f"pin_fast={pin_fast}")
            eng.reset()
            half = len(ref) // 2                                    # split calls: a run of pinned pods cut by the call boundary
            out2 = np.concatenate([eng.schedule(0, half)[0], eng.schedule(half, len(ref) - half)[0]])
        np.testing.assert_array_equal(out, ref, err_msg=f"pin_fast={pin_fast}")
        np.testing.assert_array_equal(out2, ref, err_msg=f"pin_fast={pin_fast}, two calls")
        np.testing.assert_array_equal(fp, rfp)
        np.testing.assert_array_equal(fc, rfc, err_msg=f"pin_fast={pin_fast}")
        sched = ref >= 0
        np.testing.assert_array_equal(score[sched & (rscore > 0)], rscore[sched & (rscore > 0)])
        for k in rstate:
            np.testing.assert_array_equal(st[k], rstate[k], err_msg=k)
    return out


@pytest.mark.gpu
def test_pinned_classes_gpu_matches_oracle():
    _p, c = _compiled()
    _gpu_cmp(c)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [3, 4, 5, 6, 7, 8])
def test_mixed_clusters_with_daemonsets_gpu(seed):
    cluster, apps = synth.make_mix(seed_no=seed, n_nodes=30 + 20 * (seed % 3), n_workloads=25, max_replicas=5)
    for k in range(3):
        cluster.DaemonSets.append(_ds(f"extra-{k}", cpu="50m", port=9200 + k, tolerations=[{"operator": "Exists"}] if k else None))
    p = simulator.plan(cluster, apps)
    _gpu_cmp(compile_cluster(p.nodes, p.pods, p.ctx))


@pytest.mark.gpu
def test_daemonset_heavy_cluster_gpu():
    """2,000 nodes, 5 DaemonSets (10,000 pinned pods in 5 classes) in front of and between ordinary workloads."""
    cluster, apps = synth.make_c3(n_nodes=2000, n_workloads=60, replicas=40, n_apps=3, seed_no=11)
    for k in range(4):
        cluster.DaemonSets.append(_ds(f"agent-{k}", cpu="50m", port=9100 + k, tolerations=[{"operator": "Exists"}]))
    apps[1].Resource.DaemonSets.append(_ds("app-agent", cpu="2", tolerations=[{"operator": "Exists"}]))     # some of these do not fit
    p = simulator.plan(cluster, apps)
    c = compile_cluster(p.nodes, p.pods, p.ctx)
    assert c.pods_dims["n_classes"] < 400
    out = _gpu_cmp(c)
    ds = np.array([r.tmpl.workload_kind == "DaemonSet" for r in p.pods])
    assert ds.sum() >= 9000 and (out[ds] >= 0).sum() > 8000 and (out[ds] == -1).sum() > 0


@pytest.mark.gpu
def test_pin_nodes_absent_from_a_scenario_gpu():
    """Capacity scenarios: a DaemonSet pod exists only where its pin node does (per-pod guard)."""
    from simon_b200.engine import Engine
    from oracle.binding import Oracle
    _p, c = _compiled()
    for active in ([0, 1, 2, 4, 5], [5, 4, 0], [1, 3]):
        act = np.array(active, dtype=np.uint32)
        o = Oracle(c)
        o.set_active(act)
        ref = o.schedule()[0]
        o.close()
        for pin_fast in (True, False):
            with Engine(c, device=0, pin_fast=pin_fast) as eng:
                _res, nodes = eng.run_scenarios([act], want_nodes=True)
            np.testing.assert_array_equal(nodes[0], ref, err_msg=f"pin_fast={pin_fast}")
        assert (ref == -3).sum() > 0
