"""Open-Local exclusive devices (SSD / HDD volumes; pkg/simulator/plugin/open-local.go, OL = vendor/github.com/alibaba/open-local/pkg
of the reference): hand-derived known answers of the host restatement (ProcessDevicePVC, CheckExclusiveResourceMeetsPVCSize,
ScoreDevice), the compiled device columns, the refusals, the annotation Bind writes, and on the GPU the engine's placements against
the restated Filter, Score and Bind."""
import ctypes
import json
import os

import numpy as np
import pytest

from simon_b200 import objects as O
from simon_b200.compiler import CompileError, compile_cluster
from simon_b200.storage import INT64_MIN, ClassVolumes, StorageReplay, device_place, raw_score
from simon_b200.workloads import PodRec, PodTemplate

GI = 1 << 30
HERE = os.path.dirname(os.path.abspath(__file__))
EXAMPLE = os.path.join(HERE, "golden", "reference", "example")
SCS = [{"apiVersion": "storage.k8s.io/v1", "kind": "StorageClass", "metadata": {"name": f"open-local-device-{m}"},
        "parameters": {"mediaType": m}} for m in ("ssd", "hdd")]


def _dev(name, cap, media="hdd", alloc=False):
    return {"name": name, "device": name, "capacity": cap, "mediaType": media, "isAllocated": alloc}


def _ann_dev(d):
    return dict(d, capacity=str(d["capacity"]), isAllocated="true" if d["isAllocated"] else "false")


def _node(name, vgs=None, devs=None, taint=False, annotated=True):
    n = {"apiVersion": "v1", "kind": "Node",
         "metadata": {"name": name, "labels": {"kubernetes.io/hostname": name}, "annotations": {}},
         "status": {"allocatable": {"cpu": "16", "memory": "64Gi", "pods": "110"}}}
    if annotated:
        ann = {"vgs": [{"name": f"vg{i}", "capacity": str(c), "requested": "0"} for i, c in enumerate(vgs or [])],
               "devices": [_ann_dev(d) for d in devs or []]}
        n["metadata"]["annotations"][O.ANNO_NODE_LOCAL_STORAGE] = json.dumps(ann)
    if taint:
        n["spec"] = {"taints": [{"key": "k", "value": "v", "effect": "NoSchedule"}]}
    return n


def _pod(name, vols):
    ann = {O.ANNO_POD_LOCAL_STORAGE: json.dumps({"volumes": vols})} if vols is not None else {}
    pod = {"apiVersion": "v1", "kind": "Pod", "metadata": {"name": name, "namespace": "default", "annotations": ann},
           "spec": {"containers": [{"name": "c", "image": "x", "resources": {"requests": {"cpu": "100m", "memory": "128Mi"}}}]}}
    return PodRec(PodTemplate(pod, "Pod", name, "default"), name, 0)


def _vol(size, kind):
    sc = {"LVM": "open-local-lvm", "SSD": "open-local-device-ssd", "HDD": "open-local-device-hdd"}[kind]
    return {"size": str(size), "kind": kind, "scName": sc}


# ---- device_place: hand-derived cases ---------------------------------------------------------------------------------------

def test_ascending_first_fit_skips_a_small_device():
    """Free HDDs sorted by capacity: 10Gi (#0), 60Gi (#2), 100Gi (#1).  The 50Gi PVC skips 10Gi (not the last device) and takes
    60Gi; ScoreDevice = int(50/60 * 10) = 8."""
    devs = [_dev("a", 10 * GI), _dev("b", 100 * GI), _dev("c", 60 * GI)]
    assert device_place("n", devs, [], [50 * GI]) == (None, [2], 8)


def test_last_device_too_small_reports_pvcs_free_and_total():
    """The last free HDD is smaller than the PVC: (PVCs 1, free HDDs 2, total 5).  The total counts the allocated HDD, the SSD and
    the device of another media type (len(nodeCache.Devices), common.go:384-392)."""
    devs = [_dev("a", 10 * GI), _dev("b", 20 * GI), _dev("c", 500 * GI, alloc=True), _dev("s", 500 * GI, "ssd"),
            _dev("x", 500 * GI, "nvme")]
    assert device_place("n", devs, [], [30 * GI]) == ("Insufficient Device storage, requested 1, available 2, capacity 5", [], 0)


def test_ssd_shortfall_and_the_hdd_shortfall_reporting_ssd_counts():
    """Fewer free devices than PVCs: NewInsufficientExclusiveResourceError(requested, free, total) for SSD (common.go:413-419); the
    HDD branch passes the SSD counts (:430-435)."""
    devs = [_dev("s0", 100 * GI, "ssd"), _dev("s1", 100 * GI, "ssd", alloc=True), _dev("h0", 100 * GI)]
    assert device_place("n", devs, [GI, GI], [])[0] == "Insufficient Device storage, requested 2, available 1, capacity 3"
    assert device_place("n", devs, [GI], [GI, GI])[0] == "Insufficient Device storage, requested 1, available 1, capacity 3"
    assert device_place("n", devs, [], [GI, GI])[0] == "Insufficient Device storage, requested 0, available 1, capacity 3"


def test_devices_that_run_out_leave_a_partial_allocation():
    """Free [10Gi, 100Gi], PVCs [50Gi, 60Gi]: 10Gi is skipped, 100Gi takes 50Gi, the walk ends with the 60Gi PVC unplaced and the
    node passes with one unit: int(0.5 * 10) = 5 (common.go:312-349)."""
    devs = [_dev("a", 10 * GI), _dev("b", 100 * GI)]
    assert device_place("n", devs, [], [60 * GI, 50 * GI]) == (None, [1], 5)


def test_equal_capacities_are_taken_in_annotation_order():
    devs = [_dev("x", 5 * GI), _dev("b", 100 * GI), _dev("a", 100 * GI)]
    assert device_place("n", devs, [], [50 * GI])[1] == [1]
    devs[1]["isAllocated"] = True
    assert device_place("n", devs, [], [50 * GI])[1] == [2]


def test_allocated_and_other_media_devices_are_not_free():
    devs = [_dev("a", 100 * GI, alloc=True), _dev("b", 100 * GI, "nvme"), _dev("c", 100 * GI, "ssd")]
    assert device_place("n", devs, [], [GI])[0] == "Insufficient Device storage, requested 0, available 1, capacity 3"
    assert device_place("n", devs, [GI], []) == (None, [2], 0)


def test_mixed_score_sums_ssd_units_then_hdd_units_in_ascending_pvc_order():
    """Units 1/10 and 2/10 (SSD, ascending) then 3/10 (HDD): 0.1 + 0.2 + 0.3 = 0.6000000000000001 in float64, / 3 * 10 =
    2.0000000000000004 -> 2.  Summed the other way round (0.3 + 0.2 + 0.1 = 0.6) it would give 1."""
    devs = [_dev("h", 10 * GI), _dev("s1", 10 * GI, "ssd"), _dev("s0", 10 * GI, "ssd")]
    err, chosen, score = device_place("n", devs, [2 * GI, 1 * GI], [3 * GI])
    assert err is None and chosen == [1, 2, 0]
    assert score == 2 and int((0.3 + 0.2 + 0.1) / 3 * 10) == 1


def test_min_int64_only_when_every_device_pvc_was_dropped():
    assert raw_score(ClassVolumes(local=True, dropped=1), 0) == INT64_MIN
    assert raw_score(ClassVolumes(local=True, dropped=1, lvm=[(GI, "")]), 3) == INT64_MIN + 3
    assert raw_score(ClassVolumes(local=True, dropped=1, hdd=[GI]), 3) == 3
    assert raw_score(ClassVolumes(local=True, ssd=[GI]), 7) == 7
    assert device_place("n", None, [], []) == (None, [], 0)


# ---- compiled columns and refusals ------------------------------------------------------------------------------------------

def test_compiled_device_columns_of_a_hand_cluster():
    """Slots: SSDs first, then HDDs, each ascending by capacity with ties in annotation order; other media get no slot."""
    devs = [_dev("h100", 100 * GI), _dev("s50a", 50 * GI, "ssd"), _dev("h20", 20 * GI, alloc=True), _dev("nv", 10 * GI, "nvme"),
            _dev("s50b", 50 * GI, "ssd")]
    nodes = [_node("a", [100 * GI], devs), _node("b", annotated=False), _node("c", [], [])]
    pods = [_pod("p0", [_vol(3 * GI, "SSD"), _vol(GI, "SSD"), _vol(2 * GI, "HDD"), _vol(GI, "LVM")]), _pod("q", None)]
    c = compile_cluster(nodes, pods, open_local=True, storage_classes=SCS, local_devices=True)
    st = c.storage
    g = {n: c.node_index(n) for n in "abc"}
    assert st.devices and st.n_dev_slots == 4
    assert st.node_n_ssd[g["a"]] == 2 and st.node_n_hdd[g["a"]] == 2
    assert st.dev_capacity[:, g["a"]].tolist() == [50 * GI, 50 * GI, 20 * GI, 100 * GI]
    assert st.dev_index[:, g["a"]].tolist() == [1, 4, 2, 0]
    assert st.dev_alloc[g["a"]] == 1 << 2
    for n in "bc":
        assert (st.node_n_ssd[g[n]], st.node_n_hdd[g[n]], st.dev_alloc[g[n]]) == (0, 0, 0)
    k = next(cid for cid in range(len(c.classes)) if st.class_local[cid])
    assert st.ssd_size[st.ssd_off[k]:st.ssd_off[k + 1]].tolist() == [GI, 3 * GI]
    assert st.hdd_size[st.hdd_off[k]:st.hdd_off[k + 1]].tolist() == [2 * GI]
    assert st.vol_size[st.vol_off[k]:st.vol_off[k + 1]].tolist() == [GI]
    assert st.ssd_off[-1] == 2 and st.hdd_off[-1] == 1


def test_compiled_device_columns_of_demo_1():
    """demo_1: master-1 and worker-1 carry one 100Gi HDD each (/dev/vdd), no SSD."""
    from simon_b200.objects import create_cluster_resource_from_cluster_config
    from simon_b200.simulator import plan
    cluster = create_cluster_resource_from_cluster_config(os.path.join(EXAMPLE, "cluster", "demo_1"))
    p = plan(cluster, [])
    c = compile_cluster(p.nodes, p.pods, p.ctx, open_local=True, storage_classes=list(cluster.StorageClasss), local_devices=True)
    st = c.storage
    for g, name in enumerate(c.node_names):
        if name in ("master-1", "worker-1"):
            assert (st.node_n_ssd[g], st.node_n_hdd[g], st.dev_capacity[0, g], st.dev_index[0, g]) == (0, 1, 100 * GI, 0)
        else:
            assert st.node_n_ssd[g] == 0 and st.node_n_hdd[g] == 0
    assert st.n_dev_slots == 1 and not st.dev_alloc.any()


@pytest.mark.parametrize("devs, msg", [
    ([_dev("d", GI), {**_dev("d", GI), "device": "/dev/other"}], "duplicate device names"),
    ([_dev(f"d{i}", GI, "ssd" if i % 2 else "hdd") for i in range(17)], "more than 16"),
])
def test_node_refusals_with_devices(devs, msg):
    nodes = [_node("a", [GI], devs)]
    with pytest.raises(CompileError, match=msg):
        compile_cluster(nodes, [_pod("p0", [_vol(GI, "HDD")])], open_local=True, storage_classes=SCS, local_devices=True)


def test_more_devices_of_other_media_and_duplicate_names_without_the_opt_in_pass():
    devs = [_dev(f"d{i}", GI, "nvme") for i in range(20)] + [_dev("h", GI), {**_dev("h", GI), "device": "/dev/h2"}]
    c = compile_cluster([_node("a", [GI], devs)], [_pod("p0", [_vol(GI, "LVM")])], open_local=True)
    assert not c.storage.devices
    c = compile_cluster([_node("a", [GI], devs[:20])], [_pod("p0", [_vol(GI, "HDD")])], open_local=True, storage_classes=SCS,
                        local_devices=True)
    assert c.storage.n_dev_slots == 0


def test_class_refusals_with_devices():
    nodes = [_node("a", [GI], [_dev("d", GI)])]
    with pytest.raises(CompileError, match="more than 8 SSD / HDD"):
        compile_cluster(nodes, [_pod("p0", [_vol(GI, "SSD")] * 5 + [_vol(GI, "HDD")] * 4)], open_local=True, storage_classes=SCS,
                        local_devices=True)
    with pytest.raises(ValueError, match="open_local"):
        compile_cluster(nodes, [_pod("p0", [_vol(GI, "HDD")])], storage_classes=SCS, local_devices=True)
    with pytest.raises(CompileError, match="exclusive"):
        compile_cluster(nodes, [_pod("p0", [_vol(GI, "HDD")])], open_local=True, storage_classes=SCS)


def test_annotation_bind_writes():
    """Bind sets isAllocated on the devices the Filter chose and marshals the annotation in ffjson form (open-local.go:232-246)."""
    devs = [_dev("/dev/vdb", 100 * GI, "ssd"), _dev("/dev/vdc", 50 * GI), _dev("/dev/vdd", 200 * GI)]
    c = compile_cluster([_node("a", [100 * GI], devs)], [_pod("p0", [_vol(40 * GI, "HDD"), _vol(10 * GI, "LVM")])],
                        open_local=True, storage_classes=SCS, local_devices=True)
    rep = StorageReplay(c.storage, c.node_names)
    assert rep.reason(0, 0) is None
    rep.bind(0, 0)
    assert rep.annotation(0) == (
        '{"vgs":[{"name":"vg0","capacity":"107374182400","requested":"10737418240"}],"devices":['
        '{"name":"/dev/vdb","device":"/dev/vdb","capacity":"107374182400","mediaType":"ssd","isAllocated":"false"},'
        '{"name":"/dev/vdc","device":"/dev/vdc","capacity":"53687091200","mediaType":"hdd","isAllocated":"true"},'
        '{"name":"/dev/vdd","device":"/dev/vdd","capacity":"214748364800","mediaType":"hdd","isAllocated":"false"}]}')
    assert rep.alloc_masks().tolist() == [1 << 1]       # slots: vdb (SSD), vdc, vdd
    rep.bind(0, 0)
    assert rep.alloc_masks().tolist() == [0b110]
    assert rep.reason(0, 0) == "Insufficient Device storage, requested 0, available 1, capacity 3"


# ---- on the GPU -------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_demo_1_hdd_statefulset_on_gpu():
    """Three replicas with one 50Gi HDD volume each: master-1 is tainted and master-2/3 have no annotation, so replica 0 takes
    worker-1's /dev/vdd; replicas 1-2 find no free HDD there, and the HDD shortfall reports the SSD counts (0, 0, of 1 device)."""
    from simon_b200.objects import AppResource, ResourceTypes, create_cluster_resource_from_cluster_config
    from simon_b200.simulator import Simulate, WithOpenLocal
    cluster = create_cluster_resource_from_cluster_config(os.path.join(EXAMPLE, "cluster", "demo_1"))
    sts = {"apiVersion": "apps/v1", "kind": "StatefulSet", "metadata": {"name": "hdd", "namespace": "default"},
           "spec": {"replicas": 3, "serviceName": "hdd", "selector": {"matchLabels": {"app": "hdd"}},
                    "volumeClaimTemplates": [{"metadata": {"name": "data"}, "spec": {
                        "storageClassName": "open-local-device-hdd", "resources": {"requests": {"storage": "50Gi"}}}}],
                    "template": {"metadata": {"labels": {"app": "hdd"}}, "spec": {"containers": [
                        {"name": "c", "image": "x", "resources": {"requests": {"cpu": "100m", "memory": "128Mi"}}}]}}}}
    res = Simulate(cluster, [AppResource("hdd", ResourceTypes(StatefulSets=[sts]))], WithOpenLocal(devices=True))
    placed = {p.name: O.name_of(ns.Node) for ns in res.NodeStatus for p in ns.Pods if p.name.startswith("hdd")}
    assert placed == {"hdd-0": "worker-1"}
    w = next(ns.Node for ns in res.NodeStatus if O.name_of(ns.Node) == "worker-1")
    ann = json.loads(O.annotations_of(w)[O.ANNO_NODE_LOCAL_STORAGE])
    assert [(d["device"], d["isAllocated"]) for d in ann["devices"]] == [("/dev/vdd", "true")]
    m1 = next(ns.Node for ns in res.NodeStatus if O.name_of(ns.Node) == "master-1")
    assert json.loads(O.annotations_of(m1)[O.ANNO_NODE_LOCAL_STORAGE])["devices"][0]["isAllocated"] == "false"
    un = sorted(res.UnscheduledPods, key=lambda u: u.Pod.name)
    assert [u.Pod.name for u in un] == ["hdd-1", "hdd-2"]
    for u in un:
        assert "1 Insufficient Device storage, requested 0, available 0, capacity 1" in u.Reason, u.Reason


def _random_cluster(rng, n_nodes, n_pods):
    """Nodes: 15 % without the annotation, the others with 0-3 VGs and 0-6 SSD / HDD devices (a few allocated, a few of another
    media type), capacities from a short list so that ties occur.  Pods: none, LVM only, devices only, both, and dropped device
    PVCs (yoda-device-*, a class no StorageClass defines).  Every node has one allocatable shape and every pod is bare."""
    caps = [10, 20, 50, 100, 200]
    nodes = []
    for i in range(n_nodes):
        if rng.random() < 0.15:
            nodes.append(_node(f"n{i:05d}", annotated=False))
            continue
        vgs = [int(rng.integers(1, 20)) * 10 * GI for _ in range(int(rng.integers(0, 4)))]
        devs = [_dev(f"/dev/d{k}", int(rng.choice(caps)) * GI, str(rng.choice(["ssd", "hdd", "hdd", "nvme"] if k == 0 else ["ssd", "hdd"])),
                     alloc=bool(rng.random() < 0.1)) for k in range(int(rng.integers(0, 7)))]
        nodes.append(_node(f"n{i:05d}", vgs, devs))
    pods = []
    for j in range(n_pods):
        r = rng.random()
        if r < 0.2:
            pods.append(_pod(f"q{j:05d}", None))
            continue
        vols = []
        if r < 0.55:
            vols += [_vol(int(rng.integers(1, 8)) * 5 * GI, "LVM") for _ in range(int(rng.integers(1, 3)))]
        if r >= 0.4:
            vols += [_vol(int(rng.choice([5, 10, 20, 50, 100, 150])) * GI, str(rng.choice(["SSD", "HDD"])))
                     for _ in range(int(rng.integers(1, 3)))]
        if rng.random() < 0.1:
            vols.append({"size": str(GI), "kind": "HDD", "scName": "yoda-device-hdd"})
        pods.append(_pod(f"p{j:05d}", vols))
    return nodes, pods


@pytest.mark.gpu
@pytest.mark.parametrize("seed, n_nodes, n_pods, pin_fast", [(1, 40, 300, True), (2, 700, 2000, True), (3, 3000, 4000, False),
                                                              (4, 250, 1500, False), (5, 41000, 1500, True)])
def test_engine_follows_the_restated_device_filter_and_bind(seed, n_nodes, n_pods, pin_fast):
    """Every storage pod the engine places passes the restated Filter (LVM and devices) on its turn's state; a refused storage pod
    reports Open-Local rejections (bit 20) or every node failed an earlier filter; the final VG state and device masks equal the
    replay of Bind in placement order.  41,000 nodes cover the large-cluster kernel variant."""
    from simon_b200.engine import Engine
    rng = np.random.default_rng(seed)
    nodes, pods = _random_cluster(rng, n_nodes, n_pods)
    c = compile_cluster(nodes, pods, open_local=True, storage_classes=SCS, local_devices=True)
    st = c.storage
    with Engine(c, pin_fast=pin_fast) as eng:
        out, _s, fail_counts, fail_pod = eng.schedule()
        final_vg, final_dev = eng.storage_state(), eng.device_state()
    rep = StorageReplay(st, c.node_names)
    fails = {int(p): j for j, p in enumerate(fail_pod)}
    pod_class = c.pods["pod_class"]
    placed_dev = 0
    for i, n in enumerate(out.tolist()):
        cls = int(pod_class[i])
        cv = st.class_volumes[cls]
        if n >= 0:
            if st.class_local[cls]:
                assert st.node_storage[n] is not None and rep.reason(cls, n) is None, i
                rep.bind(cls, n)
                placed_dev += bool(cv.ssd or cv.hdd)
        else:
            assert n == -1 and i in fails
            if st.class_local[cls]:
                assert int(fail_counts[fails[i]][20]) > 0 or int(fail_counts[fails[i]].sum()) == c.n_nodes
    assert np.array_equal(final_vg, rep.requested())
    assert np.array_equal(final_dev, rep.alloc_masks())
    assert placed_dev > 0


@pytest.mark.gpu
@pytest.mark.parametrize("seed, n_nodes, n_pods", [(11, 30, 160), (12, 200, 300), (13, 700, 250), (14, 41000, 60)])
def test_engine_matches_cpu_port_with_restated_devices(seed, n_nodes, n_pods):
    """Node and recorded winning score of every pod against an independent composition: the CPU port (oracle/simon_oracle.c, no
    Open-Local) replays the engine's earlier placements as bound pods and scores the pod's cycle; Open-Local's Filter, ScoreLVM +
    ScoreDevice and NormalizeScore come on top from the state the engine's earlier Binds left (storage.py).  The nodes share one
    allocatable shape and the pods are bare, so every other score plugin gives the same per-node score whatever the feasible set
    is.  Some placements must be decided by differing device scores."""
    from simon_b200.engine import Engine
    c = restated_cluster(seed, n_nodes, n_pods)
    with Engine(c, record_scores=True) as eng:
        out, score, _fc, _fp = eng.schedule()
        final_dev = eng.device_state()
    assert check_restated_devices(c, out, score, final_dev) > 0


def restated_cluster(seed, n_nodes, n_pods):
    """The cluster of _random_cluster(seed) compiled with Open-Local and its devices."""
    rng = np.random.default_rng(seed)
    nodes, pods = _random_cluster(rng, n_nodes, n_pods)
    return compile_cluster(nodes, pods, open_local=True, storage_classes=SCS, local_devices=True)


def check_restated_devices(c, out, score, final_dev):
    """The composition above, pod by pod, for a run of a cluster of restated_cluster: out / score are its placements and recorded
    winning scores, final_dev its device masks.  Returns the number of decisions with several feasible nodes whose device scores
    differ."""
    from oracle.binding import Oracle
    from simon_b200.storage import lvm_place, normalize_scores
    st = c.storage
    orc = Oracle(c)
    orc.enable_dump()
    P = c.pods_dims["n_pods"]
    fixed = np.ctypeslib.as_array((ctypes.c_int32 * P).from_address(orc.pods.pod_fixed_node))
    rep = StorageReplay(st, c.node_names)
    pod_class = c.pods["pod_class"]
    by_device = 0
    for i in range(P):
        assert fixed[i] == -1
        fixed[:i] = np.where(out[:i] >= 0, out[:i], -2)
        fixed[i] = -1
        orc.reset()
        orc.schedule(0, i + 1)
        code, sc = orc.last_detail()
        cls = int(pod_class[i])
        cv = st.class_volumes[cls]
        feas = [g for g in range(c.n_nodes) if code[g] == 0]
        raw, dev = {}, {}
        if st.class_local[cls]:
            keep = []
            for g in feas:
                if st.node_storage[g] is None:
                    continue
                err, _u, _chosen, s = rep.place(cls, g)
                if err is None:
                    keep.append(g)
                    raw[g] = raw_score(cv, s)
                    dev[g] = s - lvm_place(c.node_names[g], rep.vgs[g], cv.lvm)[2]
            feas = keep
        if not feas:
            assert out[i] == -1, i
            continue
        if len(feas) == 1:
            assert (out[i], score[i]) == (feas[0], 0), i
        else:
            norm = dict(zip(feas, normalize_scores([raw.get(g, 0) for g in feas])))
            tot = {g: int(sc[g, 8]) + norm[g] for g in feas}
            best = max(feas, key=lambda g: (tot[g], -g))
            assert (out[i], score[i]) == (best, tot[best]), i
            if len(set(dev.values())) > 1:
                by_device += 1
        if st.class_local[cls]:
            rep.bind(cls, int(out[i]))
    orc.close()
    assert np.array_equal(final_dev, rep.alloc_masks())
    return by_device


@pytest.mark.gpu
def test_daemonset_with_device_volumes_agrees_with_and_without_the_pinned_run():
    """A DaemonSet whose template asks for a 50Gi HDD: one pod pinned per node; the pinned-run fast path and the general path agree,
    pods pinned to nodes without a free HDD of 50Gi or more are refused, and the device state matches."""
    from simon_b200.engine import Engine
    from simon_b200.workloads import make_valid_pods_by_daemonset
    rng = np.random.default_rng(7)
    nodes = [_node(f"n{i:03d}", [], [_dev("/dev/h0", int(rng.choice([20, 50, 100])) * GI, alloc=bool(i % 7 == 0))])
             if i % 4 else _node(f"n{i:03d}", annotated=False) for i in range(60)]
    ds = {"apiVersion": "apps/v1", "kind": "DaemonSet", "metadata": {"name": "ds", "namespace": "default"},
          "spec": {"template": {"metadata": {"annotations": {O.ANNO_POD_LOCAL_STORAGE: json.dumps({"volumes": [_vol(50 * GI, "HDD")]})}},
                                "spec": {"containers": [{"name": "c", "image": "x", "resources": {"requests": {"cpu": "100m"}}}]}}}}
    pods = make_valid_pods_by_daemonset(ds, nodes) + [_pod(f"p{j}", [_vol(10 * GI, "HDD")]) for j in range(40)]
    c = compile_cluster(nodes, pods, open_local=True, storage_classes=SCS, local_devices=True)
    assert any(c.classes[k].pinned and c.storage.class_local[k] for k in range(len(c.classes)))
    res = []
    for fast in (True, False):
        with Engine(c, pin_fast=fast) as eng:
            out = eng.schedule()[0]
            res.append((out, eng.device_state()))
    assert np.array_equal(res[0][0], res[1][0]) and np.array_equal(res[0][1], res[1][1])
    out = res[0][0]
    for i in range(60):
        g = c.node_index(O.name_of(nodes[i]))
        st = c.storage
        free = st.node_n_hdd[g] == 1 and not st.dev_alloc[g] and st.dev_capacity[0, g] >= 50 * GI
        assert (out[i] >= 0) == free, i
    assert (out[:60] >= 0).sum() > 0 and (out[:60] == -1).sum() > 0


@pytest.mark.gpu
def test_two_passes_separated_by_a_state_reset_are_identical():
    from simon_b200.engine import Engine
    nodes, pods = _random_cluster(np.random.default_rng(21), 300, 1200)
    c = compile_cluster(nodes, pods, open_local=True, storage_classes=SCS, local_devices=True)
    with Engine(c) as eng:
        a = eng.schedule()[0], eng.storage_state(), eng.device_state()
        assert a[2].any()
        eng.reset()
        assert np.array_equal(eng.device_state(), c.storage.dev_alloc)
        b = eng.schedule()[0], eng.storage_state(), eng.device_state()
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


@pytest.mark.gpu
def test_abi_refusals():
    """simon_devices_upload: SIMON_ERR_STATE before simon_storage_upload, SIMON_ERR_INVALID / LIMIT on malformed columns; a scenario
    batch stays refused after it; a new storage upload drops the device tables."""
    from simon_b200 import abi
    from simon_b200.engine import Engine, lib
    L = lib()
    nodes = [_node("a", [100 * GI], [_dev("s", 50 * GI, "ssd"), _dev("h0", 100 * GI), _dev("h1", 200 * GI)]), _node("b", annotated=False)]
    pods = [_pod("p0", [_vol(GI, "HDD")]), _pod("q", None)]
    c = compile_cluster(nodes, pods, open_local=True, storage_classes=SCS, local_devices=True)
    st = c.storage
    plain = compile_cluster(nodes, [_pod("q", None)])
    with Engine(plain) as eng:
        s, _k = abi.marshal_devices(st)
        assert L.simon_devices_upload(eng.h, ctypes.byref(s)) == -3
        m = np.zeros(2, np.uint32)
        assert L.simon_devices_state_download(eng.h, m.ctypes.data) == -3
    with Engine(c) as eng:
        k_local = next(k for k in range(len(c.classes)) if st.class_local[k])
        k_plain = 1 - k_local
        g = c.node_index("a")

        def upload(**changes):
            import copy
            t = copy.copy(st)
            for name, val in changes.items():
                setattr(t, name, val)
            s, keep = abi.marshal_devices(t)
            return L.simon_devices_upload(eng.h, ctypes.byref(s))
        cap = st.dev_capacity.copy()
        cap[1, g], cap[2, g] = cap[2, g], cap[1, g]
        assert upload(dev_capacity=cap) == -1                           # HDD slots not ascending
        alloc = st.dev_alloc.copy()
        alloc[g] = 1 << 3
        assert upload(dev_alloc=alloc) == -1                            # allocated bit of an empty slot
        n_hdd = st.node_n_hdd.copy()
        n_hdd[g] = 3
        assert upload(node_n_hdd=n_hdd) == -1                           # more devices than slots
        off = np.zeros(3, np.uint32)
        off[k_plain + 1:] = 1
        assert upload(ssd_off=off, ssd_size=np.array([GI], np.int64)) == -1     # device volume on a class without the local flag
        assert upload(hdd_size=np.zeros_like(st.hdd_size)) == -1        # size 0
        assert upload(n_dev_slots=17) == -4
        off = np.zeros(3, np.uint32)
        off[k_local + 1:] = 9
        assert upload(hdd_off=off, hdd_size=np.full(9, GI, np.int64)) == -4     # more than 8 device volumes
        assert upload() == 0
        out = eng.schedule()[0]
        assert out[[i for i in range(2) if int(c.pods["pod_class"][i]) == k_local][0]] == g
        assert eng.device_state()[g] == 1 << 1
        with pytest.raises(RuntimeError):
            eng.run_scenarios([np.arange(c.n_nodes, dtype=np.uint32)])
        assert L.simon_storage_upload(eng.h, ctypes.byref(eng.storage)) == 0
        m = np.zeros(2, np.uint32)
        assert L.simon_devices_state_download(eng.h, m.ctypes.data) == -3
