"""Open-Local LVM volumes (pkg/simulator/plugin/open-local.go; OL = vendor/github.com/alibaba/open-local/pkg of the reference):
hand-derived known answers of the host restatement, the compiled storage columns, the refusals, and on the GPU the engine's
placements against the restated Filter and Bind."""
import json
import os

import numpy as np
import pytest

from simon_b200 import objects as O
from simon_b200.compiler import CompileError, compile_cluster
from simon_b200.storage import binary_si, lvm_place
from simon_b200.workloads import PodRec, PodTemplate

GI = 1 << 30
HERE = os.path.dirname(os.path.abspath(__file__))
EXAMPLE = os.path.join(HERE, "golden", "reference", "example")


def test_binary_si_string():
    """resource.NewQuantity(x, BinarySI).String(): |x| < 1024 stays decimal (quantity.go CanonicalizeBytes), otherwise the largest
    power of 1024 dividing x is the suffix (amount.go AsCanonicalBase1024Bytes, suffix.go)."""
    assert binary_si(107374182400) == "100Gi"
    assert binary_si(40 * GI) == "40Gi"
    assert binary_si(90 * GI) == "90Gi"
    assert binary_si(0) == "0"
    assert binary_si(1000) == "1000"
    assert binary_si(1536) == "1536"
    assert binary_si(1 << 20) == "1Mi"
    assert binary_si(3 * 1024 + 0) == "3Ki"
    assert binary_si(-2048) == "-2Ki"
    assert binary_si(1 << 62) == "4Ei"


def test_binpack_takes_the_least_free_vg_and_ties_in_annotation_order():
    """Binpack (common.go:574-619): VGs sorted by free size ascending, first that holds the PVC.  A: free 100Gi, B: free 60Gi,
    C: free 60Gi -> a 50Gi PVC goes to B (least free that fits; B before C by annotation order), a second 50Gi PVC to C (B has
    10Gi left), and a 20Gi PVC to A (B and C have 10Gi left).  ScoreLVM (:660-692): per VG used by this pod, size / capacity,
    summed in annotation order: 0.2 + 0.5 + 0.5 = 1.2 in float64, / 3 = 0.39999999999999997, * 10 = 3.9999999999999996 -> int 3."""
    vgs = [["A", 100 * GI, 0], ["B", 100 * GI, 40 * GI], ["C", 100 * GI, 40 * GI]]
    err, units, score = lvm_place("n1", vgs, [(50 * GI, ""), (50 * GI, ""), (20 * GI, "")])
    assert err is None
    assert units == [(1, 50 * GI), (2, 50 * GI), (0, 20 * GI)]
    assert score == 3


def test_named_vg_first_and_its_errors():
    """ProcessLVMPVCPredicate (common.go:59-143): PVCs whose class names a vgName are processed first, whatever their position;
    a missing VG is NotSuchVGError "not LVM named <vg>" (errors/predicate.go:44-57); too little free space on it is
    InsufficientLVMError with that VG's requested / capacity (:90-110)."""
    vgs = [["pool0", 100 * GI, 0], ["pool1", 100 * GI, 0]]
    err, units, score = lvm_place("n1", vgs, [(10 * GI, ""), (30 * GI, "pool1")])
    # pool1 takes 30Gi first (free 70Gi), then the 10Gi PVC goes to the least free VG: pool1
    assert err is None and units == [(1, 30 * GI), (1, 10 * GI)]
    assert score == int(40 / 100 * 10)
    assert lvm_place("n1", vgs, [(1 * GI, "nope")])[0] == "not LVM named nope"
    err = lvm_place("n1", [["pool0", 100 * GI, 90 * GI]], [(40 * GI, "pool0")])[0]
    assert err == "Insufficient LVM storage, requested 40Gi, used 90Gi, capacity 100Gi"


def test_no_vg_and_insufficient_lvm_report_the_last_vg():
    """A node with zero VGs: NoAvailableVGError "not LVM on node <name>" (predicate.go:60-78).  No VG holds the PVC: the error
    names the LAST VG of the sorted slice = the one with the most free space (ties: the later one in annotation order)."""
    assert lvm_place("w1", [], [(GI, "")])[0] == "not LVM on node w1"
    vgs = [["a", 100 * GI, 70 * GI], ["b", 50 * GI, 20 * GI], ["c", 10 * GI, 0]]
    err = lvm_place("w1", vgs, [(40 * GI, "")])[0]
    # free: a 30Gi, b 30Gi, c 10Gi -> sorted c, a, b: the last is b
    assert err == "Insufficient LVM storage, requested 40Gi, used 20Gi, capacity 50Gi"


def test_zero_valued_vgs_ahead_of_the_real_ones():
    """Quirk 4 (common.go:98-101): make([]SharedResource, len(map)) + append leaves len(map) zero-valued VGs in the slice.  When
    every real VG is over-committed (free < 0) a zero entry (free 0) sorts last, so the error reports used 0, capacity 0."""
    err = lvm_place("w1", [["a", 10 * GI, 20 * GI]], [(GI, "")])[0]
    assert err == "Insufficient LVM storage, requested 1Gi, used 0, capacity 0"


def _node(name, storage=None, taint=False):
    n = {"apiVersion": "v1", "kind": "Node",
         "metadata": {"name": name, "labels": {"kubernetes.io/hostname": name}, "annotations": {}},
         "status": {"allocatable": {"cpu": "16", "memory": "64Gi", "pods": "110"}}}
    if storage is not None:
        n["metadata"]["annotations"][O.ANNO_NODE_LOCAL_STORAGE] = storage if isinstance(storage, str) else json.dumps(storage)
    if taint:
        n["spec"] = {"taints": [{"key": "k", "value": "v", "effect": "NoSchedule"}]}
    return n


def _vgs(*caps):
    return {"vgs": [{"name": f"vg{i}", "capacity": str(c), "requested": "0"} for i, c in enumerate(caps)]}


def _pod(name, vols):
    ann = {O.ANNO_POD_LOCAL_STORAGE: json.dumps({"volumes": vols})}
    pod = {"apiVersion": "v1", "kind": "Pod", "metadata": {"name": name, "namespace": "default", "annotations": ann},
           "spec": {"containers": [{"name": "c", "image": "x", "resources": {"requests": {"cpu": "100m", "memory": "128Mi"}}}]}}
    return PodRec(PodTemplate(pod, "Pod", name, "default"), name, 0)


def _lvm(size, sc="open-local-lvm"):
    return {"size": str(size), "kind": "LVM", "scName": sc}


def test_refused_without_the_opt_in_and_compiled_with_it():
    nodes = [_node("a", _vgs(100 * GI)), _node("b")]
    pods = [_pod("p0", [_lvm(10 * GI)])]
    with pytest.raises(CompileError):
        compile_cluster(nodes, pods)
    c = compile_cluster(nodes, pods, open_local=True)
    st = c.storage
    assert st.n_vgs == 1
    assert st.node_n_vg.tolist() == [1, -1]
    assert st.vg_capacity[0, 0] == 100 * GI
    assert st.class_local.tolist() == [1]
    assert st.vol_off.tolist() == [0, 1] and st.vol_size.tolist() == [10 * GI] and st.vol_vg.tolist() == [-1]


@pytest.mark.parametrize("storage, msg", [
    ("{not json", "malformed"),
    ({"vgs": [{"name": "x", "capacity": "1", "requested": "0"}, {"name": "x", "capacity": "2", "requested": "0"}]}, "duplicate VG"),
    ({"vgs": [{"name": "", "capacity": "1", "requested": "0"}]}, "named"),
    ({"vgs": [{"name": "x", "capacity": 5, "requested": "0"}]}, "quoted"),
    ({"vgs": [], "devices": [{"name": "d", "device": "/dev/a", "capacity": "1", "mediaType": "hdd", "isAllocated": "false"},
                             {"name": "e", "device": "/dev/a", "capacity": "1", "mediaType": "hdd", "isAllocated": "false"}]},
     "duplicate device"),
    (_vgs(*([GI] * 9)), "more than 8 VGs"),
])
def test_node_annotation_refusals(storage, msg):
    with pytest.raises(CompileError, match=msg):
        compile_cluster([_node("a", storage)], [_pod("p0", [_lvm(GI)])], open_local=True)


def test_volume_refusals():
    nodes = [_node("a", _vgs(100 * GI))]
    with pytest.raises(CompileError, match="size 0"):
        compile_cluster(nodes, [_pod("p0", [_lvm(0)])], open_local=True)
    with pytest.raises(CompileError, match="more than 8"):
        compile_cluster(nodes, [_pod("p0", [_lvm(GI)] * 9)], open_local=True)
    with pytest.raises(CompileError, match="size 0"):
        compile_cluster(nodes, [_pod("p0", [{"size": "0", "kind": "HDD", "scName": "yoda-device-hdd"}])], open_local=True)
    sc = {"apiVersion": "storage.k8s.io/v1", "kind": "StorageClass", "metadata": {"name": "open-local-device-hdd"},
          "parameters": {"mediaType": "hdd"}}
    with pytest.raises(CompileError, match="exclusive"):
        compile_cluster(nodes, [_pod("p0", [{"size": str(GI), "kind": "HDD", "scName": "open-local-device-hdd"}])],
                        open_local=True, storage_classes=[sc])


def test_dropped_device_volumes_compile_to_no_lvm_volume():
    """Quirk 1 (DividePVCAccordingToMediaType, common.go:247-260): a device PVC whose class is missing is dropped; the pod still
    requests local storage (GetPodLocalPVCs counted it), so nodes without the annotation fail, and it has no LVM volume."""
    c = compile_cluster([_node("a", _vgs(GI)), _node("b")], [_pod("p0", [{"size": str(GI), "kind": "HDD", "scName": "yoda-device-hdd"}])],
                        open_local=True)
    assert c.storage.class_local.tolist() == [1]
    assert c.storage.vol_off.tolist() == [0, 0]


def _example(apps):
    from simon_b200.objects import AppResource, create_cluster_resource_from_cluster_config, get_object_from_yaml_content, \
        get_yaml_content_from_directory
    cluster = create_cluster_resource_from_cluster_config(os.path.join(EXAMPLE, "cluster", "demo_1"))
    out = []
    for a in apps:
        out.append(AppResource(a, get_object_from_yaml_content(get_yaml_content_from_directory(
            os.path.join(EXAMPLE, "application", a)))))
    return cluster, out


def test_example_storage_columns():
    """demo_1: master-1 and worker-1 carry two 100Gi VGs each; the open_local StatefulSet asks for 10Gi + 40Gi on yoda-lvm-default
    (no vgName: Binpack) and 100Gi on yoda-device-hdd, a class demo_1 does not define (dropped, quirk 1)."""
    from simon_b200.simulator import plan
    cluster, apps = _example(["open_local"])
    p = plan(cluster, apps)
    c = compile_cluster(p.nodes, p.pods, p.ctx, open_local=True, storage_classes=list(cluster.StorageClasss))
    st = c.storage
    names = c.node_names
    with_vg = sorted(names[g] for g in range(c.n_nodes) if st.node_n_vg[g] >= 0)
    assert with_vg == ["master-1", "worker-1"]
    sts = [cid for cid, cl in enumerate(c.classes) if st.class_local[cid]]
    assert len(sts) == 1
    k = sts[0]
    assert st.vol_size[st.vol_off[k]:st.vol_off[k + 1]].tolist() == [10 * GI, 40 * GI]
    assert st.vol_vg[st.vol_off[k]:st.vol_off[k + 1]].tolist() == [-1, -1]


@pytest.mark.gpu
def test_example_open_local_on_gpu():
    """Known answer: only master-1 and worker-1 have storage, master-1 is tainted NoSchedule, so the 4 nginx-lvm pods land on
    worker-1.  Each pod's 10Gi + 40Gi go to the least free VG that holds them: pods 0-1 fill yoda-pool0 (0 -> 50 -> 100Gi),
    pods 2-3 fill yoda-pool1; /dev/vdd stays unallocated (its PVC was dropped).  Bind's annotation is what NodeStatus carries."""
    from simon_b200.simulator import Simulate, WithOpenLocal
    cluster, apps = _example(["open_local"])
    res = Simulate(cluster, apps, WithOpenLocal())
    assert res.UnscheduledPods == []
    placed = {}
    for ns in res.NodeStatus:
        for p in ns.Pods:
            if p.name.startswith("nginx-lvm"):
                placed[p.name] = O.name_of(ns.Node)
    assert placed == {f"nginx-lvm-{i}": "worker-1" for i in range(4)}
    w = next(ns.Node for ns in res.NodeStatus if O.name_of(ns.Node) == "worker-1")
    ann = json.loads(O.annotations_of(w)[O.ANNO_NODE_LOCAL_STORAGE])
    assert [v["requested"] for v in ann["vgs"]] == ["107374182400", "107374182400"]
    assert ann["devices"][0]["isAllocated"] == "false"


def _random_cluster(rng, n_nodes, n_pods):
    nodes = []
    for i in range(n_nodes):
        r = rng.random()
        if r < 0.15:
            nodes.append(_node(f"n{i:05d}"))
        else:
            nv = int(rng.integers(0, 4))
            vgs = {"vgs": [{"name": f"pool{v}", "capacity": str(int(rng.integers(1, 20)) * 10 * GI),
                            "requested": str(int(rng.integers(0, 5)) * 10 * GI)} for v in range(nv)]}
            nodes.append(_node(f"n{i:05d}", vgs))
    scs = [{"apiVersion": "storage.k8s.io/v1", "kind": "StorageClass", "metadata": {"name": "open-local-lvm"},
            "parameters": {"vgName": "pool1"}}] if rng.random() < 0.3 else []
    pods = []
    for j in range(n_pods):
        r = rng.random()
        if r < 0.3:
            vols = []
        elif r < 0.9:
            vols = [_lvm(int(rng.integers(1, 8)) * 5 * GI, "yoda-lvm-default") for _ in range(int(rng.integers(1, 4)))]
            if rng.random() < 0.3:
                vols.append(_lvm(int(rng.integers(1, 4)) * 5 * GI, "open-local-lvm"))
        else:
            vols = [{"size": str(GI), "kind": "SSD", "scName": "yoda-device-ssd"}]
        pods.append(_pod(f"p{j:05d}-{len(vols)}", vols) if vols else _pod(f"q{j:05d}", []))
        if not vols:
            del pods[-1].tmpl.pod["metadata"]["annotations"][O.ANNO_POD_LOCAL_STORAGE]
    return nodes, pods, scs


@pytest.mark.gpu
@pytest.mark.parametrize("seed, n_nodes, n_pods, pin_fast", [(1, 40, 300, True), (2, 700, 2000, True), (3, 3000, 4000, False),
                                                              (4, 250, 1500, True), (5, 41000, 1500, True)])
def test_engine_follows_the_restated_filter_and_bind(seed, n_nodes, n_pods, pin_fast):
    """Every storage pod the engine places passes the restated Open-Local Filter on the node state of its turn; a refused storage
    pod reports Open-Local rejections (or every node failed an earlier filter); the engine's final VG state equals the replay of
    Bind in placement order.  Sizes up to 41,000 nodes cover the large-cluster kernel variant."""
    from simon_b200.engine import Engine
    from simon_b200.storage import StorageReplay
    rng = np.random.default_rng(seed)
    nodes, pods, scs = _random_cluster(rng, n_nodes, n_pods)
    c = compile_cluster(nodes, pods, open_local=True, storage_classes=scs)
    with Engine(c, pin_fast=pin_fast) as eng:
        out, _s, fail_counts, fail_pod = eng.schedule()
        final = eng.storage_state()
        rep = StorageReplay(c.storage, c.node_names)
        fails = {int(p): j for j, p in enumerate(fail_pod)}
        pod_class = c.pods["pod_class"]
        for i, n in enumerate(out.tolist()):
            cls = int(pod_class[i])
            if n >= 0:
                if c.storage.class_local[cls]:
                    assert rep.reason(cls, n) is None and c.storage.node_n_vg[n] >= 0
                    rep.bind(cls, n)
            else:
                assert n == -1 and i in fails
                if c.storage.class_local[cls]:
                    assert int(fail_counts[fails[i]][20]) > 0 or int(fail_counts[fails[i]].sum()) == c.n_nodes
        assert np.array_equal(final, rep.requested())
        assert (out >= 0).sum() > 0


def test_no_lvm_volume_passes_any_annotated_node():
    """ProcessLVMPVCPredicate runs only when the pod has LVM PVCs (open-local.go:76-81); dropped device PVCs pass ProcessDevicePVC
    with zero units (common.go:394-448).  So a pod whose only volumes are dropped device PVCs passes a node whose annotation has no
    VG at all - NoAvailableVGError is an LVM error - and ScoreLVMVolume returns 0 for it (:500-503)."""
    assert lvm_place("w1", [], []) == (None, [], 0)
    assert lvm_place("w1", None, []) == (None, [], 0)
    assert lvm_place("w1", [["a", GI, GI]], []) == (None, [], 0)


def test_normalisation_and_the_dropped_device_offset():
    """NormalizeScore (open-local.go:146-171): (s - lowest) * 100 / (highest - lowest), 0 for a zero range.  A class whose device
    PVCs were all dropped adds ScoreDevice of no units = int(NaN) = MinInt64 (common.go:753-762, amd64) to every node's raw score:
    the differences, so the normalised scores, are those of the LVM part alone.  With the LVM part 0 everywhere every raw score is
    MinInt64, below the loop's start value highest = -MaxInt64, so the range is -MaxInt64 - MinInt64 = 1 and every score is
    (MinInt64 - MinInt64) * 100 / 1 = 0 - the same as a zero range."""
    from simon_b200.storage import INT64_MIN, ClassVolumes, normalize_scores, raw_score
    assert normalize_scores([2, 5, 9]) == [0, 42, 100]
    assert normalize_scores([3, 3]) == [0, 0]
    dropped = ClassVolumes(local=True, lvm=[(GI, "")], dropped=1)
    raws = [raw_score(dropped, s) for s in (3, 7, 3)]
    assert raws == [INT64_MIN + 3, INT64_MIN + 7, INT64_MIN + 3]
    assert normalize_scores(raws) == normalize_scores([3, 7, 3]) == [0, 100, 0]
    only_dropped = ClassVolumes(local=True, lvm=[], dropped=1)
    assert normalize_scores([raw_score(only_dropped, 0)] * 3) == [0, 0, 0]


def _oracle_cluster(rng, n_nodes, n_pods):
    """Nodes of one allocatable shape and bare pods without affinity, spread or taints: every score plugin but Open-Local then
    gives the same per-node score whatever the feasible set is, so the CPU port's totals hold with Open-Local's filter on top."""
    nodes = []
    for i in range(n_nodes):
        r = rng.random()
        if r < 0.15:
            nodes.append(_node(f"n{i:05d}"))
        elif r < 0.25:
            nodes.append(_node(f"n{i:05d}", rng.choice(["null", '{"vgs": []}', '{"devices": [{"name": "d", "device": "/dev/d", '
                                                         '"capacity": "1", "mediaType": "hdd", "isAllocated": "false"}]}'])))
        else:
            nv = int(rng.integers(1, 4))
            nodes.append(_node(f"n{i:05d}", {"vgs": [{"name": f"pool{v}", "capacity": str(int(rng.integers(1, 20)) * 10 * GI),
                                                      "requested": str(int(rng.integers(0, 5)) * 10 * GI)} for v in range(nv)]}))
    scs = [{"apiVersion": "storage.k8s.io/v1", "kind": "StorageClass", "metadata": {"name": "open-local-lvm"},
            "parameters": {"vgName": "pool1"}}]
    pods = []
    for j in range(n_pods):
        r = rng.random()
        if r < 0.25:
            p = _pod(f"q{j:05d}", [])
            del p.tmpl.pod["metadata"]["annotations"][O.ANNO_POD_LOCAL_STORAGE]
        elif r < 0.35:
            p = _pod(f"d{j:05d}", [{"size": str(GI), "kind": "SSD", "scName": "yoda-device-ssd"}])
        else:
            vols = [_lvm(int(rng.integers(1, 8)) * 5 * GI, "yoda-lvm-default") for _ in range(int(rng.integers(1, 4)))]
            if rng.random() < 0.25:
                vols.append(_lvm(int(rng.integers(1, 4)) * 5 * GI, "open-local-lvm"))
            if rng.random() < 0.2:
                vols.append({"size": str(GI), "kind": "HDD", "scName": "yoda-device-hdd"})
            p = _pod(f"p{j:05d}-{len(vols)}", vols)
        pods.append(p)
    return nodes, pods, scs


@pytest.mark.gpu
@pytest.mark.parametrize("seed, n_nodes, n_pods", [(11, 30, 160), (12, 200, 300), (13, 700, 250), (14, 41000, 60)])
def test_engine_matches_cpu_port_with_restated_open_local(seed, n_nodes, n_pods):
    """Node and recorded winning score of every pod against an independent composition: the CPU port (oracle/simon_oracle.c,
    which has no Open-Local) replays the engine's earlier placements as bound pods and scores the pod's cycle; Open-Local's
    Filter, ScoreLVM and NormalizeScore are applied on top from the VG state the engine's earlier Binds left (storage.py).
    Clusters with several feasible storage nodes whose raw scores differ exercise the score path; 41,000 nodes the
    large-cluster variant; zero-VG annotated nodes and dropped-device-only pods the no-LVM case."""
    from simon_b200.engine import Engine
    rng = np.random.default_rng(seed)
    nodes, pods, scs = _oracle_cluster(rng, n_nodes, n_pods)
    c = compile_cluster(nodes, pods, open_local=True, storage_classes=scs)
    with Engine(c, record_scores=True) as eng:
        out, score, _fc, _fp = eng.schedule()
        final = eng.storage_state()
    assert check_restated_open_local(c, out, score, final) > 0     # the score path decided some placements


def check_restated_open_local(c, out, score, final):
    """The composition above, pod by pod, for an engine run of a cluster of _oracle_cluster: out / score are its placements and
    recorded winning scores, final its VG requested state.  Returns the number of storage pods that had several feasible nodes
    with different raw Open-Local scores."""
    import ctypes
    from oracle.binding import Oracle
    orc = Oracle(c)
    orc.enable_dump()
    # the oracle reads c's own pod_fixed_node array: it is restored afterwards, so that c can be checked again
    fixed = np.ctypeslib.as_array((ctypes.c_int32 * c.pods_dims["n_pods"]).from_address(orc.pods.pod_fixed_node))
    orig = fixed.copy()
    try:
        return _restated_open_local_pods(c, out, score, final, orc, fixed, orig)
    finally:
        fixed[:] = orig
        orc.close()


def _restated_open_local_pods(c, out, score, final, orc, fixed, orig):
    from simon_b200.storage import StorageReplay, lvm_place, normalize_scores
    st = c.storage
    P = c.pods_dims["n_pods"]
    rep = StorageReplay(st, c.node_names)
    pod_class = c.pods["pod_class"]
    multi = 0
    for i in range(P):
        assert orig[i] == -1
        fixed[:i] = np.where(out[:i] >= 0, out[:i], -2)
        fixed[i] = -1
        orc.reset()
        orc.schedule(0, i + 1)
        code, sc = orc.last_detail()
        cls = int(pod_class[i])
        cv = st.class_volumes[cls]
        feas = [g for g in range(c.n_nodes) if code[g] == 0]
        raw = {}
        if st.class_local[cls]:
            keep = []
            for g in feas:
                ns = st.node_storage[g]
                if ns is None:
                    continue
                err, _u, s = lvm_place(c.node_names[g], rep.vgs[g], cv.lvm)
                if err is None:
                    keep.append(g)
                    raw[g] = s
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
            if st.class_local[cls] and len(set(raw.values())) > 1:
                multi += 1
        if st.class_local[cls]:
            rep.bind(cls, int(out[i]))
    assert np.array_equal(final, rep.requested())
    return multi


@pytest.mark.gpu
def test_daemonset_pods_with_volumes_agree_with_and_without_the_pinned_run():
    """A DaemonSet whose template carries LVM volumes: its pods are pinned, one per node, and with the fast path on the engine
    would place a run of them by the pin node's node-local filters alone.  simon_storage_upload takes them off it, so both paths
    agree, pods pinned to nodes without storage or VG room are refused, and the VG state matches."""
    from simon_b200.engine import Engine
    from simon_b200.workloads import make_valid_pods_by_daemonset
    rng = np.random.default_rng(5)
    nodes = [_node(f"n{i:03d}", _vgs(int(rng.integers(1, 6)) * 10 * GI) if i % 4 else None) for i in range(60)]
    ds = {"apiVersion": "apps/v1", "kind": "DaemonSet", "metadata": {"name": "ds", "namespace": "default"},
          "spec": {"template": {"metadata": {"annotations": {O.ANNO_POD_LOCAL_STORAGE: json.dumps({"volumes": [_lvm(25 * GI)]})}},
                                "spec": {"containers": [{"name": "c", "image": "x",
                                                         "resources": {"requests": {"cpu": "100m"}}}]}}}}
    pods = make_valid_pods_by_daemonset(ds, nodes) + [_pod(f"p{j}", [_lvm(10 * GI)]) for j in range(40)]
    c = compile_cluster(nodes, pods, open_local=True)
    assert any(c.classes[k].pinned and c.storage.class_local[k] for k in range(len(c.classes)))
    res = []
    for fast in (True, False):
        with Engine(c, pin_fast=fast) as eng:
            out = eng.schedule()[0]
            res.append((out, eng.storage_state()))
    assert np.array_equal(res[0][0], res[1][0]) and np.array_equal(res[0][1], res[1][1])
    out = res[0][0]
    n_ds = 60
    for i in range(n_ds):
        g = c.node_index(O.name_of(nodes[i]))
        if c.storage.node_n_vg[g] < 0 or c.storage.vg_capacity[0, g] < 25 * GI:
            assert out[i] == -1, i
    assert (out[:n_ds] >= 0).sum() > 0 and (out[:n_ds] == -1).sum() > 0


def test_native_host_refuses_the_open_local_opt_in():
    """The native host side does not implement Open-Local: a request that asks for it is refused (SIMON_ERR_LIMIT), not run with
    the volumes refused or ignored differently from the Python host side."""
    import ctypes
    from simon_b200 import native_host
    L = native_host.lib()
    h = ctypes.c_void_p()
    req = json.dumps({"cluster": {"Nodes": [_node("a", _vgs(GI))]}, "apps": [], "openLocal": True}).encode()
    assert L.simon_host_compile(req, len(req), ctypes.byref(h)) == -4
    assert b"openLocal" in L.simon_host_last_error()
    req = json.dumps({"cluster": {"Nodes": [_node("a", _vgs(GI))]}, "apps": [], "openLocal": False}).encode()
    assert L.simon_host_compile(req, len(req), ctypes.byref(h)) == 0
    L.simon_host_plan_free(h)
