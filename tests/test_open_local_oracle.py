"""Open-Local in the CPU oracle (oracle/simon_oracle.c, Oracle(c, open_local=True)) on clusters that mix it with every other
plugin: against the object-level reference (oracle/pyref.py with Open-Local), against the restated compositions of
test_open_local.py / test_open_local_devices.py on their own clusters, and on the reference example's known answers.  The coverage
test counts, on the oracle side, the decisions where Open-Local changes the feasible set that the other plugins read, so that the
GPU tests of tests/test_zz_open_local_oracle_gpu.py (which compare every Open-Local kernel path with this oracle) exercise them.

make_mixed_local is the generator both modules use: synth.make_mix (every predicate, GPU share, pre-bound pods, DaemonSets,
StatefulSets, Jobs and bare pods) with Open-Local layered on top."""
import json
import os

import numpy as np
import pytest

from simon_b200 import abi, simulator, synth
from simon_b200 import objects as O
from simon_b200.compiler import compile_cluster
from util import assert_matches_walk, pyref_walk

GI = 1 << 30
HERE = os.path.dirname(os.path.abspath(__file__))

# the StorageClasses of the generator: Binpack LVM, LVM with a vgName, both device media types, and one whose mediaType no
# device has (DividePVCAccordingToMediaType drops its PVCs, common.go:247-260)
STORAGE_CLASSES = [
    {"apiVersion": "storage.k8s.io/v1", "kind": "StorageClass", "metadata": {"name": "open-local-lvm"}, "parameters": {}},
    {"apiVersion": "storage.k8s.io/v1", "kind": "StorageClass", "metadata": {"name": "yoda-lvm-default"},
     "parameters": {"vgName": "pool1"}},
    {"apiVersion": "storage.k8s.io/v1", "kind": "StorageClass", "metadata": {"name": "open-local-device-ssd"},
     "parameters": {"mediaType": "ssd"}},
    {"apiVersion": "storage.k8s.io/v1", "kind": "StorageClass", "metadata": {"name": "open-local-device-hdd"},
     "parameters": {"mediaType": "hdd"}},
    {"apiVersion": "storage.k8s.io/v1", "kind": "StorageClass", "metadata": {"name": "yoda-device-hdd"},
     "parameters": {"mediaType": "nvme"}},
]


def _node_storage(rng):
    """A node annotation: 0-3 VGs of a few volumes' worth (some nodes none at all), 0-6 SSD / HDD devices with capacity ties, a
    few allocated, and sometimes a device of another media type."""
    if rng.random() < 0.12:
        vgs = []
    else:
        vgs = [{"name": f"pool{v}", "capacity": str(int(rng.choice([20, 30, 40, 60, 80])) * GI),
                "requested": str(int(rng.choice([0, 0, 0, 5, 10])) * GI)} for v in range(int(rng.integers(1, 4)))]
    devs = []
    for k in range(int(rng.integers(0, 7))):
        devs.append({"name": f"/dev/vd{k}", "device": f"/dev/vd{k}", "capacity": str(int(rng.choice([50, 100, 100, 200])) * GI),
                     "mediaType": str(rng.choice(["ssd", "hdd"])), "isAllocated": "true" if rng.random() < 0.1 else "false"})
    if rng.random() < 0.2:
        devs.append({"name": "/dev/nv0", "device": "/dev/nv0", "capacity": str(400 * GI), "mediaType": "nvme",
                     "isAllocated": "false"})
    return {"vgs": vgs, "devices": devs}


def _volumes(rng):
    """A workload's volumes: LVM only (Binpack and vgName), devices only, both, or only PVCs that are dropped, with or without
    LVM ones."""
    kind = int(rng.integers(0, 5))
    vols = []
    if kind in (0, 2, 4):
        for _ in range(int(rng.integers(1, 4))):
            sc = "yoda-lvm-default" if rng.random() < 0.25 else "open-local-lvm"
            vols.append({"size": str(int(rng.choice([5, 10, 15, 20, 25])) * GI), "kind": "LVM", "scName": sc})
    if kind in (1, 2):
        for _ in range(int(rng.integers(1, 3))):
            m = str(rng.choice(["SSD", "HDD"]))
            vols.append({"size": str(int(rng.choice([40, 80, 100, 150])) * GI), "kind": m, "scName": f"open-local-device-{m.lower()}"})
    if kind in (3, 4):
        vols.append({"size": str(10 * GI), "kind": "HDD", "scName": "yoda-device-hdd"})
    return vols


def _vcts(vols):
    """The volumeClaimTemplates a StatefulSet states the same volumes with (SetStorageAnnotationOnPods)."""
    return [{"metadata": {"name": f"v{i}"}, "spec": {"storageClassName": v["scName"], "resources": {"requests": {"storage": v["size"]}}}}
            for i, v in enumerate(vols)]


def _annotate(meta, vols):
    meta["annotations"] = dict(meta.get("annotations") or {}, **{O.ANNO_POD_LOCAL_STORAGE: json.dumps({"volumes": vols})})


def make_mixed_local(seed, n_nodes=40, n_workloads=30, max_replicas=6, devices=True):
    """synth.make_mix with Open-Local layered on top: the annotation on about 2/3 of the nodes, StorageClasses of every kind, and
    volumes on a random half of the workload templates of every kind (Deployments, StatefulSets, Jobs, bare pods, DaemonSets) and
    on some pre-bound pods, so that volumes cross spread, (anti-)affinity, taints and GPU share.  -> (plan, compiled cluster,
    PyRef's Open-Local setting)."""
    cluster, apps = synth.make_mix(seed_no=seed, n_nodes=n_nodes, n_workloads=n_workloads, max_replicas=max_replicas)
    rng = np.random.default_rng(0x0100CA1 + seed)
    for n in cluster.Nodes:
        if rng.random() < 0.67:
            O.meta(n).setdefault("annotations", {})
            O.meta(n)["annotations"][O.ANNO_NODE_LOCAL_STORAGE] = json.dumps(_node_storage(rng))
    cluster.StorageClasss.extend(STORAGE_CLASSES)
    for pod in cluster.Pods:                     # pre-bound pods: they hold volumes, but never go through Bind
        if rng.random() < 0.3:
            _annotate(pod["metadata"], _volumes(rng))
    res = apps[0].Resource
    for w in res.Deployments + res.Jobs + res.DaemonSets + cluster.DaemonSets:
        if rng.random() < 0.5:
            _annotate(w["spec"]["template"].setdefault("metadata", {}), _volumes(rng))
    for w in res.StatefulSets:
        if rng.random() < 0.5:
            w["spec"]["volumeClaimTemplates"] = _vcts(_volumes(rng))
    for w in res.Pods:
        if rng.random() < 0.5:
            _annotate(w["metadata"], _volumes(rng))
    p = simulator.plan(cluster, apps)
    c = compile_cluster(p.nodes, p.pods, p.ctx, open_local=True, storage_classes=list(cluster.StorageClasss),
                        local_devices=devices)
    return p, c, (list(cluster.StorageClasss), devices)


def oracle_run(c, threads=1):
    """A full oracle run with Open-Local: (out, score, fail_counts, fail_pod, VG state, device state)."""
    from oracle.binding import Oracle
    o = Oracle(c, threads=threads, open_local=True)
    try:
        out, score, fc, fp = o.schedule()
        vg, dev = o.storage_state()
        return out, score, fc, fp, vg, dev
    finally:
        o.close()


def _pyref_final(ref, c):
    """The VG requested [V][N] and device slot masks [N] of PyRef's nodes after its walk, in the layouts of the engine."""
    st = c.storage
    vg = np.array(st.vg_requested, copy=True).reshape(st.n_vgs, c.n_nodes)
    dev = np.zeros(c.n_nodes, np.uint32)
    for g, ns in enumerate(ref.nodes):
        for v, x in enumerate(ns.vgs or []):
            vg[v, g] = x[2]
        if st.devices and ns.devs:
            dev[g] = st.alloc_mask(g, ns.devs)
    return vg, dev


# ---- the oracle against the object-level reference on mixed clusters ----

MIX_SEEDS = list(range(300, 324))


@pytest.mark.parametrize("seed", MIX_SEEDS)
def test_oracle_matches_pyref_on_mixed_open_local(seed):
    """Per pod the node, the winning total and the failure histogram, and at the end the VG state and the device masks, of the
    oracle with Open-Local against PyRef with Open-Local on a mixed cluster."""
    p, c, ol = make_mixed_local(seed, n_nodes=30 + seed % 20, n_workloads=24, max_replicas=6)
    assert c.storage.class_local.any()
    out, score, fc, fp, vg, dev = oracle_run(c)
    refs = []
    walk = pyref_walk(p, c, open_local=ol, ref_out=refs)
    assert_matches_walk(walk, out, score, fc, fp, what=f"seed {seed}")
    rvg, rdev = _pyref_final(refs[0], c)
    np.testing.assert_array_equal(vg, rvg, err_msg="VG state")
    np.testing.assert_array_equal(dev, rdev, err_msg="device state")


def test_oracle_threads_do_not_change_open_local_results():
    """set_threads shares the per-node stages, the Open-Local ones included: the results do not depend on the thread count."""
    _p, c, _ol = make_mixed_local(7, n_nodes=300, n_workloads=60, max_replicas=8)
    a = oracle_run(c, threads=1)
    b = oracle_run(c, threads=5)
    for x, y in zip(a, b):
        np.testing.assert_array_equal(x, y)


def test_without_open_local_the_oracle_is_unchanged():
    """Oracle(c) without open_local has no Open-Local (the storage-less oracle the restated compositions use): it has no storage
    state, and on a cluster where Open-Local decides something its placements differ from Oracle(c, open_local=True)'s."""
    from oracle.binding import Oracle
    _p, c, _ol = make_mixed_local(3)
    o = Oracle(c)
    out = o.schedule()
    with pytest.raises(RuntimeError):
        o.storage_state()
    o.close()
    lo = oracle_run(c)
    assert (out[0] != lo[0]).any()      # Open-Local decides something on this cluster


# ---- the oracle against the restated compositions on their own clusters ----

def test_oracle_matches_restated_lvm_composition():
    """test_open_local.py's _oracle_cluster: the storage-less oracle with storage.py's Filter and Score on top is valid there.  The
    oracle with Open-Local places every pod on the same node with the same score, and ends in the same VG state."""
    from test_open_local import _oracle_cluster, check_restated_open_local
    for seed, n_nodes, n_pods in ((11, 30, 160), (12, 120, 300)):
        rng = np.random.default_rng(seed)
        nodes, pods, scs = _oracle_cluster(rng, n_nodes, n_pods)
        c = compile_cluster(nodes, pods, open_local=True, storage_classes=scs)
        out, score, _fc, _fp, vg, _dev = oracle_run(c)
        assert check_restated_open_local(c, out, score, vg) > 0


def test_oracle_matches_restated_device_composition():
    """test_open_local_devices.py's generator and composition, with the oracle with Open-Local as the run checked."""
    from test_open_local_devices import check_restated_devices, restated_cluster
    for seed, n_nodes, n_pods in ((11, 30, 160), (12, 200, 300)):
        c = restated_cluster(seed, n_nodes, n_pods)
        out, score, _fc, _fp, _vg, dev = oracle_run(c)
        assert check_restated_devices(c, out, score, dev) > 0


# ---- known answers ----

EXAMPLE = os.path.join(HERE, "golden", "reference", "example")


def _example(apps):
    from simon_b200.objects import AppResource, create_cluster_resource_from_cluster_config, get_object_from_yaml_content, \
        get_yaml_content_from_directory
    cluster = create_cluster_resource_from_cluster_config(os.path.join(EXAMPLE, "cluster", "demo_1"))
    out = [AppResource(a, get_object_from_yaml_content(get_yaml_content_from_directory(os.path.join(EXAMPLE, "application", a))))
           for a in apps]
    return cluster, out


def test_known_answer_reference_example():
    """The reference example: only master-1 and worker-1 have storage, master-1 is tainted NoSchedule, so the 4 nginx-lvm pods
    land on worker-1, and each pod's 10Gi + 40Gi fill yoda-pool0 (pods 0-1), then yoda-pool1 (pods 2-3): 100Gi requested each."""
    cluster, apps = _example(["open_local"])
    p = simulator.plan(cluster, apps)
    c = compile_cluster(p.nodes, p.pods, p.ctx, open_local=True, storage_classes=list(cluster.StorageClasss))
    out, _score, _fc, _fp, vg, _dev = oracle_run(c)
    w = c.node_index("worker-1")
    lvm = [i for i, r in enumerate(p.pods) if r.tmpl.pod["metadata"].get("name", "").startswith("nginx-lvm")
           or O.name_of(r.tmpl.pod).startswith("nginx-lvm")]
    assert len(lvm) == 4 and all(out[i] == w for i in lvm)
    assert vg[:, w].tolist() == [100 * GI, 100 * GI]
    m = c.node_index("master-1")
    np.testing.assert_array_equal(vg[:, m], c.storage.vg_requested.reshape(c.storage.n_vgs, -1)[:, m])


def test_known_answer_demo_1_devices():
    """demo_1 with three replicas of one 50Gi HDD volume each: master-1 is tainted and master-2/3 have no annotation, so hdd-0
    takes worker-1's only HDD (/dev/vdd) and hdd-1 / hdd-2 find no free HDD: unschedulable, master-1 failing its taint and every
    other node Open-Local (SFC_LOCAL: worker-1 for the HDD, the others for having no annotation)."""
    from simon_b200.objects import AppResource, ResourceTypes, create_cluster_resource_from_cluster_config
    cluster = create_cluster_resource_from_cluster_config(os.path.join(EXAMPLE, "cluster", "demo_1"))
    sts = {"apiVersion": "apps/v1", "kind": "StatefulSet", "metadata": {"name": "hdd", "namespace": "default"},
           "spec": {"replicas": 3, "serviceName": "hdd", "selector": {"matchLabels": {"app": "hdd"}},
                    "volumeClaimTemplates": [{"metadata": {"name": "data"}, "spec": {
                        "storageClassName": "open-local-device-hdd", "resources": {"requests": {"storage": "50Gi"}}}}],
                    "template": {"metadata": {"labels": {"app": "hdd"}}, "spec": {"containers": [
                        {"name": "c", "image": "x", "resources": {"requests": {"cpu": "100m", "memory": "128Mi"}}}]}}}}
    p = simulator.plan(cluster, [AppResource("hdd", ResourceTypes(StatefulSets=[sts]))])
    c = compile_cluster(p.nodes, p.pods, p.ctx, open_local=True, storage_classes=list(cluster.StorageClasss), local_devices=True)
    names = [O.name_of(r.tmpl.pod) if not r.name else r.name for r in p.pods]
    out, _score, fc, fp, _vg, dev = oracle_run(c)
    w, m = c.node_index("worker-1"), c.node_index("master-1")
    assert out[names.index("hdd-0")] == w
    assert dev[w] == 1 and dev[m] == 0
    for nm in ("hdd-1", "hdd-2"):
        i = names.index(nm)
        assert out[i] == -1
        row = fc[list(fp).index(i)]
        assert row[abi.SFC_STATIC] == 1 and row[abi.SFC_LOCAL] == c.n_nodes - 1 and row.sum() == c.n_nodes


# ---- coverage: the interactions the GPU tests are meant to exercise ----

def coverage(c, threads=1):
    """Walk the oracle with Open-Local pod by pod and count, from its per-node detail:
      left       decisions where a node that was feasible for the previous decision of the same class fails Open-Local now
      left_win   ... where that node is the previous decision's winner
      soft_cut   local decisions with soft spread or pod-affinity score terms where Open-Local removed an otherwise feasible node
      decided    decisions whose winner differs from the winner without the normalised Open-Local term
      gpu_local  placed pods of classes that request both GPU share and volumes
      mixed_fail failure histograms with SFC_LOCAL next to another reason
      decisions  decisions compared (pods that went through the cycle)."""
    from oracle.binding import Oracle
    o = Oracle(c, threads=threads, open_local=True)
    o.enable_dump()
    P = c.pods_dims["n_pods"]
    pod_class, fixed = c.pods["pod_class"], c.pods["pod_fixed_node"]
    off, blob = c.pods["class_off"], c.pods["class_blob"]
    cnt = dict(left=0, left_win=0, soft_cut=0, decided=0, gpu_local=0, mixed_fail=0, decisions=0)
    prev = {}
    try:
        for i in range(P):
            out, _s, fc, _fp = o.schedule(i, 1)
            if fixed[i] != -1 or out[0] == -3:
                continue
            cls = int(pod_class[i])
            cw = blob[int(off[cls]):]
            code, sc = o.last_detail()
            cnt["decisions"] += 1
            local = bool(c.storage.class_local[cls])
            if not local:
                continue
            feas = code == 0
            cut = code == 16
            if cls in prev:
                pfeas, pwin = prev[cls]
                if (cut & pfeas).any():
                    cnt["left"] += 1
                if pwin >= 0 and cut[pwin]:
                    cnt["left_win"] += 1
            prev[cls] = (feas, int(out[0]))
            if (cw[abi.SCW_N_PTS_SOFT] > 0 or cw[abi.SCW_N_IPA_SCORE] > 0) and cut.any() and feas.sum() > 1:
                cnt["soft_cut"] += 1
            if feas.sum() > 1:
                tot, ol = sc[:, 8], sc[:, 9]
                idx = np.nonzero(feas)[0]
                if idx[np.argmax(tot[idx])] != idx[np.argmax((tot - ol)[idx])]:
                    cnt["decided"] += 1
            if out[0] >= 0 and cw[abi.SCW_GPU_MEM] > 0:
                cnt["gpu_local"] += 1
            if len(fc):
                row = fc[0]
                if row[abi.SFC_LOCAL] > 0 and (np.delete(row, abi.SFC_LOCAL) > 0).any():
                    cnt["mixed_fail"] += 1
    finally:
        o.close()
    return cnt


def test_coverage_of_the_interactions():
    """Across the generator's seeds each interaction occurs: Open-Local removing nodes (and the last winner) after a Bind, cutting
    the feasible set that spread / affinity scores read, deciding the winner, pods with GPU share and volumes, and failure
    histograms where SFC_LOCAL stands next to other reasons."""
    tot = {}
    for seed in MIX_SEEDS[:8]:
        _p, c, _ol = make_mixed_local(seed, n_nodes=30 + seed % 20, n_workloads=24, max_replicas=6)
        for k, v in coverage(c).items():
            tot[k] = tot.get(k, 0) + v
    for k, v in tot.items():
        assert v > 0, (k, tot)
