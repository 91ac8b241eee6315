"""Capacity-planning scenario batches with Open-Local storage (pkg/apply/apply.go:203-259 with the open-local plugin, and
satisfyResourceSetting's MaxVG cap, apply.go:712-719, 746-772): the superset compiled with storage, the VG occupancy test, and on
the GPU the reference example's known answers and every scenario of a batch against an independent single-scenario run."""
import ctypes
import json
import os

import numpy as np
import pytest

from simon_b200 import objects as O

GI = 1 << 30
HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.path.join(HERE, "golden", "reference")
SCS = [{"apiVersion": "storage.k8s.io/v1", "kind": "StorageClass", "metadata": {"name": f"open-local-device-{m}"},
        "parameters": {"mediaType": m}} for m in ("ssd", "hdd")]


def _example(tmp_path, with_open_local=True):
    """example/simon-config.yaml with the cluster as customConfig (demo_1), the non-chart apps and newNode demo_1."""
    import yaml
    from simon_b200 import apply as A
    names = ["simple", "complicate"] + (["open_local"] if with_open_local else []) + ["more_pods"]
    cfg = {"apiVersion": "simon/v1alpha1", "kind": "Config", "metadata": {"name": "simon-config"},
           "spec": {"cluster": {"customConfig": "example/cluster/demo_1"},
                    "appList": [{"name": n, "path": f"example/application/{n}"} for n in names],
                    "newNode": "example/newnode/demo_1"}}
    path = tmp_path / "simon-config.yaml"
    path.write_text(yaml.safe_dump(cfg))
    return A.load_config(str(path), base_dir=REF)


# ---- CPU --------------------------------------------------------------------------------------------------------------------

def test_build_scenarios_with_open_local_on_the_reference_example(tmp_path):
    from simon_b200 import capacity
    from simon_b200.compiler import CompileError, compile_cluster
    cluster, apps, new_node = _example(tmp_path)
    ss = capacity.build_scenarios(cluster, apps, [new_node], [0, 1, 3], open_local=True, local_devices=True)
    c, st = ss.compiled, ss.compiled.storage
    assert st is not None and st.devices
    pool = [g for g, nm in enumerate(c.node_names) if nm.startswith(O.NEW_NODE_NAME_PREFIX)]
    assert len(pool) == 3
    for g in pool:          # every copy carries node-1.json: one 500 GiB VG and one HDD
        assert st.node_n_vg[g] == 1 and st.vg_capacity[0, g] == 500 * GI and st.vg_requested[0, g] == 0
        assert st.node_n_ssd[g] == 0 and st.node_n_hdd[g] == 1 and st.dev_capacity[0, g] == 100 * GI and st.dev_alloc[g] == 0
    scs = list(cluster.StorageClasss) + [sc for a in apps for sc in a.Resource.StorageClasss]
    base = compile_cluster(list(cluster.Nodes), [], open_local=True, storage_classes=scs, local_devices=True)
    bs = base.storage
    for b, nm in enumerate(base.node_names):
        g = c.node_index(nm)
        nv = int(bs.node_n_vg[b])
        assert st.node_n_vg[g] == nv, nm
        assert st.vg_capacity[:nv, g].tolist() == bs.vg_capacity[:nv, b].tolist()
        assert st.vg_requested[:nv, g].tolist() == bs.vg_requested[:nv, b].tolist()
        assert (st.node_n_ssd[g], st.node_n_hdd[g], st.dev_alloc[g]) == (bs.node_n_ssd[b], bs.node_n_hdd[b], bs.dev_alloc[b])
        nd = int(bs.node_n_ssd[b]) + int(bs.node_n_hdd[b])
        assert st.dev_capacity[:nd, g].tolist() == bs.dev_capacity[:nd, b].tolist()
    # the storage app still needs the opt-in
    with pytest.raises(CompileError):
        capacity.build_scenarios(cluster, apps, [new_node], [0])
    # and the defaults compile without storage tables, as before
    plain = capacity.build_scenarios(*_example(tmp_path, with_open_local=False)[:2], [new_node], [0, 1])
    assert plain.compiled.storage is None


def test_vg_occupancy_known_answers(monkeypatch):
    from simon_b200 import capacity
    r = dict(req_mcpu=0, alloc_mcpu=0, req_mem=0, alloc_mem=0, vg_requested=200, vg_capacity=1900)
    assert int(200 / 1900 * 100) == 10                             # truncation
    assert capacity.occupancy_ok(r, max_vg=10) and not capacity.occupancy_ok(r, max_vg=9)
    assert capacity.occupancy_ok(dict(r, vg_capacity=0, vg_requested=50), max_vg=0)     # no VG capacity: no test
    assert capacity.occupancy_ok(dict(r, vg_requested=0), max_vg=0)
    plain = {k: v for k, v in r.items() if not k.startswith("vg")}
    assert capacity.occupancy_ok(plain, max_vg=0)                  # results without VG sums (no storage) are not tested
    monkeypatch.delenv("MaxVG", raising=False)
    assert capacity.env_vg_cap() == 100
    for v, want in (("", 100), ("0", 0), ("37", 37), ("100", 100), ("101", 100), ("-1", 100), ("+5", 5)):
        monkeypatch.setenv("MaxVG", v)
        assert capacity.env_vg_cap() == want, v
    for bad in ("abc", "1.5", " 5"):
        monkeypatch.setenv("MaxVG", bad)
        with pytest.raises(ValueError):
            capacity.env_vg_cap()
    monkeypatch.setenv("MaxCPU", "50")
    assert capacity.env_caps() == (50, 100)


def _fake_factory(ss):
    """Every pod fits from k = 2 on; ΣVG requested 200, ΣVG capacity 400 + 500 k (the reference example's numbers in GiB)."""
    def run(ss, shard):
        return [dict(n_unscheduled=0 if sc.k >= 2 else 1, n_scheduled=10, req_mcpu=1, alloc_mcpu=100, req_mem=1, alloc_mem=100,
                     vg_requested=200, vg_capacity=400 + 500 * sc.k) for sc in shard]
    return run


def test_sweep_and_bisect_honour_max_vg(tmp_path, monkeypatch):
    from simon_b200 import apply as A, capacity
    cluster, apps, new_node = _example(tmp_path)
    monkeypatch.delenv("MaxVG", raising=False)
    # int(20000 / (400 + 500 k)): 3 at k = 12, 2 at 13 .. 19, 1 at 20 .. 39, 0 from 40 on
    for max_vg, kmax, want in ((None, 24, 2), (100, 24, 2), (2, 24, 13), (1, 19, -1), (1, 40, 20), (0, 40, 40)):
        got = [A.auto_add_nodes(cluster, apps, new_node, _fake_factory, kmax=kmax, method=m, open_local=True, local_devices=True,
                                max_vg=max_vg) for m in ("sweep", "bisect")]
        assert [g.new_node_num for g in got] == [want, want], (max_vg, kmax)
        assert set(got[0].per_k[0]) >= {"vg_requested", "vg_capacity"}
    monkeypatch.setenv("MaxVG", "1")
    assert A.auto_add_nodes(cluster, apps, new_node, _fake_factory, kmax=40, method="bisect", open_local=True).new_node_num == 20
    ss = capacity.build_scenarios(cluster, apps, [new_node], [0, 2, 19, 20], open_local=True)
    assert capacity.decode_key(capacity.search(ss, _fake_factory(ss))[0])["k"] == 20
    assert capacity.decode_key(capacity.search(ss, _fake_factory(ss), max_vg=100)[0])["k"] == 2


# ---- GPU --------------------------------------------------------------------------------------------------------------------

def _solo(ss, sc, scs, local_devices=True, ctx=None):
    """The scenario as a cluster of its own: its nodes, the superset pods that exist there (in superset order), compiled with
    Open-Local storage (and the superset's Services / ReplicaSets / StatefulSets, ctx) and placed by a single-scenario run, its
    result checked against the restated Bind."""
    from simon_b200.compiler import compile_cluster
    from simon_b200.engine import Engine
    from simon_b200.storage import StorageReplay
    c = ss.compiled
    act = sorted(int(g) for g in sc.nodes)
    names = {c.node_names[g] for g in act}
    nodes = [c.node_objs[g] for g in sorted(act, key=lambda g: c.node_orig_index[g])]
    keep = [i for i, p in enumerate(ss.pods) if not getattr(p.tmpl, "guard_node_name", "") or p.tmpl.guard_node_name in names]
    solo = compile_cluster(nodes, [ss.pods[i] for i in keep], ctx, open_local=True, storage_classes=scs, local_devices=local_devices)
    with Engine(solo) as eng:
        out = eng.schedule()[0]
        vg, dev = eng.storage_state(), eng.device_state() if local_devices else None
    rep = StorageReplay(solo.storage, solo.node_names)
    fixed, pod_class = solo.pods["pod_fixed_node"], solo.pods["pod_class"]
    for i, n in enumerate(out.tolist()):
        if n >= 0 and int(fixed[i]) == -1:
            rep.bind(int(pod_class[i]), n)
    assert np.array_equal(vg, rep.requested())
    if local_devices:
        assert np.array_equal(dev, rep.alloc_masks())
    return keep, solo, out, vg, dev


def _check_batch_against_solo(ss, sids, scs, local_devices=True, ctx=None):
    from simon_b200.engine import Engine
    c = ss.compiled
    with Engine(c) as eng:
        res, nodes = eng.run_scenarios_local([sc.nodes for sc in ss.scenarios], want_nodes=True)
        states = {i: eng.scenario_storage_state(i) for i in sids}
    for i in sids:
        sc = ss.scenarios[i]
        keep, solo, out, vg, dev = _solo(ss, sc, scs, local_devices, ctx)
        got = [c.node_names[g] if g >= 0 else int(g) for g in nodes[i][keep].tolist()]
        want = [solo.node_names[g] if g >= 0 else int(g) for g in out.tolist()]
        assert got == want, f"scenario {i}"
        assert res[i]["n_unscheduled"] == int((out == -1).sum()), i
        bvg, bdev = states[i]
        st, ss_st = solo.storage, c.storage
        req = cap = 0
        for g2, nm in enumerate(solo.node_names):
            g = c.node_index(nm)
            nv = int(st.node_n_vg[g2])
            assert bvg[:nv, g].tolist() == vg[:nv, g2].tolist(), (i, nm)
            req += int(vg[:nv, g2].sum())
            cap += int(st.vg_capacity[:nv, g2].sum())
            if local_devices:
                assert int(bdev[g]) == int(dev[g2]), (i, nm)
        assert (res[i]["vg_requested"], res[i]["vg_capacity"]) == (req, cap), i
        # inactive nodes keep the uploaded state
        inactive = np.setdiff1d(np.arange(c.n_nodes), sc.nodes)
        assert np.array_equal(bvg[:, inactive], ss_st.vg_requested[:, inactive])
        if local_devices:
            assert np.array_equal(bdev[inactive], ss_st.dev_alloc[inactive])
    return res


@pytest.mark.gpu
def test_reference_example_known_answers(tmp_path, monkeypatch):
    """demo_1 + simple, complicate, open_local, more_pods + newnode/demo_1: the four nginx-lvm replicas ask 10 + 40 GiB of LVM each
    (their HDD claim names a StorageClass nobody defines and is dropped).  The base VGs (master-1, worker-1: 2 x 100 GiB each) start
    empty; each new node brings 500 GiB."""
    from simon_b200 import apply as A, capacity
    from simon_b200.engine import Engine
    monkeypatch.delenv("MaxVG", raising=False)
    cluster, apps, new_node = _example(tmp_path)
    engines = []

    def factory(ss):
        e = Engine(ss.compiled, device=0)
        engines.append(e)
        return capacity.gpu_runner(0, engine=e)

    kw = dict(open_local=True, local_devices=True)
    sweep = A.auto_add_nodes(cluster, apps, new_node, factory, kmax=45, method="sweep", **kw)
    bis = A.auto_add_nodes(cluster, apps, new_node, factory, kmax=45, method="bisect", **kw)
    k0 = sweep.new_node_num
    assert k0 > 0 and bis.new_node_num == k0
    assert sweep.per_k[k0 - 1]["n_unscheduled"] > 0 or not capacity.occupancy_ok(sweep.per_k[k0 - 1])
    for k, r in sweep.per_k.items():
        assert r["vg_capacity"] == (400 + 500 * k) * GI, k
        if r["n_unscheduled"] == 0:
            assert r["vg_requested"] == 4 * (10 + 40) * GI, k
    for k in range(k0, 46):
        assert sweep.per_k[k]["n_unscheduled"] == 0
    for max_vg, kmax, want in ((1, 45, max(k0, 20)), (0, 45, max(k0, 40))):
        for m in ("sweep", "bisect"):
            assert A.auto_add_nodes(cluster, apps, new_node, factory, kmax=kmax, method=m, max_vg=max_vg, **kw).new_node_num == want
    for e in engines:
        e.close()
    # every scenario of a smaller sweep against its own single-scenario run
    ss = capacity.build_scenarios(cluster, apps, [new_node], list(range(0, k0 + 2)), **kw)
    from simon_b200.compiler import ClusterContext
    ctx = ClusterContext(services=list(cluster.Services), replicasets=list(cluster.ReplicaSets), statefulsets=list(cluster.StatefulSets))
    scs = list(cluster.StorageClasss) + [sc for a in apps for sc in a.Resource.StorageClasss]
    _check_batch_against_solo(ss, range(len(ss.scenarios)), scs, ctx=ctx)


def _node(name, zone, vgs=None, devs=None, annotated=True, cpu="16"):
    n = {"apiVersion": "v1", "kind": "Node",
         "metadata": {"name": name, "labels": {"kubernetes.io/hostname": name, "topology.kubernetes.io/zone": zone}, "annotations": {}},
         "status": {"allocatable": {"cpu": cpu, "memory": "64Gi", "pods": "110"}}}
    if annotated:
        ann = {"vgs": [{"name": f"vg{i}", "capacity": str(c), "requested": str(r)} for i, (c, r) in enumerate(vgs or [])],
               "devices": [{"name": f"/dev/d{k}", "device": f"/dev/d{k}", "capacity": str(c), "mediaType": m,
                            "isAllocated": "true" if a else "false"} for k, (c, m, a) in enumerate(devs or [])]}
        n["metadata"]["annotations"][O.ANNO_NODE_LOCAL_STORAGE] = json.dumps(ann)
    return n


def _random_node(rng, name, zone):
    if rng.random() < 0.15:
        return _node(name, zone, annotated=False, cpu=str(int(rng.choice([4, 8, 16]))))
    vgs = [(int(rng.integers(1, 20)) * 10 * GI, int(rng.integers(0, 3)) * 5 * GI) for _ in range(int(rng.integers(0, 4)))]
    devs = [(int(rng.choice([10, 20, 50, 100, 200])) * GI, str(rng.choice(["ssd", "hdd"])), bool(rng.random() < 0.1))
            for _ in range(int(rng.integers(0, 5)))]
    return _node(name, zone, vgs, devs, cpu=str(int(rng.choice([4, 8, 16]))))


def _vols(rng):
    vols = []
    r = rng.random()
    if r < 0.2:
        return None
    if r < 0.6:
        vols += [{"size": str(int(rng.integers(1, 8)) * 5 * GI), "kind": "LVM", "scName": "open-local-lvm"} for _ in range(int(rng.integers(1, 3)))]
    if r >= 0.45:
        m = str(rng.choice(["SSD", "HDD"]))
        vols.append({"size": str(int(rng.choice([5, 10, 20, 50])) * GI), "kind": m, "scName": f"open-local-device-{m.lower()}"})
    return vols


def _random_set(seed, n_base, n_pool, n_scen, n_pods, ds=True):
    """A superset of n_base + n_pool nodes (random VGs and devices, some without the annotation), Deployments with random volumes,
    a DaemonSet with an LVM volume (one guarded pod per node), and n_scen scenarios: the base plus a random subset of the pool,
    each in its own nodeTree order."""
    from simon_b200 import capacity
    from simon_b200.algo import order_app_pods
    from simon_b200.compiler import compile_cluster, node_tree_list
    from simon_b200.workloads import generate_valid_pods_from_app_resources, make_valid_pods_by_daemonset
    rng = np.random.default_rng(seed)
    nodes = [_random_node(rng, f"n{i:05d}", f"z{i % 3}") for i in range(n_base + n_pool)]
    deps = []
    for w in range(max(1, n_pods // 10)):
        tmpl = {"metadata": {"labels": {"app": f"w{w}"}},
                "spec": {"containers": [{"name": "c", "image": "x", "resources": {"requests": {
                    "cpu": f"{int(rng.integers(1, 20)) * 100}m", "memory": f"{int(rng.integers(1, 16)) * 256}Mi"}}}]}}
        v = _vols(rng)
        if v:
            tmpl["metadata"]["annotations"] = {O.ANNO_POD_LOCAL_STORAGE: json.dumps({"volumes": v})}
        deps.append({"apiVersion": "apps/v1", "kind": "Deployment", "metadata": {"name": f"w{w}", "namespace": "default"},
                     "spec": {"replicas": 10, "selector": {"matchLabels": {"app": f"w{w}"}}, "template": tmpl}})
    pods = []
    if ds:
        d = {"apiVersion": "apps/v1", "kind": "DaemonSet", "metadata": {"name": "ds", "namespace": "default"},
             "spec": {"template": {"metadata": {"annotations": {O.ANNO_POD_LOCAL_STORAGE: json.dumps(
                 {"volumes": [{"size": str(5 * GI), "kind": "LVM", "scName": "open-local-lvm"}]})}},
                 "spec": {"containers": [{"name": "c", "image": "x", "resources": {"requests": {"cpu": "100m"}}}]}}}}
        pods += make_valid_pods_by_daemonset(d, nodes)
    app_pods = generate_valid_pods_from_app_resources(nodes, "app", O.ResourceTypes(Deployments=deps))
    order_app_pods(app_pods)
    pods += app_pods
    c = compile_cluster(nodes, pods, open_local=True, storage_classes=SCS, local_devices=True)
    orig_to_compiled = np.zeros(len(nodes), np.int64)
    for ci, oi in enumerate(c.node_orig_index):
        orig_to_compiled[oi] = ci
    scen = []
    for s in range(n_scen):
        members = list(range(n_base)) + [n_base + j for j in np.flatnonzero(rng.random(n_pool) < rng.random())]
        order = node_tree_list([nodes[m] for m in members])
        scen.append(capacity.Scenario(s, 0, len(members) - n_base, np.array([orig_to_compiled[members[o]] for o in order], np.uint32)))
    return capacity.ScenarioSet(c, scen, pods, n_base)


@pytest.mark.gpu
def test_batch_of_several_waves_equals_solo_runs():
    """600 small scenarios: more clusters than the device holds at once, so the batch runs in at least two waves; each scenario's
    placements, VG state, device masks and VG sums equal those of its own single-scenario run."""
    ss = _random_set(31, 24, 40, 600, 120)
    res = _check_batch_against_solo(ss, range(len(ss.scenarios)), SCS)
    assert sum(r["n_scheduled"] for r in res) > 0 and len({r["vg_requested"] for r in res}) > 1


@pytest.mark.gpu
@pytest.mark.parametrize("seed, n_base, n_pool, n_scen, n_pods", [(32, 200, 300, 40, 400), (33, 1500, 1500, 6, 600)])
def test_batch_equals_solo_runs(seed, n_base, n_pool, n_scen, n_pods):
    ss = _random_set(seed, n_base, n_pool, n_scen, n_pods)
    _check_batch_against_solo(ss, range(len(ss.scenarios)), SCS)


@pytest.mark.gpu
def test_batch_without_devices_equals_solo_runs():
    """LVM volumes only, no device upload: the batch keeps no device state and still equals the solo runs."""
    from simon_b200 import capacity
    from simon_b200.compiler import compile_cluster, node_tree_list
    from simon_b200.workloads import PodRec, PodTemplate
    rng = np.random.default_rng(35)
    nodes = [_random_node(rng, f"m{i:04d}", f"z{i % 2}") for i in range(150)]
    pods = []
    for j in range(300):
        ann = {O.ANNO_POD_LOCAL_STORAGE: json.dumps({"volumes": [{"size": str(int(rng.integers(1, 8)) * 5 * GI), "kind": "LVM",
                                                                  "scName": "open-local-lvm"}]})} if j % 3 else {}
        pod = {"apiVersion": "v1", "kind": "Pod", "metadata": {"name": f"p{j}", "namespace": "default", "annotations": ann},
               "spec": {"containers": [{"name": "c", "image": "x", "resources": {"requests": {"cpu": "100m", "memory": "128Mi"}}}]}}
        pods.append(PodRec(PodTemplate(pod, "Pod", f"p{j}", "default"), f"p{j}", 0))
    c = compile_cluster(nodes, pods, open_local=True, storage_classes=SCS)
    scen = []
    for s in range(12):
        members = [m for m in range(150) if m < 50 or rng.random() < 0.5]
        order = node_tree_list([nodes[m] for m in members])
        o2c = {oi: ci for ci, oi in enumerate(c.node_orig_index)}
        scen.append(capacity.Scenario(s, 0, len(members) - 50, np.array([o2c[members[o]] for o in order], np.uint32)))
    ss = capacity.ScenarioSet(c, scen, pods, 50)
    _check_batch_against_solo(ss, range(len(scen)), SCS, local_devices=False)


@pytest.mark.gpu
def test_large_cluster_batch_equals_solo_runs():
    """A superset of about 41,000 nodes, two scenarios: the large-cluster local variant (per-node arrays in global memory)."""
    ss = _random_set(36, 40000, 1000, 2, 150, ds=False)
    assert max(len(sc.nodes) for sc in ss.scenarios) > 40000
    _check_batch_against_solo(ss, range(2), SCS)


@pytest.mark.gpu
def test_context_isolation_and_refusals():
    """A batch leaves the single-scenario storage state alone; the new entry points refuse what they cannot serve."""
    from simon_b200 import abi
    from simon_b200.compiler import compile_cluster
    from simon_b200.engine import Engine, lib
    L = lib()
    ss = _random_set(37, 60, 40, 8, 150)
    c = ss.compiled
    vg = np.zeros(max(c.storage.n_vgs * c.n_nodes, 1), np.int64)
    dev = np.zeros(c.n_nodes, np.uint32)
    with Engine(c) as eng:
        assert L.simon_scenarios_storage_download(eng.h, 0, vg.ctypes.data, None) == -3         # no batch yet
        a = eng.schedule()[0], eng.storage_state(), eng.device_state()
        assert a[1].any() and a[2].any()
        res, _ = eng.run_scenarios_local([sc.nodes for sc in ss.scenarios])
        assert np.array_equal(eng.storage_state(), a[1]) and np.array_equal(eng.device_state(), a[2])
        eng.reset()
        b = eng.schedule()[0], eng.storage_state(), eng.device_state()
        for x, y in zip(a, b):
            assert np.array_equal(x, y)
        assert L.simon_scenarios_storage_download(eng.h, 8, vg.ctypes.data, None) == -1         # scenario out of range
        assert L.simon_scenarios_storage_download(eng.h, 7, vg.ctypes.data, dev.ctypes.data) == 0
        # bad node lists
        dup = np.array([0, 1, 1], np.uint32)
        for bad in (dup, np.array([c.n_nodes], np.uint32), np.arange(c.n_nodes + 1, dtype=np.uint32) % max(c.n_nodes, 1)):
            arr = (abi.SimonScenario * 1)()
            arr[0].n_nodes, arr[0].nodes = len(bad), bad.ctypes.data
            out, loc = (abi.SimonScenarioResult * 1)(), (abi.SimonScenarioLocalResult * 1)()
            assert L.simon_scenarios_run_local(eng.h, arr, 1, out, loc, None) == -1
        # the plain entry still refuses a context with storage
        arr = (abi.SimonScenario * 1)()
        nodes = np.ascontiguousarray(ss.scenarios[0].nodes)
        arr[0].n_nodes, arr[0].nodes = len(nodes), nodes.ctypes.data
        out = (abi.SimonScenarioResult * 1)()
        assert L.simon_scenarios_run(eng.h, arr, 1, out, None) == -4
        # a batch, then a new storage upload: the batch state is gone
        eng.run_scenarios_local([sc.nodes for sc in ss.scenarios[:2]])
        assert L.simon_scenarios_storage_download(eng.h, 1, vg.ctypes.data, None) == 0
        assert L.simon_storage_upload(eng.h, ctypes.byref(eng.storage)) == 0
        assert L.simon_scenarios_storage_download(eng.h, 0, vg.ctypes.data, None) == -3
        # without a device upload the device state of a batch is not available
        eng.run_scenarios_local([sc.nodes for sc in ss.scenarios[:2]])
        assert L.simon_scenarios_storage_download(eng.h, 0, vg.ctypes.data, dev.ctypes.data) == -3
        assert L.simon_scenarios_storage_download(eng.h, 0, vg.ctypes.data, None) == 0
    # without storage the new entry is a call-order error
    plain = compile_cluster([c.node_objs[0]], [])
    with Engine(plain) as eng:
        arr = (abi.SimonScenario * 1)()
        one = np.zeros(1, np.uint32)
        arr[0].n_nodes, arr[0].nodes = 1, one.ctypes.data
        out, loc = (abi.SimonScenarioResult * 1)(), (abi.SimonScenarioLocalResult * 1)()
        assert L.simon_scenarios_run_local(eng.h, arr, 1, out, loc, None) == -3
        assert L.simon_scenarios_storage_download(eng.h, 0, vg.ctypes.data, None) == -3
        assert eng.run_scenarios([one])[0][0]["n_unscheduled"] == 0
