"""Grow batches on the device (simon_grow_run, Engine.grow_run, Simulator.PlanAddNodes).

Every batch placement variant a grow batch launches - with and without the static-verdict cache, the large-cluster variant and forced
geometries with several node slots per thread - against the grow checker (tests/checkers.c) on plain, GPU-share and Open-Local
clusters; the recompile-and-resume equivalence that pins the definition; chunking; the batch pool shared with drains and probes; the
C-entry refusals; and PlanAddNodes end to end on the reference example."""
import copy
import json
import os
from dataclasses import replace

import numpy as np
import pytest

from simon_b200 import abi, grow, objects as O, simulator, synth
from simon_b200.compiler import compile_cluster
from test_grow import session

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "tests", "golden", "reference")


def _mixed_local(seed, n_nodes):
    """make_mixed_local of tests/test_open_local_oracle.py as (cluster, apps): synth.make_mix with Open-Local volumes and annotations."""
    import test_open_local_oracle as T
    cluster, apps = synth.make_mix(seed_no=seed, n_nodes=n_nodes, n_workloads=30, max_replicas=6)
    rng = np.random.default_rng(0x0100CA1 + seed)
    for n in cluster.Nodes:
        if rng.random() < 0.67:
            O.meta(n).setdefault("annotations", {})
            O.meta(n)["annotations"][O.ANNO_NODE_LOCAL_STORAGE] = json.dumps(T._node_storage(rng))
    cluster.StorageClasss.extend(T.STORAGE_CLASSES)
    res = apps[0].Resource
    for w in res.Deployments + res.Jobs + res.DaemonSets + cluster.DaemonSets:
        if rng.random() < 0.5:
            T._annotate(w["spec"]["template"].setdefault("metadata", {}), T._volumes(rng))
    for w in res.StatefulSets:
        if rng.random() < 0.5:
            w["spec"]["volumeClaimTemplates"] = T._vcts(T._volumes(rng))
    return cluster, apps


def _case(kind, n_nodes=200):
    """(session on the cluster, the app to grow for, candidate specs).  plain: a C2-shaped cluster (CPU and memory only), one app
    running and one to grow for; mix: synth.make_mix (GPU share, taints, affinity, spread, ...) with its app to grow for; gpu: the
    same mix with every other Deployment of its app running, so that the prefix holds GPU-share pods the scheduler placed;
    local: the mix with Open-Local volumes."""
    if kind == "plain":
        cluster, apps = synth.make_c2(n_nodes=n_nodes, n_workloads=24, replicas=30, n_apps=2, seed_no=23)
        sim = session(cluster, apps[:1])
        return sim, apps[1], [copy.deepcopy(cluster.Nodes[0]), copy.deepcopy(cluster.Nodes[-1])]
    if kind == "local":
        cluster, apps = _mixed_local(11, n_nodes)
        sim = session(cluster, [], simulator.WithOpenLocal(devices=True))
        ann = [n for n in cluster.Nodes if O.ANNO_NODE_LOCAL_STORAGE in (O.meta(n).get("annotations") or {})]
        specs = [copy.deepcopy(ann[0]), copy.deepcopy(ann[-1])]
    else:
        cluster, apps = synth.make_mix(seed_no=21 if kind == "mix" else 22, n_nodes=n_nodes, n_workloads=30, max_replicas=6)
        if kind == "gpu":
            res = apps[0].Resource
            running = O.AppResource("running", O.ResourceTypes(Deployments=res.Deployments[::2]))
            apps = [O.AppResource(apps[0].Name, replace(res, Deployments=res.Deployments[1::2]))]
            sim = session(cluster, [running])
        else:
            sim = session(cluster)
        gpu = [n for n in cluster.Nodes if "alibabacloud.com/gpu-count" in (n.get("status") or {}).get("allocatable", {})]
        specs = [copy.deepcopy(cluster.Nodes[0]), copy.deepcopy(gpu[0] if kind == "gpu" and gpu else cluster.Nodes[-1])]
    for s in specs:
        (s.get("spec") or {}).pop("unschedulable", None)
    return sim, apps[0], specs


def _check(eng, gs, raw, sids):
    """Every scenario of `raw` (Engine.grow_run with detail) against the grow checker, the Open-Local state too."""
    from oracle.binding import Oracle
    import checkers
    c = gs.compiled
    local = c.storage is not None
    o = Oracle(c, open_local=local)
    try:
        for i, (sid, r) in enumerate(zip(sids, raw)):
            sc = gs.scenarios[sid]
            w = checkers.grow(o, gs.placed, gs.n_prefix, sc.nodes)
            for key in ("node", "score", "gpu_slots", "fail_counts", "fail_pod"):
                assert np.array_equal(r[key], w[key]), (sid, key)
            assert (r["n_scheduled"], r["n_unscheduled"]) == (w["n_scheduled"], w["n_unscheduled"]), sid
            st = o.state()
            act = sc.nodes.astype(np.int64)
            assert r["req_mcpu"] == int(st["req_mcpu"][act].sum()) and r["req_mem"] == int(st["req_mem"][act].sum()), sid
            assert r["alloc_mcpu"] == int(c.snap["alloc_mcpu"][act].sum()), sid
            if local:
                vg, dev = o.storage_state()
                gvg, gdev = eng.scenario_storage_state(i)
                assert np.array_equal(gvg[:, act], vg[:, act]), sid
                if dev is not None:
                    assert np.array_equal(gdev[act], dev[act]), sid
                nvg = np.asarray(c.storage.node_n_vg)
                cap = np.asarray(c.storage.vg_capacity)
                assert r["vg_requested"] == sum(int(vg[a, g]) for g in act.tolist() for a in range(int(nvg[g]))), sid
                assert r["vg_capacity"] == sum(int(cap[a, g]) for g in act.tolist() for a in range(int(nvg[g]))), sid
    finally:
        o.close()


ENGINES = {
    "default": {},
    "no_static_cache": dict(static_cache=False),
    "large": dict(force_large=True),
    "1x64": dict(cluster_ctas=1, threads_per_cta=64),
    "2x64": dict(cluster_ctas=2, threads_per_cta=64),
}


@pytest.mark.parametrize("kind", ["plain", "mix", "gpu", "local"])
@pytest.mark.parametrize("opts", list(ENGINES))
def test_grow_variants_match_checker(kind, opts):
    from simon_b200.engine import Engine
    sim, app, specs = _case(kind)
    gs = grow.build(sim, [app], specs, 4)
    with Engine(gs.compiled, device=0, record_scores=True, **ENGINES[opts]) as eng:
        sids = list(range(len(gs.scenarios)))
        raw = eng.grow_run(gs.placed, gs.n_prefix, [gs.scenarios[s].nodes for s in sids])
        li = eng.last_grow["launches"][-1]
        assert li["kernel"].startswith("simon_local_kernel" if kind == "local" else "simon_place_kernel"), li
        if kind == "gpu":
            # live GPU-share device memory in the prefix, and GPU-share pods in the tail
            assert sim.gpu_slots[:gs.n_prefix].any() and any(r["gpu_slots"].any() for r in raw)
        assert li["n_scenarios"] == len(sids)
        if opts == "large":
            assert li["large"]
        if "cluster_ctas" in ENGINES[opts]:
            ctas = ENGINES[opts]["cluster_ctas"]
            assert li["cluster_ctas"] == ctas and li["node_slots"] == -(-li["n_nodes"] // (ctas * 64)) >= 2, li
        _check(eng, gs, raw, sids)


def _resume_equivalent(sim, gs, s, k, eng_raw):
    """Scenario (s, k) against the recompile-and-resume definition: the base plus the first k copies of spec s compiled with the
    superset's pod list filtered to the pods that exist there, resumed from the session's placements remapped by node name."""
    from simon_b200.engine import Engine
    from simon_b200.scaledown import pod_guard
    c = gs.compiled
    sc = gs.scenario(s, k)
    active = set(sc.nodes.tolist())
    guard = pod_guard(c)
    keep = [q for q in range(c.pods_dims["n_pods"]) if not (guard[q] >= 0 and guard[q] not in active)]
    assert keep[:gs.n_prefix] == list(range(gs.n_prefix))
    nodes = [c.node_objs[g] for g in sorted(active, key=lambda g: c.node_orig_index[g])]
    p = sim._plan()
    o = sim.options
    scs = None
    if o.openLocal:
        scs = list(sim.cluster.StorageClasss) + [x for a in sim.apps for x in a.Resource.StorageClasss]
    c2 = compile_cluster(nodes, [c.pod_recs[q] for q in keep], p.ctx, open_local=o.openLocal, storage_classes=scs,
                         local_devices=o.openLocalDevices)
    assert c2.node_names == [c.node_names[g] for g in sc.nodes]
    with Engine(c2, device=0, record_scores=True) as e2:
        out, score, fc, fp = e2.schedule_resume(grow.remap(sim.compiled, c2, sim.placements))
        slots = e2.gpu_slot_words()
        if c.storage is not None:
            vg2, dev2 = e2.storage_state(), (e2.device_state() if c2.storage.devices else None)
    to_super = np.array([c.node_index(nm) for nm in c2.node_names], np.int32)
    tail = np.array(keep[gs.n_prefix:], np.int64) - gs.n_prefix
    r = eng_raw
    got = r["node"][tail]
    want = np.where(out[gs.n_prefix:] >= 0, to_super[np.maximum(out[gs.n_prefix:], 0)], out[gs.n_prefix:])
    assert np.array_equal(got, want), (s, k)
    assert np.array_equal(r["score"][tail], score[gs.n_prefix:]), (s, k)
    assert np.array_equal(r["gpu_slots"][tail], slots[gs.n_prefix:]), (s, k)
    assert np.array_equal(r["fail_counts"], fc), (s, k)
    assert [keep[q] for q in fp.tolist()] == r["fail_pod"].tolist(), (s, k)
    if c.storage is not None:
        return vg2, dev2, to_super
    return None


def test_resume_equivalence_gpu_share_session():
    """A C3-shaped session with GPU share, several specs, k from 0 to kmax."""
    from simon_b200.engine import Engine
    cluster, apps = synth.make_c3(n_nodes=300, n_workloads=60, replicas=10, n_apps=2, seed_no=31, gpu_pct=25)
    sim = session(cluster, apps[:1])
    # the prefix holds GPU-share pods placed by the scheduler: their device memory must reach every scenario
    fixed = np.asarray(sim.compiled.pods["pod_fixed_node"])
    assert (sim.gpu_slots[:len(sim.placements)][fixed == -1] != 0).any()
    specs = [copy.deepcopy(n) for n in cluster.Nodes[:3]]
    gs = grow.build(sim, apps[1:], specs, 6)
    with Engine(gs.compiled, device=0, record_scores=True) as eng:
        picks = [(0, 0), (0, 6), (1, 3), (2, 1), (2, 6)]
        raw = eng.grow_run(gs.placed, gs.n_prefix, [gs.scenario(s, k).nodes for s, k in picks])
    assert any(r["gpu_slots"].any() for r in raw)
    for (s, k), r in zip(picks, raw):
        _resume_equivalent(sim, gs, s, k, r)


def test_resume_equivalence_open_local_session():
    from simon_b200.engine import Engine
    sim, app, specs = _case("local", n_nodes=60)
    gs = grow.build(sim, [app], specs, 3)
    picks = [(0, 0), (0, 3), (1, 2)]
    with Engine(gs.compiled, device=0, record_scores=True) as eng:
        raw = eng.grow_run(gs.placed, gs.n_prefix, [gs.scenario(s, k).nodes for s, k in picks])
        states = [eng.scenario_storage_state(i) for i in range(len(picks))]
    for (s, k), r, (vg, dev) in zip(picks, raw, states):
        vg2, dev2, to_super = _resume_equivalent(sim, gs, s, k, r)
        assert np.array_equal(vg[:, to_super], vg2), (s, k)
        if dev2 is not None:
            assert np.array_equal(dev[to_super], dev2), (s, k)


def test_chunks_batch_pool_and_refusals():
    from simon_b200.engine import Engine, lib
    sim, app, specs = _case("gpu", n_nodes=60)
    gs = grow.build(sim, [app], specs, 3)
    c = gs.compiled
    lists = [sc.nodes for sc in gs.scenarios]
    with Engine(c, device=0, record_scores=True) as eng:
        one = eng.grow_run(gs.placed, gs.n_prefix, lists)
        assert eng.last_grow["chunks"] == 1
        chunked = eng.grow_run(gs.placed, gs.n_prefix, lists, chunk=3)
        assert eng.last_grow["chunks"] == 3
        for a, b in zip(one, chunked):
            for key in a:
                assert np.array_equal(a[key], b[key]), key
        # the single-scenario downloads describe the prefix afterwards
        assert np.array_equal(eng.results(0, gs.n_prefix), gs.placed)
        L, h = lib(), eng.h
        node = np.zeros(c.pods_dims["n_pods"], np.int32)
        # a full placement with the tail pending: what a single run reports for the tail pods that never reach the scheduler
        from simon_b200.scaledown import pod_guard
        fixed, guard = np.asarray(c.pods["pod_fixed_node"]), pod_guard(c)
        full = np.where(guard == -2, -3, np.where(fixed >= 0, fixed, np.where(fixed == -1, -1, -2))).astype(np.int32)
        full[:gs.n_prefix] = gs.placed
        # drains and probes refuse after a grow batch, and a grow download after them
        assert L.simon_drain_download(h, 0, None, None, None, None, None, None, None) == -3
        assert L.simon_probe_download(h, 0, None, None, None, None) == -3
        eng.drain_run(full, [lists[0][1:]], detail=False)
        assert L.simon_grow_download(h, 0, node.ctypes.data, None, None, None, None) == -3
        eng.grow_run(gs.placed, gs.n_prefix, lists[:2])
        assert L.simon_drain_download(h, 0, None, None, None, None, None, None, None) == -3
        assert L.simon_grow_download(h, 2, node.ctypes.data, None, None, None, None) == -1
        # the C-entry refusals, before any device work
        arr, keep = eng._scenario_array([lists[0]])
        res = (abi.SimonScenarioResult * 1)()
        pl = np.ascontiguousarray(gs.placed)
        P = c.pods_dims["n_pods"]
        assert L.simon_grow_run(h, pl.ctypes.data, P + 1, arr, 1, res, None) == -1
        assert b"n_prefix" in L.simon_last_error(h)
        bad = pl.copy()
        bad[np.nonzero(bad >= 0)[0][0]] = c.n_nodes
        assert L.simon_grow_run(h, bad.ctypes.data, gs.n_prefix, arr, 1, res, None) == -1
        for nodes in ([], [lists[0][0], lists[0][0]], [c.n_nodes]):
            a2, k2 = eng._scenario_array([np.array(nodes, np.uint32)])
            assert L.simon_grow_run(h, pl.ctypes.data, gs.n_prefix, a2, 1, res, None) == -1
        # a scenario without a node that holds a placed prefix pod
        held = int(pl[pl >= 0][0])
        a3, k3 = eng._scenario_array([np.array([g for g in lists[0].tolist() if g != held], np.uint32)])
        assert L.simon_grow_run(h, pl.ctypes.data, gs.n_prefix, a3, 1, res, None) == -1
        assert b"holds a placed prefix pod" in L.simon_last_error(h)
        loc = (abi.SimonScenarioLocalResult * 1)()
        assert L.simon_grow_run(h, pl.ctypes.data, gs.n_prefix, arr, 1, res, loc) == -3
        # the refusals left the last batch readable
        assert L.simon_grow_download(h, 1, node.ctypes.data, None, None, None, None) == 0


def test_plan_add_nodes_reference_example():
    """demo_1 running simple and complicated, then more_pods, which does not fit: PlanAddNodes with newnode/demo_1 equals a per-k loop of
    recompile plus simon_schedule_resume, and leaves the session as it was."""
    import yaml
    from simon_b200 import apply as A
    from simon_b200.engine import Engine
    cfg = {"apiVersion": "simon/v1alpha1", "kind": "Config", "metadata": {"name": "c"},
           "spec": {"cluster": {"customConfig": "example/cluster/demo_1"},
                    "appList": [{"name": "simple", "path": "example/application/simple"},
                                {"name": "complicated", "path": "example/application/complicate"},
                                {"name": "more_pods", "path": "example/application/more_pods"}],
                    "newNode": "example/newnode/demo_1"}}
    path = os.path.join(os.environ.get("TMPDIR", "/tmp"), f"grow-cfg-{os.getpid()}.yaml")
    with open(path, "w") as fh:
        fh.write(yaml.safe_dump(cfg))
    try:
        cluster, apps, new_node = A.load_config(path, base_dir=REF)
    finally:
        os.remove(path)
    sim = simulator.NewSimulator()
    sim.RunCluster(simulator.PrepareCluster(cluster))
    for a in apps[:2]:
        sim.ScheduleApp(a)
    before = (sim.placements.copy(), sim.gpu_slots.copy(), sim.engine, sim.compiled)
    kmax = 12
    plan = sim.PlanAddNodes(apps[2:], [new_node], kmax=kmax)
    bis = sim.PlanAddNodes(apps[2:], [new_node], kmax=kmax, method="bisect")
    assert sim.engine is before[2] and sim.compiled is before[3]
    assert np.array_equal(sim.placements, before[0]) and np.array_equal(sim.gpu_slots, before[1])
    sp = plan.Specs[0]
    assert sp.PerK[0]["n_unscheduled"] > 0 and sp.NewNodeNum > 0 and bis.Specs[0].NewNodeNum == sp.NewNodeNum
    gs = grow.build(sim, apps[2:], [new_node], kmax)
    with Engine(gs.compiled, device=0, record_scores=True) as eng:
        raw = eng.grow_run(gs.placed, gs.n_prefix, [gs.scenario(0, k).nodes for k in range(kmax + 1)])
    for k in range(kmax + 1):
        _resume_equivalent(sim, gs, 0, k, raw[k])
        assert sp.PerK[k]["n_unscheduled"] == raw[k]["n_unscheduled"]
    k = sp.NewNodeNum
    got = [(p.Pod.name, p.Node) for p in sp.Pods]
    want = [(gs.compiled.pod_recs[gs.n_prefix + t].name, gs.compiled.node_names[g]) for t, g in enumerate(raw[k]["node"].tolist()) if g >= 0]
    assert got == want and not sp.UnscheduledPods
    # a later ScheduleApp places what it placed without the call
    ref = simulator.NewSimulator()
    ref.RunCluster(simulator.PrepareCluster(cluster))
    for a in apps:
        ref.ScheduleApp(a)
    sim.ScheduleApp(apps[2])
    assert np.array_equal(sim.placements, ref.placements)
    sim.Close()
    ref.Close()
