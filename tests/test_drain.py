"""Node drains (simon_drain_run, simon_b200.scaledown) and the scale-down planner.

CPU: remaining-node orders against node_tree_list, the classification of a removed node's pods, the planner's prefix rule with a
fake runner, the drain checker (tests/checkers.c) on hand-derived answers.  GPU: every drain kernel variant against the checker,
drains against the recompile + simon_schedule_resume equivalence that pins the definition, the live state after a drain batch, and
the session entry points end to end."""
import numpy as np
import pytest

from simon_b200 import objects as O, scaledown, simulator, synth
from simon_b200.compiler import compile_cluster, node_tree_list
from util import compiled_kernels


def _compiled(cluster, apps, **kw):
    p = simulator.plan(cluster, apps)
    return compile_cluster(p.nodes, p.pods, p.ctx, **kw)


def _live(c):
    from oracle.binding import Oracle
    o = Oracle(c)
    return o, o.schedule()[0]


def _node(name, mcpu="4000m", mem="16Gi", zone=None):
    labels = {"kubernetes.io/hostname": name}
    if zone:
        labels["topology.kubernetes.io/zone"] = zone
    return {"apiVersion": "v1", "kind": "Node", "metadata": {"name": name, "labels": labels},
            "status": {"allocatable": {"cpu": mcpu, "memory": mem, "pods": "110"}, "capacity": {"cpu": mcpu, "memory": mem, "pods": "110"}}}


def known_answer():
    """4 nodes of 4000m, one Deployment of 8 pods of 1000m: two per node in the live state."""
    cluster = O.ResourceTypes(Nodes=[_node(f"node-{i}") for i in range(4)])
    dep = {"apiVersion": "apps/v1", "kind": "Deployment", "metadata": {"name": "web", "namespace": "default"},
           "spec": {"replicas": 8, "selector": {"matchLabels": {"app": "web"}},
                    "template": {"metadata": {"labels": {"app": "web"}},
                                 "spec": {"containers": [{"name": "c", "image": "nginx",
                                                          "resources": {"requests": {"cpu": "1000m", "memory": "1Gi"}}}]}}}}
    return cluster, [O.AppResource("web", O.ResourceTypes(Deployments=[dep]))]


def checker_runner(c, placed):
    """plan_scale_down's runner on the CPU: the drain checker, plus the occupancy sums of its end state."""
    import checkers
    o, _ = _live(c)
    ac, am = c.snap["alloc_mcpu"], c.snap["alloc_mem"]

    def run(remain_lists):
        out = []
        for rl in remain_lists:
            r = checkers.drain(o, placed, rl)
            st = o.state()
            idx = np.asarray(rl, dtype=np.int64)
            r.update(req_mcpu=int(st["req_mcpu"][idx].sum()), alloc_mcpu=int(ac[idx].sum()),
                     req_mem=int(st["req_mem"][idx].sum()), alloc_mem=int(am[idx].sum()))
            out.append(r)
        return out
    return run


# ---- CPU --------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("seed", [0, 3, 7])
def test_remaining_orders_equal_node_tree_list(seed):
    c = _compiled(*synth.make_mix(seed_no=seed, n_nodes=40))
    order = scaledown.NodeOrder(c)
    assert order.remaining([]).tolist() == list(range(c.n_nodes))        # the snapshot is in nodeTree order
    rng = np.random.default_rng(seed)
    for _ in range(40):
        rm = rng.choice(c.n_nodes, size=int(rng.integers(1, c.n_nodes)), replace=False)
        keep = sorted(set(range(c.n_nodes)) - set(rm.tolist()), key=lambda g: c.node_orig_index[g])
        want = [keep[i] for i in node_tree_list([c.node_objs[g] for g in keep])]
        assert order.remaining(rm).tolist() == want


def test_classification_static_bare_daemonset_pods():
    for seed in (0, 1, 2, 5):
        c = _compiled(*synth.make_mix(seed_no=seed, n_nodes=30))
        _o, placed = _live(c)
        fixed = c.pods["pod_fixed_node"]
        guard = scaledown.pod_guard(c)
        seen_kinds = set()
        for g in range(c.n_nodes):
            ev, bl, va = scaledown.classify(c, placed, [g])
            on = np.nonzero(placed == g)[0].tolist()
            assert sorted(ev + [q for q, _ in bl] + va) == on and ev == sorted(ev)
            for q in va:
                assert guard[q] == g
            for q, why in bl:
                assert fixed[q] >= 0 and why == scaledown.BLOCK_NODE_NAME
            for q in ev:
                assert fixed[q] == -1 and guard[q] != g
            seen_kinds |= {k for k, v in (("ev", ev), ("bl", bl), ("va", va)) if v}
        assert seen_kinds == {"ev", "bl", "va"}, seen_kinds


def test_classification_open_local_pods_block(tmp_path):
    from test_open_local_capacity import _example
    cluster, apps, _new = _example(tmp_path)
    scs = list(cluster.StorageClasss) + [sc for a in apps for sc in a.Resource.StorageClasss]
    p = simulator.plan(cluster, apps)
    c = compile_cluster(p.nodes, p.pods, p.ctx, open_local=True, storage_classes=scs, local_devices=True)
    local = c.storage.class_local
    cls = c.pods["pod_class"]
    # a synthetic live state: every pod that reaches the scheduler on node 0 (classification reads nothing else of it)
    placed = np.where(c.pods["pod_fixed_node"] >= 0, c.pods["pod_fixed_node"], 0).astype(np.int32)
    ev, bl, va = scaledown.classify(c, placed, [0])
    vol = [q for q in range(len(placed)) if placed[q] == 0 and local[int(cls[q])] and c.pods["pod_fixed_node"][q] < 0
           and scaledown.pod_guard(c)[q] != 0]
    assert vol and all((q, scaledown.BLOCK_LOCAL_STORAGE) in bl for q in vol)
    assert not any(local[int(cls[q])] for q in ev)


def _fake_plan(seq, candidates=None):
    """plan_scale_down on the known-answer cluster with a runner whose k-prefix verdicts come from seq[k - 1] (True: drains)."""
    c = _compiled(*known_answer())
    calls = []

    def runner(remain_lists):
        calls.append([len(r) for r in remain_lists])
        out = []
        for rl in remain_lists:
            k = c.n_nodes - len(rl)
            ok = True if k == 1 and len(calls) == 1 else seq[k - 1]
            out.append(dict(n_blocked=0, n_unscheduled=0 if ok else 1, n_evicted=2, req_mcpu=0, alloc_mcpu=1, req_mem=0, alloc_mem=1))
        return out
    placed = np.repeat(np.arange(c.n_nodes), 2).astype(np.int32)
    return scaledown.plan_scale_down(c, placed, runner, candidates=candidates, batch=2, max_cpu=100, max_mem=100), calls


def test_planner_first_failing_prefix_ends_the_plan():
    plan, calls = _fake_plan([True, False, True])          # k = 3 would pass again: not monotone
    assert len(plan.RemovedNodes) == 1
    assert [p["k"] for p in plan.Prefixes] == [1, 2] and [p["ok"] for p in plan.Prefixes] == [True, False]
    assert calls[0] == [3, 3, 3, 3]                          # the sweep: every node alone, in one run
    plan, _ = _fake_plan([True, True, True])
    assert len(plan.RemovedNodes) == 3                       # at most N - 1 nodes


def test_planner_drops_repeated_candidates():
    plan, calls = _fake_plan([True, True, True], candidates=[2, 0, 2, 0, 1])
    assert calls[0] == [3, 3, 3] and [s.Node for s in plan.Sweep] == ["node-2", "node-0", "node-1"]
    assert plan.RemovedNodes == ["node-0", "node-1", "node-2"]          # equal utilisation: nodeTree order


def test_gpu_index_joins_one_device_per_slot_with_dashes():
    assert scaledown.gpu_index(0) is None
    assert scaledown.gpu_index(0x1) == "0"
    assert scaledown.gpu_index(0x11) == "0-1"                            # AllocateGpuId: "0-1"
    assert scaledown.gpu_index(0x2100) == "2-3-3"                        # two slots on device 3


def test_checker_with_nothing_removed_reproduces_the_live_state():
    import checkers
    for seed in (0, 4):
        c = _compiled(*synth.make_mix(seed_no=seed, n_nodes=30))
        o, placed = _live(c)
        st, ext, slots = o.state(), o.state_ext(), o.gpu_slot_words()
        r = checkers.drain(o, placed, np.arange(c.n_nodes))
        assert (r["n_evicted"], r["n_blocked"], r["n_vanished"]) == (0, 0, 0)
        for k, v in o.state().items():
            assert np.array_equal(v, st[k]), k
        for k, v in o.state_ext().items():
            assert np.array_equal(v, ext[k]), k
        assert np.array_equal(o.gpu_slot_words(), slots)


def test_known_answer_plan(monkeypatch):
    c = _compiled(*known_answer())
    _o, placed = _live(c)
    assert np.bincount(placed, minlength=4).tolist() == [2, 2, 2, 2]
    run = checker_runner(c, placed)
    order = scaledown.NodeOrder(c)
    r = run([order.remaining([0]), order.remaining([0, 1]), order.remaining([0, 1, 2])])
    assert [(x["n_evicted"], x["n_unscheduled"]) for x in r] == [(2, 0), (4, 0), (6, 4)]
    plan = scaledown.plan_scale_down(c, placed, run, max_cpu=100, max_mem=100)
    assert len(plan.RemovedNodes) == 2 and [p["ok"] for p in plan.Prefixes] == [True, True, False]
    monkeypatch.setenv("MaxCPU", "75")
    plan = scaledown.plan_scale_down(c, placed, run)
    assert len(plan.RemovedNodes) == 1 and [p["ok"] for p in plan.Prefixes] == [True, False]


def test_session_refusals_without_a_device():
    sim = simulator.NewSimulator()
    with pytest.raises(RuntimeError, match="RunCluster"):
        sim.DrainNodes([["node-0"]])
    with pytest.raises(RuntimeError, match="RunCluster"):
        sim.PlanScaleDown()


DRAIN_VARIANTS = {
    # kernel -> (CTAs per scenario, threads per CTA, force_large)
    "simon_drain_kernel_256": (2, 128, False),
    "simon_drain_kernel_320": (2, 288, False),
    "simon_drain_kernel_384": (1, 352, False),
    "simon_drain_kernel_big": (4, 64, True),
}


def test_drain_variant_table_names_every_drain_kernel_of_the_variant_list():
    assert set(DRAIN_VARIANTS) == compiled_kernels("simon_drain_kernel_")


# ---- GPU --------------------------------------------------------------------------------------------------------------------

def _drains(c, rng, n_single=None):
    """Single-node drains of every node (or n_single of them) and a few multi-node drains."""
    nodes = list(range(c.n_nodes)) if n_single is None else rng.choice(c.n_nodes, size=n_single, replace=False).tolist()
    multi = [rng.choice(c.n_nodes, size=int(rng.integers(2, max(3, c.n_nodes // 3))), replace=False).tolist() for _ in range(6)]
    return [[g] for g in nodes] + multi


def _assert_drain_equal(a, b, what):
    for k in ("n_evicted", "n_placed", "n_unscheduled", "n_blocked", "n_vanished"):
        assert a[k] == b[k], (what, k, a[k], b[k])
    for k in ("evicted", "node", "gpu_slots", "blocked", "fail_pod"):
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), (what, k, a[k], b[k])
    assert np.array_equal(a["fail_counts"], b["fail_counts"]), what


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", sorted(DRAIN_VARIANTS))
def test_drain_variant_matches_checker(kernel):
    import checkers
    from simon_b200.engine import Engine
    cs, t, big = DRAIN_VARIANTS[kernel]
    rng = np.random.default_rng(11)
    for seed in (0, 2, 5):
        c = _compiled(*synth.make_mix(seed_no=seed, n_nodes=40))
        o, placed = _live(c)
        order = scaledown.NodeOrder(c)
        drains = _drains(c, rng, n_single=12)
        remain = [order.remaining(d) for d in drains]
        with Engine(c, record_scores=True, cluster_ctas=cs, threads_per_cta=t, force_large=big) as eng:
            got = eng.drain_run(placed, remain)
            assert eng.last_launch()["kernel"] == kernel
        for d, rl, g in zip(drains, remain, got):
            want = checkers.drain(o, placed, rl)
            _assert_drain_equal(g, want, f"{kernel} seed {seed} drain {d}")
            pos = g["node"] >= 0
            assert np.array_equal(g["score"][pos], want["score"][pos]), d
            st = o.state()
            idx = np.asarray(rl, dtype=np.int64)
            assert g["req_mcpu"] == int(st["req_mcpu"][idx].sum()) and g["req_mem"] == int(st["req_mem"][idx].sum())
            assert g["alloc_mcpu"] == int(c.snap["alloc_mcpu"][idx].sum())


def _recompiled(p, c, placed, removed, open_local=False, scs=None):
    """The equivalence that pins a drain: the cluster without the removed nodes, pod list [pods not on them, in order] +
    [evicted pods, in order], resumed with the first part's nodes as the prefix.  -> (compiled, out_node, gpu slot words, n first)."""
    from simon_b200.engine import Engine
    ev, bl, va = scaledown.classify(c, placed, removed)
    gone = set(ev) | {q for q, _ in bl} | set(va)
    names = c.node_names
    rm_names = {names[g] for g in removed}
    nodes = [n for n in p.nodes if O.name_of(n) not in rm_names]
    first = [q for q in range(len(p.pods)) if q not in gone]
    pods = [p.pods[q] for q in first] + [p.pods[q] for q in ev]
    c2 = compile_cluster(nodes, pods, p.ctx, open_local=open_local, storage_classes=scs, local_devices=open_local)
    prefix = np.array([c2.node_index(names[placed[q]]) if placed[q] >= 0 else placed[q] for q in first], np.int32)
    with Engine(c2) as eng:
        out = eng.schedule_resume(prefix)[0]
        slots = eng.gpu_slot_words()
    return c2, out, slots, len(first), ev


def _check_equivalence(p, c, placed, drains, open_local=False, scs=None):
    from simon_b200.engine import Engine
    order = scaledown.NodeOrder(c)
    remain = [order.remaining(d) for d in drains]
    with Engine(c) as eng:
        got = eng.drain_run(placed, remain)
    n_blocked = 0
    for d, rl, g in zip(drains, remain, got):
        c2, out, slots, nf, ev = _recompiled(p, c, placed, d, open_local, scs)
        assert [c.node_names[x] for x in rl] == c2.node_names          # the recompiled snapshot is the remaining nodes' order
        assert g["evicted"].tolist() == ev
        want = [c2.node_names[x] if x >= 0 else None for x in out[nf:]]
        have = [c.node_names[x] if x >= 0 else None for x in g["node"]]
        assert have == want, d
        assert np.array_equal(g["gpu_slots"], slots[nf:]), d
        n_blocked += g["n_blocked"]
    return got, n_blocked


@pytest.mark.gpu
def test_drains_equal_recompile_and_resume_gpu_share_c3():
    cluster, apps = synth.make_c3(n_nodes=2000, n_workloads=200, replicas=60, n_apps=2, gpu_pct=25, seed_no=9)
    p = simulator.plan(cluster, apps)
    c = compile_cluster(p.nodes, p.pods, p.ctx)
    from simon_b200.engine import Engine
    with Engine(c) as eng:
        placed = eng.schedule()[0]
    rng = np.random.default_rng(5)
    gpu_nodes = np.nonzero(c.snap["gpu_count"] > 0)[0]
    drains = [[int(g)] for g in rng.choice(gpu_nodes, 4, replace=False)] + [[int(g)] for g in rng.choice(c.n_nodes, 3, replace=False)]
    drains += [rng.choice(c.n_nodes, 40, replace=False).tolist()]
    # nodes holding a scheduler-placed pod with two GPU slots: its gpu-index names two devices
    from simon_b200.compiler import SCW_GPU_COUNT, SCW_GPU_MEM
    off, blob, cls = c.pods["class_off"], c.pods["class_blob"], c.pods["pod_class"]
    multi = [q for q in range(len(placed)) if placed[q] >= 0 and c.pods["pod_fixed_node"][q] == -1
             and blob[off[cls[q]] + SCW_GPU_MEM] > 0 and blob[off[cls[q]] + SCW_GPU_COUNT] >= 2]
    drains += [[int(placed[q])] for q in multi[:3]]
    got, _ = _check_equivalence(p, c, placed, drains)
    assert any((g["gpu_slots"] != 0).any() for g in got)                 # GPU-share pods were evicted and placed again
    # alibabacloud.com/gpu-index of the evicted pods: one device id per slot, "-"-joined, as the reference's GpuIdStrToIntList reads it
    order = scaledown.NodeOrder(c)
    res = scaledown.drain_results(c, placed, drains, [order.remaining(d) for d in drains], got)
    n_multi = 0
    for r, g in zip(res, got):
        for e, w in zip(r.EvictedPods, g["gpu_slots"].tolist()):
            if e.To is None or w == 0:
                assert e.GpuIndex is None
                continue
            ids = [int(x) for x in e.GpuIndex.split("-")]
            assert ids == sorted(ids) and all(ids.count(d) == (w >> (4 * d)) & 15 for d in range(8)), (e.GpuIndex, hex(w))
            n_multi += len(ids) >= 2
    assert n_multi > 0


@pytest.mark.gpu
def test_drains_equal_recompile_and_resume_config1_open_local(tmp_path):
    from test_open_local_capacity import _example
    from simon_b200.engine import Engine
    cluster, apps, _new = _example(tmp_path)
    scs = list(cluster.StorageClasss) + [sc for a in apps for sc in a.Resource.StorageClasss]
    p = simulator.plan(cluster, apps)
    c = compile_cluster(p.nodes, p.pods, p.ctx, open_local=True, storage_classes=scs, local_devices=True)
    with Engine(c) as eng:
        placed = eng.schedule()[0]
    drains = [[g] for g in range(c.n_nodes)] + [[0, 1]]
    got, n_blocked = _check_equivalence(p, c, placed, drains, open_local=True, scs=scs)
    assert n_blocked > 0                                                 # the volume pods (and static pods) block
    assert any(g["n_evicted"] for g in got)


@pytest.mark.gpu
def test_live_state_after_a_drain_batch_and_moves_unchanged():
    from simon_b200.engine import Engine
    c = _compiled(*synth.make_mix(seed_no=3, n_nodes=40))
    o, placed = _live(c)
    with Engine(c) as eng:
        out = eng.schedule()[0]
        assert np.array_equal(out, placed)
        st, ext, slots = eng.state(), eng.state_ext(), eng.gpu_slot_words()
        moves = np.array([(q, g) for q in range(0, len(placed), 3) for g in range(0, c.n_nodes, 7)], np.uint32)
        eng.moves_upload(moves)
        before = eng.moves_run(k=8)
        order = scaledown.NodeOrder(c)
        eng.drain_run(placed, [order.remaining([g]) for g in range(c.n_nodes)])
        for k, v in eng.state().items():
            assert np.array_equal(v, st[k]), k
        for k, v in eng.state_ext().items():
            assert np.array_equal(v, ext[k]), k
        assert np.array_equal(eng.gpu_slot_words(), slots)
        after = eng.moves_run(k=8)
        assert np.array_equal(after["gain"], before["gain"]) and np.array_equal(after["code"], before["code"])
        assert after["topk"] == before["topk"]


@pytest.mark.gpu
def test_drain_refusals():
    from simon_b200.engine import Engine
    c = _compiled(*known_answer())
    _o, placed = _live(c)
    with Engine(c) as eng:
        with pytest.raises(RuntimeError, match="leaves no node"):
            eng.drain_run(placed, [np.zeros(0, np.uint32)])
        with pytest.raises(RuntimeError, match="listed twice"):
            eng.drain_run(placed, [np.array([0, 0], np.uint32)])
        with pytest.raises(RuntimeError, match="out of range"):
            eng.drain_run(placed, [np.array([0, 9], np.uint32)])
        bad = placed.copy()
        bad[0] = 17
        with pytest.raises(RuntimeError, match="out of range"):
            eng.drain_run(bad, [np.array([1, 2, 3], np.uint32)])
        # a single run after refused and completed drains launches the placement kernels and places as before
        assert np.array_equal(eng.schedule()[0], placed)
        assert eng.last_launch()["kernel"].startswith("simon_place_kernel_")
        eng.drain_run(placed, [np.array([1, 2, 3], np.uint32)])
        assert eng.last_launch()["kernel"].startswith("simon_drain_kernel_")
        assert np.array_equal(eng.schedule()[0], placed)
        assert eng.last_launch()["kernel"].startswith("simon_place_kernel_")
        eng.reset()
        assert eng.run_scenarios([np.arange(c.n_nodes, dtype=np.uint32)])[0][0]["n_unscheduled"] == 0
        assert eng.last_launch()["kernel"].startswith("simon_place_kernel_")


@pytest.mark.gpu
def test_session_drain_nodes_and_plan_scale_down(monkeypatch):
    cluster, apps = known_answer()
    with simulator.NewSimulator() as sim:
        sim.RunCluster(simulator.PrepareCluster(cluster))
        sim.ScheduleApp(apps[0])
        res = sim.DrainNodes([["node-0"], ["node-0", "node-1"], ["node-0", "node-1", "node-2"]])
        assert [r.Drainable for r in res] == [True, True, False]
        assert [len(r.EvictedPods) for r in res] == [2, 4, 6] and len(res[2].UnscheduledPods) == 4
        assert all(e.From in r.RemovedNodes and (e.To is None or e.To not in r.RemovedNodes) for r in res for e in r.EvictedPods)
        assert res[2].UnscheduledPods[0].Reason.startswith("failed to schedule pod") and "0/1 nodes are available" in res[2].UnscheduledPods[0].Reason
        assert res[1].CapsOk and res[1].Occupancy["req_mcpu"] == 8000 and res[1].Occupancy["alloc_mcpu"] == 8000
        plan = sim.PlanScaleDown()
        assert len(plan.RemovedNodes) == 2 and len(plan.Sweep) == 4 and all(s.Drainable for s in plan.Sweep)
        monkeypatch.setenv("MaxCPU", "75")
        assert len(sim.PlanScaleDown().RemovedNodes) == 1
    monkeypatch.delenv("MaxCPU")
    res = scaledown.drain(cluster, apps, [["node-3"]])
    assert res[0].Drainable and len(res[0].EvictedPods) == 2
