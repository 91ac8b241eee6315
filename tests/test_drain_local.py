"""Node drains that move pods with Open-Local volumes (simon_drain_run_local, Engine.drain_run(..., local=True), local_volumes=True in
simon_b200.scaledown and the session), and the MaxVG cap on drains.

CPU: the classification with and without the opt-in, the variant table, the planner's MaxVG rule with a fake runner, the session's
refusal.  GPU: drains against the recompile + simon_schedule_resume equivalence with storage and devices, the final VG and device
state against the host's replay of Bind, every drain-local kernel variant, batches split into chunks, PDBs, the context state a local
drain batch leaves, and the session entry points on the reference example."""
import copy
import ctypes

import numpy as np
import pytest

from simon_b200 import objects as O, scaledown, simulator, synth
from simon_b200.compiler import compile_cluster
from util import compiled_kernels

GI = 1 << 30


def _example_compiled(tmp_path):
    from test_open_local_capacity import _example
    cluster, apps, _new = _example(tmp_path)
    scs = list(cluster.StorageClasss) + [sc for a in apps for sc in a.Resource.StorageClasss]
    p = simulator.plan(cluster, apps)
    return p, compile_cluster(p.nodes, p.pods, p.ctx, open_local=True, storage_classes=scs, local_devices=True), scs


def _synth_compiled(n_nodes, seed):
    cluster, apps = synth.make_open_local(n_nodes=n_nodes, n_workloads=24, replicas=12, seed_no=seed)
    scs = list(cluster.StorageClasss)
    p = simulator.plan(cluster, apps)
    return p, compile_cluster(p.nodes, p.pods, p.ctx, open_local=True, storage_classes=scs, local_devices=True), scs


# ---- CPU --------------------------------------------------------------------------------------------------------------------

def test_classification_with_local_volumes(tmp_path):
    _p, c, _scs = _example_compiled(tmp_path)
    local = c.storage.class_local
    cls = c.pods["pod_class"]
    fixed = c.pods["pod_fixed_node"]
    guard = scaledown.pod_guard(c)
    # a synthetic live state: every pod that reaches the scheduler on node 0 (classification reads nothing else of it)
    placed = np.where(fixed >= 0, fixed, 0).astype(np.int32)
    for g in range(c.n_nodes):
        ev0, bl0, va0 = scaledown.classify(c, placed, [g])
        ev1, bl1, va1 = scaledown.classify(c, placed, [g], local_volumes=True)
        assert va1 == va0
        vol = [q for q, why in bl0 if why == scaledown.BLOCK_LOCAL_STORAGE]
        assert all(local[int(cls[q])] and fixed[q] < 0 for q in vol)
        # pods with volumes move from blocked to evicted, in pod order; spec.nodeName pods still block
        assert ev1 == sorted(ev0 + vol)
        assert bl1 == [(q, why) for q, why in bl0 if why == scaledown.BLOCK_NODE_NAME]
        assert all(fixed[q] >= 0 for q, _ in bl1)
        if g == 0:
            assert vol and bl1, "node 0 holds pods with volumes and spec.nodeName pods"
            assert any(local[int(cls[q])] for q in ev1) and all(guard[q] != 0 for q in ev1)
    # a pod bound by spec.nodeName whose class has volumes blocks either way
    q_fixed_local = [q for q in range(len(fixed)) if fixed[q] >= 0 and local[int(cls[q])]]
    for q in q_fixed_local:
        g = int(fixed[q])
        if guard[q] == g:
            continue
        assert (q, scaledown.BLOCK_NODE_NAME) in scaledown.classify(c, placed, [g], local_volumes=True)[1]


DRAIN_LOCAL_VARIANTS = {
    # kernel -> (CTAs per scenario, threads per CTA, force_large)
    "simon_drain_local_kernel_256": (2, 128, False),
    "simon_drain_local_kernel_320": (2, 288, False),
    "simon_drain_local_kernel_384": (1, 352, False),
    "simon_drain_local_kernel_big": (4, 64, True),
}


def test_drain_local_variant_table_names_every_drain_local_kernel():
    assert set(DRAIN_LOCAL_VARIANTS) == compiled_kernels("simon_drain_local_kernel_")
    # the plain drain kernels keep their prefix to themselves
    assert not compiled_kernels("simon_drain_kernel_") & set(DRAIN_LOCAL_VARIANTS)


def _fake_vg_plan(vg_pct, max_vg, with_vg=True):
    """plan_scale_down on the 4-node known-answer cluster with a runner whose k-prefix results carry VG occupancy vg_pct[k - 1] %
    (the sweep: 10 %), CPU and memory at 0 %."""
    from test_drain import _compiled, known_answer
    c = _compiled(*known_answer())

    def runner(remain_lists):
        out = []
        for rl in remain_lists:
            k = c.n_nodes - len(rl)
            r = dict(n_blocked=0, n_unscheduled=0, n_evicted=2, req_mcpu=0, alloc_mcpu=1, req_mem=0, alloc_mem=1)
            if with_vg:
                r.update(vg_requested=vg_pct[k - 1], vg_capacity=100)
            out.append(r)
        return out
    placed = np.repeat(np.arange(c.n_nodes), 2).astype(np.int32)
    return scaledown.plan_scale_down(c, placed, runner, batch=2, max_cpu=100, max_mem=100, max_vg=max_vg)


def test_planner_applies_max_vg_to_results_with_vg_sums(monkeypatch):
    monkeypatch.delenv("MaxVG", raising=False)
    plan = _fake_vg_plan([10, 40, 70], None)                  # MaxVG unset: 100
    assert len(plan.RemovedNodes) == 3 and all(p["ok"] for p in plan.Prefixes)
    plan = _fake_vg_plan([10, 40, 70], 50)                    # k = 3 is the first prefix over the cap
    assert len(plan.RemovedNodes) == 2 and [p["ok"] for p in plan.Prefixes] == [True, True, False]
    plan = _fake_vg_plan([10, 60, 30], 50)                    # k = 2 ends the plan, though k = 3 would pass again
    assert len(plan.RemovedNodes) == 1 and [p["k"] for p in plan.Prefixes] == [1, 2]
    monkeypatch.setenv("MaxVG", "5")
    assert len(_fake_vg_plan([10, 40, 70], None).RemovedNodes) == 0      # the default reads MaxVG
    # results without VG sums (drains that block local volumes) ignore MaxVG
    assert len(_fake_vg_plan([10, 40, 70], None, with_vg=False).RemovedNodes) == 3
    assert len(_fake_vg_plan([10, 40, 70], 0, with_vg=False).RemovedNodes) == 3
    monkeypatch.setenv("MaxVG", "x")
    assert len(_fake_vg_plan([10, 40, 70], None, with_vg=False).RemovedNodes) == 3
    with pytest.raises(ValueError, match="MaxVG"):
        _fake_vg_plan([10, 40, 70], None)


def test_drain_results_carry_vg_sums_and_apply_max_vg():
    from test_drain import _compiled, known_answer
    c = _compiled(*known_answer())
    placed = np.repeat(np.arange(c.n_nodes), 2).astype(np.int32)
    order = scaledown.NodeOrder(c)
    raw = dict(n_evicted=0, n_placed=0, n_unscheduled=0, n_blocked=0, n_vanished=0, req_mcpu=0, alloc_mcpu=1, req_mem=0, alloc_mem=1,
               evicted=np.zeros(0, np.uint32), node=np.zeros(0, np.int32), gpu_slots=np.zeros(0, np.uint32), blocked=np.zeros(0, np.uint32),
               fail_counts=np.zeros((0, 24), np.uint32), fail_pod=np.zeros(0, np.uint32))
    with_vg = dict(raw, vg_requested=60, vg_capacity=100)
    rl = [order.remaining([0])]
    r = scaledown.drain_results(c, placed, [[0]], rl, [with_vg], max_vg=50)[0]
    assert not r.CapsOk and r.Occupancy["vg_requested"] == 60 and r.Occupancy["vg_capacity"] == 100
    assert scaledown.drain_results(c, placed, [[0]], rl, [with_vg], max_vg=60)[0].CapsOk
    r = scaledown.drain_results(c, placed, [[0]], rl, [raw], max_vg=0)[0]
    assert r.CapsOk and "vg_requested" not in r.Occupancy


def test_session_refuses_local_volumes_without_open_local():
    sim = simulator.NewSimulator()
    with pytest.raises(ValueError, match="WithOpenLocal"):
        sim.DrainNodes([["node-0"]], local_volumes=True)
    with pytest.raises(ValueError, match="WithOpenLocal"):
        sim.PlanScaleDown(local_volumes=True)


# ---- GPU --------------------------------------------------------------------------------------------------------------------

def _drains(c, rng, n_single=None, n_multi=4):
    nodes = list(range(c.n_nodes)) if n_single is None else sorted(rng.choice(c.n_nodes, size=n_single, replace=False).tolist())
    multi = [rng.choice(c.n_nodes, size=int(rng.integers(2, max(3, min(c.n_nodes - 1, 12)))), replace=False).tolist()
             for _ in range(n_multi)]
    return [[g] for g in nodes] + multi


def _recompiled_local(p, c, placed, removed, scs):
    """The equivalence that pins a local drain: the cluster without the removed nodes, compiled with Open-Local storage and devices,
    pod list [pods not on them, in order] + [evicted pods, in order], resumed with the first part's nodes as the prefix.
    -> (compiled, out_node, gpu slot words, VG requested [V][N], device masks [N], n first, evicted)."""
    from simon_b200.engine import Engine
    ev, bl, va = scaledown.classify(c, placed, removed, local_volumes=True)
    gone = set(ev) | {q for q, _ in bl} | set(va)
    names = c.node_names
    rm_names = {names[g] for g in removed}
    nodes = [n for n in p.nodes if O.name_of(n) not in rm_names]
    first = [q for q in range(len(p.pods)) if q not in gone]
    pods = [p.pods[q] for q in first] + [p.pods[q] for q in ev]
    c2 = compile_cluster(nodes, pods, p.ctx, open_local=True, storage_classes=scs, local_devices=True)
    prefix = np.array([c2.node_index(names[placed[q]]) if placed[q] >= 0 else placed[q] for q in first], np.int32)
    with Engine(c2) as eng:
        out = eng.schedule_resume(prefix)[0]
        slots = eng.gpu_slot_words()
        vg, dev = eng.storage_state(), eng.device_state()
    return c2, out, slots, vg, dev, len(first), ev


def _host_replay(c, placed, d, rl):
    """The final VG requested and device masks of drain d by the host's restatement of Bind (storage.StorageReplay): the live pods in
    pod order (the scheduler-placed ones: spec.nodeName pods bypass Bind), then the evicted pods at their new nodes in pod order.
    Per node that is its remaining live pods, then its evicted arrivals; a removed node keeps its live state."""
    from simon_b200.storage import StorageReplay
    rep = StorageReplay(c.storage, c.node_names)
    cls, fixed = c.pods["pod_class"], c.pods["pod_fixed_node"]
    for q, g in enumerate(placed.tolist()):
        if g >= 0 and fixed[q] < 0:
            rep.bind(int(cls[q]), g)
    for q, g in zip(d["evicted"].tolist(), d["node"].tolist()):
        if g >= 0:
            rep.bind(int(cls[q]), g)
    vg, dev = rep.requested(), rep.alloc_masks()
    st = c.storage
    req = cap = 0
    for g in rl.tolist():
        nv = int(st.node_n_vg[g])
        if nv >= 0:
            req += int(vg[:nv, g].sum())
            cap += int(st.vg_capacity[:nv, g].sum())
    return vg, dev, req, cap


def _check_local_drains(p, c, placed, drains, scs, eng_kw=None, chunk=None, recompile=None):
    """Every drain of a local batch against the recompile + resume path (drains listed in `recompile`, all by default) and against
    the host's replay of Bind; -> the results."""
    from simon_b200.engine import Engine
    order = scaledown.NodeOrder(c)
    remain = [order.remaining(d) for d in drains]
    with Engine(c, **(eng_kw or {})) as eng:
        got = eng.drain_run(placed, remain, local=True, chunk=chunk)
        kernel = eng.last_launch()["kernel"]
        n_last = len(drains) - (len(drains) // chunk) * chunk if chunk else len(drains)
        n_last = n_last or (chunk or len(drains))
        states = {len(drains) - n_last + i: eng.scenario_storage_state(i) for i in range(n_last)}
    assert kernel.startswith("simon_drain_local_kernel_"), kernel
    V = c.storage.n_vgs
    for j, (d, rl, g) in enumerate(zip(drains, remain, got)):
        vg_h, dev_h, req, cap = _host_replay(c, placed, g, rl)
        assert (g["vg_requested"], g["vg_capacity"]) == (req, cap), d
        if j in states:
            vg_d, dev_d = states[j]
            assert np.array_equal(vg_d, vg_h), d
            assert np.array_equal(dev_d, dev_h), d
        if recompile is not None and j not in recompile:
            continue
        c2, out, slots, vg2, dev2, nf, ev = _recompiled_local(p, c, placed, d, scs)
        assert [c.node_names[x] for x in rl] == c2.node_names
        assert g["evicted"].tolist() == ev, d
        want = [c2.node_names[x] if x >= 0 else None for x in out[nf:]]
        have = [c.node_names[x] if x >= 0 else None for x in g["node"]]
        assert have == want, d
        assert np.array_equal(g["gpu_slots"], slots[nf:]), d
        for g2, nm in enumerate(c2.node_names):
            x = c.node_index(nm)
            nv = int(c2.storage.node_n_vg[g2])
            assert vg_h[:max(nv, 0), x].tolist() == vg2[:max(nv, 0), g2].tolist(), (d, nm)
            assert int(dev_h[x]) == int(dev2[g2]), (d, nm)
        assert V >= c2.storage.n_vgs
    return got


def _volume_stats(c, got):
    local = c.storage.class_local
    cls = c.pods["pod_class"]
    moved = [(q, n) for g in got for q, n in zip(g["evicted"].tolist(), g["node"].tolist()) if local[int(cls[q])]]
    return len(moved), sum(1 for _, n in moved if n >= 0)


@pytest.mark.gpu
def test_local_drains_equal_recompile_and_resume_reference_example(tmp_path):
    from simon_b200.engine import Engine
    p, c, scs = _example_compiled(tmp_path)
    with Engine(c) as eng:
        placed = eng.schedule()[0]
    drains = [[g] for g in range(c.n_nodes)] + [[0, 1], [1, 3], [0, 2, 3]]
    got = _check_local_drains(p, c, placed, drains, scs)
    n_vol, n_landed = _volume_stats(c, got)
    assert n_vol > 0


@pytest.mark.gpu
@pytest.mark.parametrize("n_nodes,seed", [(200, 3), (300, 8)])
def test_local_drains_equal_recompile_and_resume_synthetic(n_nodes, seed):
    from simon_b200.engine import Engine
    p, c, scs = _synth_compiled(n_nodes, seed)
    with Engine(c) as eng:
        placed = eng.schedule()[0]
    rng = np.random.default_rng(seed)
    drains = _drains(c, rng)
    got = _check_local_drains(p, c, placed, drains, scs)
    n_vol, n_landed = _volume_stats(c, got)
    assert n_vol > 0 and n_landed > 0, (n_vol, n_landed)
    assert any(g["n_unscheduled"] == 0 and g["n_evicted"] > 0 for g in got)


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", sorted(DRAIN_LOCAL_VARIANTS))
def test_drain_local_variant_matches_equivalence(kernel):
    from simon_b200.engine import Engine
    cs, t, big = DRAIN_LOCAL_VARIANTS[kernel]
    p, c, scs = _synth_compiled(120, 5)
    with Engine(c) as eng:
        placed = eng.schedule()[0]
    rng = np.random.default_rng(17)
    drains = _drains(c, rng, n_single=10, n_multi=3)
    eng_kw = dict(record_scores=True, cluster_ctas=cs, threads_per_cta=t, force_large=big)
    with Engine(c, **eng_kw) as eng:
        eng.drain_run(placed, [scaledown.NodeOrder(c).remaining(drains[0])], local=True)
        li = eng.last_launch()
        assert li["kernel"] == kernel and li["local"] and li["large"] == big
    got = _check_local_drains(p, c, placed, drains, scs, eng_kw=eng_kw, recompile=range(0, len(drains), 2))
    assert _volume_stats(c, got)[0] > 0


@pytest.mark.gpu
def test_local_drain_batch_split_into_chunks_equals_one_batch():
    from simon_b200.engine import Engine
    p, c, scs = _synth_compiled(150, 4)
    with Engine(c) as eng:
        placed = eng.schedule()[0]
        order = scaledown.NodeOrder(c)
        drains = _drains(c, np.random.default_rng(2), n_single=40, n_multi=5)
        remain = [order.remaining(d) for d in drains]
        one = eng.drain_run(placed, remain, local=True)
        states_one = [eng.scenario_storage_state(i) for i in range(len(drains))]
        parts = eng.drain_run(placed, remain, local=True, chunk=7)
        assert eng.last_drain["chunks"] == -(-len(drains) // 7)
        n_last = len(drains) - 7 * (len(drains) // 7) or 7
        for i in range(n_last):
            j = len(drains) - n_last + i
            vg, dev = eng.scenario_storage_state(i)
            assert np.array_equal(vg, states_one[j][0]) and np.array_equal(dev, states_one[j][1]), j
    for a, b in zip(one, parts):
        for k in ("n_evicted", "n_placed", "n_unscheduled", "n_blocked", "n_vanished", "vg_requested", "vg_capacity",
                  "req_mcpu", "req_mem"):
            assert a[k] == b[k], k
        for k in ("evicted", "node", "gpu_slots", "score", "blocked", "fail_pod", "fail_counts"):
            assert np.array_equal(a[k], b[k]), k


@pytest.mark.gpu
def test_local_drain_pdb_names_the_budget(tmp_path):
    """A PDB with maxUnavailable 0 over the nginx-lvm StatefulSet: a local drain of a node holding one of its pods evicts it and
    violates the PDB; a plain drain of that node reports the pod as blocked instead."""
    from simon_b200 import disruption
    from simon_b200.engine import Engine
    p, c, scs = _example_compiled(tmp_path)
    pdb = {"apiVersion": "policy/v1beta1", "kind": "PodDisruptionBudget", "metadata": {"name": "lvm", "namespace": "default"},
           "spec": {"maxUnavailable": 0, "selector": {"matchLabels": {"app": "nginx-lvm"}}}}
    tables = disruption.compile_pdbs([pdb], c)
    with Engine(c) as eng:
        placed = eng.schedule()[0]
        local = c.storage.class_local
        cls = c.pods["pod_class"]
        members = [q for q in range(len(placed)) if placed[q] >= 0 and local[int(cls[q])] and c.pods["pod_fixed_node"][q] < 0
                   and "nginx-lvm" in c.pod_recs[q].name]
        assert members
        g = int(placed[members[0]])
        eng.pdbs_upload(tables)
        order = scaledown.NodeOrder(c)
        loc = eng.drain_run(placed, [order.remaining([g])], local=True)[0]
        assert loc["n_pdb_violated"] == 1 and not scaledown.drainable(loc)
        assert set(members) & set(loc["evicted"].tolist()) and not set(members) & set(loc["blocked"].tolist())
        allowed = eng.pdbs_allowed()
        res = scaledown.drain_results(c, placed, [[g]], [order.remaining([g])], [loc], pdbs=tables, allowed=allowed)[0]
        assert [v.Name for v in res.PdbViolations] == ["default/lvm"] and not res.Drainable
        plain = eng.drain_run(placed, [order.remaining([g])])[0]
        assert plain["n_pdb_violated"] == 0 and set(members) & set(plain["blocked"].tolist())
        assert not set(members) & set(plain["evicted"].tolist())


@pytest.mark.gpu
def test_context_state_after_a_local_drain_batch():
    from simon_b200.engine import Engine, lib
    p, c, scs = _synth_compiled(160, 6)
    with Engine(c) as eng:
        placed = eng.schedule()[0]
        st, ext, slots = eng.state(), eng.state_ext(), eng.gpu_slot_words()
        vg, dev = eng.storage_state(), eng.device_state()
        movable = [q for q in range(len(placed)) if placed[q] >= 0 and not c.storage.class_local[int(c.pods["pod_class"][q])]]
        moves = np.array([(q, g) for q in movable[::5] for g in range(0, c.n_nodes, 11)], np.uint32)
        eng.moves_upload(moves)
        before = eng.moves_run(k=8)
        order = scaledown.NodeOrder(c)
        remain = [order.remaining([g]) for g in range(0, c.n_nodes, 3)]
        plain_before = eng.drain_run(placed, remain)
        assert eng.last_launch()["kernel"].startswith("simon_drain_kernel_") and not eng.last_launch()["local"]
        with pytest.raises(RuntimeError, match="simon_drain_run_local"):
            eng.scenario_storage_state(0)                     # a plain drain batch serves no storage download
        eng.drain_run(placed, remain, local=True)
        assert eng.last_launch()["kernel"].startswith("simon_drain_local_kernel_") and eng.last_launch()["local"]
        eng.scenario_storage_state(len(remain) - 1)
        for k, v in eng.state().items():
            assert np.array_equal(v, st[k]), k
        for k, v in eng.state_ext().items():
            assert np.array_equal(v, ext[k]), k
        assert np.array_equal(eng.gpu_slot_words(), slots)
        assert np.array_equal(eng.storage_state(), vg) and np.array_equal(eng.device_state(), dev)
        after = eng.moves_run(k=8)
        assert np.array_equal(after["gain"], before["gain"]) and np.array_equal(after["code"], before["code"])
        assert after["topk"] == before["topk"]
        # a plain drain afterwards runs the plain kernels and gives what it gave before; the storage download then refuses
        plain_after = eng.drain_run(placed, remain)
        assert eng.last_launch()["kernel"].startswith("simon_drain_kernel_")
        for a, b in zip(plain_before, plain_after):
            for k in ("n_evicted", "n_placed", "n_unscheduled", "n_blocked", "req_mcpu", "req_mem"):
                assert a[k] == b[k], k
            for k in ("evicted", "node", "gpu_slots", "blocked", "fail_counts"):
                assert np.array_equal(a[k], b[k]), k
        with pytest.raises(RuntimeError, match="simon_drain_run_local"):
            eng.scenario_storage_state(0)
        # a local batch, then an upload: the download refuses
        eng.drain_run(placed, remain, local=True)
        eng.scenario_storage_state(0)
        eng._check(lib().simon_storage_upload(eng.h, ctypes.byref(eng.storage)))
        with pytest.raises(RuntimeError, match="simon_drain_run_local"):
            eng.scenario_storage_state(0)
        eng._check(lib().simon_devices_upload(eng.h, ctypes.byref(eng.devices)))     # a storage upload drops the devices
        eng.drain_run(placed, remain, local=True)
        eng.scenario_storage_state(0)
        eng._check(lib().simon_devices_upload(eng.h, ctypes.byref(eng.devices)))
        with pytest.raises(RuntimeError, match="simon_drain_run_local"):
            eng.scenario_storage_state(0)
        # a later scenario batch replaces the drain batch and is served
        eng.reset()
        res, _ = eng.run_scenarios_local([np.arange(c.n_nodes, dtype=np.uint32)])
        vg_b, _dev_b = eng.scenario_storage_state(0)
        assert int(vg_b.sum()) >= int(c.storage.vg_requested.sum())
        # the batch pool's per-scenario bytes count the Open-Local columns: VG requested [V][N], the raw-score scratch [N], the
        # device masks [N] and the local result
        per_local, _free = eng.drain_budget()
    plain_c = copy.copy(c)
    plain_c.storage = None
    with Engine(plain_c) as eng:
        per_plain, _free = eng.drain_budget()
        with pytest.raises(RuntimeError, match="before simon_storage_upload"):
            eng.drain_run(placed, remain[:1], local=True)
    N, V = c.n_nodes, c.storage.n_vgs
    assert per_local - per_plain == 8 * V * N + 4 * N + 4 * N + 24


def _session_example(tmp_path):
    """The reference example's demo_1 cluster plus one node of newnode/demo_1 (named simon-new-0), with the open_local app alone."""
    from test_open_local_capacity import _example
    from simon_b200.workloads import make_valid_node_by_node
    cluster, apps, new_node = _example(tmp_path)
    app = [a for a in apps if a.Name == "open_local"][0]
    n = make_valid_node_by_node(O.deep_copy(new_node), "simon-new-0")
    cluster = copy.copy(cluster)
    cluster.Nodes = list(cluster.Nodes) + [n]
    return cluster, app


@pytest.mark.gpu
def test_session_drains_and_plans_with_local_volumes(tmp_path, monkeypatch):
    """demo_1 + simon-new-0 with the open_local app: the four nginx-lvm replicas (1 CPU, 10 + 40 GiB of LVM each; their HDD claim names
    a StorageClass nobody defines and is dropped) can go only to worker-1 (2 x 100 GiB) and simon-new-0 (500 GiB): master-1 is tainted,
    master-2 / master-3 carry no storage.  The live state has all four on worker-1, whose VGs they fill.  The masters hold static pods
    (spec.nodeName), so they block with or without the opt-in; simon-new-0 holds nothing that moves.  Without the opt-in worker-1's
    volume pods block its drain; with it they move to simon-new-0, and the remaining annotated nodes are master-1 and simon-new-0
    (700 GiB), of which the four pods request 200 GiB.  The plan: by utilisation simon-new-0 comes first, then worker-1; k = 1
    removes simon-new-0 (worker-1 keeps its pods: 200 of master-1 + worker-1's 400 GiB), k = 2 leaves the nginx-lvm pods no node,
    so the plan is [simon-new-0] either way, with an order one node longer.  MaxVG = 0 rejects k = 1 (200 GiB requested): no node."""
    for k in ("MaxVG", "MaxCPU", "MaxMemory"):
        monkeypatch.delenv(k, raising=False)
    cluster, app = _session_example(tmp_path)
    with simulator.NewSimulator(simulator.WithOpenLocal(devices=True)) as sim:
        sim.RunCluster(simulator.PrepareCluster(cluster))
        sim.ScheduleApp(app)
        names = ["master-1", "master-2", "master-3", "simon-new-0", "worker-1"]
        plain = sim.DrainNodes([[nm] for nm in names])
        loc = sim.DrainNodes([[nm] for nm in names], local_volumes=True)
        assert [r.Drainable for r in plain] == [False, False, False, True, False]
        assert [r.Drainable for r in loc] == [False, False, False, True, True]
        w0, w1 = plain[4], loc[4]
        assert [b.Reason for b in w0.BlockedPods] == [scaledown.BLOCK_LOCAL_STORAGE] * 4 and not w0.EvictedPods
        assert [(e.Pod.name, e.From, e.To) for e in w1.EvictedPods] == [(f"nginx-lvm-{i}", "worker-1", "simon-new-0") for i in range(4)]
        assert not w1.BlockedPods and not w1.UnscheduledPods and w1.CapsOk
        assert (w1.Occupancy["vg_requested"], w1.Occupancy["vg_capacity"]) == (200 * GI, 700 * GI)
        assert "vg_requested" not in w0.Occupancy
        for a, b in zip(plain[:3], loc[:3]):                     # static pods block the masters either way
            assert all(x.Reason == scaledown.BLOCK_NODE_NAME for x in a.BlockedPods + b.BlockedPods) and len(b.BlockedPods) == 4
        plan0 = sim.PlanScaleDown()
        plan1 = sim.PlanScaleDown(local_volumes=True)
        assert plan0.RemovedNodes == ["simon-new-0"] and plan0.Order == ["simon-new-0"]
        assert {s.Node: s.Drainable for s in plan1.Sweep}["worker-1"]
        assert plan1.Order == ["simon-new-0", "worker-1"] and plan1.RemovedNodes == ["simon-new-0"]
        assert [(q["k"], q["ok"]) for q in plan1.Prefixes] == [(1, True), (2, False)]
        assert (plan1.Prefixes[0]["vg_requested"], plan1.Prefixes[0]["vg_capacity"]) == (200 * GI, 400 * GI)
        assert plan1.Prefixes[1]["n_unscheduled"] == 4
        monkeypatch.setenv("MaxVG", "0")
        plan_vg = sim.PlanScaleDown(local_volumes=True)
        assert plan_vg.RemovedNodes == [] and [(q["k"], q["ok"]) for q in plan_vg.Prefixes] == [(1, False)]
        assert sim.PlanScaleDown().RemovedNodes == ["simon-new-0"]        # without the opt-in MaxVG does not apply
    monkeypatch.delenv("MaxVG")
    res = scaledown.drain(cluster, [app], [["worker-1"]], simulator.WithOpenLocal(devices=True), local_volumes=True)
    assert res[0].Drainable and [e.To for e in res[0].EvictedPods] == ["simon-new-0"] * 4
