"""Move scope (simon_moves_set_scope): candidate moves of GPU-share classes and of classes with DoNotSchedule spread constraints.
CPU: the scoped checker (tests/checkers.c, the oracle's own cycle stages) against the unscoped oracle, hand-derived known
answers, and an object-level replay of sampled moves.  GPU: the engine's scoped runs against the checker."""
import numpy as np
import pytest

import checkers
from simon_b200.abi import SFC_GPU, SFC_PTS_MISSING, SFC_PTS_SKEW, SFC_STATIC
from util import make_case

GI = 1 << 30
GPU, HARD = 1, 2
# the four clusters of test_moves.py's GPU parity test
CASES = [
    ("mix", dict(seed_no=103, n_nodes=95, n_workloads=40, max_replicas=7), 30000),
    ("mix", dict(seed_no=215, n_nodes=45, n_workloads=30, max_replicas=9), 20000),
    ("c3", dict(n_nodes=1500, n_workloads=200, replicas=20, n_apps=4, seed_no=5), 200000),
    ("c2", dict(n_nodes=300, n_workloads=30, replicas=30, seed_no=2), 50000),
]
# clusters with GPU-share pods placed by the scheduler and DoNotSchedule zone spread (synth.make_c3(gpu_pct=...))
GPU_CASES = [
    ("c3", dict(n_nodes=400, n_workloads=80, replicas=10, n_apps=2, seed_no=21, gpu_pct=25), 40000),
    ("c3", dict(n_nodes=1500, n_workloads=200, replicas=20, n_apps=4, seed_no=5, gpu_pct=25), 200000),
]


def _state(kind, **kw):
    from oracle.binding import Oracle
    p, c = make_case(kind, **kw)
    o = Oracle(c)
    out = o.schedule()[0]
    return p, c, o, out


def _moves(out, c, n, seed=11):
    from simon_b200 import moves as M
    mv = M.sample_moves(len(out), c.n_nodes, n, seed=seed, placement=out)
    mv[:50, 0] = np.arange(50) % max(len(out), 1)           # some arbitrary pods too (unscheduled / pre-bound ones among them)
    return mv


def _class_word(c, w):
    blob, off = c.pods["class_blob"], c.pods["class_off"]
    return np.array([int(blob[int(off[k]) + w]) for k in range(len(off) - 1)], np.int64)


def _needs(c):
    """per class: the scope bits it needs (0: movable without a scope), -1 if never movable (pinned)"""
    from simon_b200 import compiler as K
    need = (_class_word(c, K.SCW_GPU_MEM) > 0) * GPU + (_class_word(c, K.SCW_N_PTS_HARD) > 0) * HARD
    return np.where(_class_word(c, K.SCW_FLAGS) & K.CLS_PINNED, -1, need)


# ---------------------------------------------------------------------------------------------------------------- CPU ----

@pytest.mark.parametrize("kind,kw,n", CASES)
def test_scope0_checker_equals_moves_score(kind, kw, n):
    p, c, o, out = _state(kind, **kw)
    mv = _moves(out, c, n)
    g0, c0 = o.moves_score(mv, out)
    g1, c1, sl = checkers.moves_score(o, mv, out, 0)
    np.testing.assert_array_equal(c1, c0)
    np.testing.assert_array_equal(g1, g0)
    assert sl is None


@pytest.mark.parametrize("kind,kw,n", CASES[:2] + GPU_CASES[:1])
def test_scope_bits_change_only_admitted_not_movable_codes(kind, kw, n):
    from simon_b200 import abi
    p, c, o, out = _state(kind, **kw)
    mv = _moves(out, c, n)
    g0, c0 = o.moves_score(mv, out)
    need = _needs(c)
    cls = c.pods["pod_class"][np.minimum(mv[:, 0], len(out) - 1)]
    for scope in (GPU, HARD, GPU | HARD):
        g, code, sl = checkers.moves_score(o, mv, out, scope)
        admitted = (c0 == abi.MOVE_NOT_MOVABLE) & (need[cls] > 0) & ((need[cls] & ~scope) == 0)
        np.testing.assert_array_equal(code[~admitted], c0[~admitted])
        np.testing.assert_array_equal(g[~admitted], g0[~admitted])
        assert not (code[admitted] == abi.MOVE_NOT_MOVABLE).any()
        assert admitted.sum() > 0 and (code[admitted] == 0).sum() > 0
        if scope & GPU:
            assert ((sl != 0) == ((code == 0) & ((need[cls] & GPU) != 0))).all()
    # the oracle's state is restored after every scoped call
    g2, c2 = o.moves_score(mv, out)
    np.testing.assert_array_equal(c2, c0)


def test_open_local_and_pinned_classes_stay_not_movable():
    from oracle.binding import Oracle
    from simon_b200 import abi, simulator, synth
    from simon_b200.compiler import compile_cluster
    cluster, apps = synth.make_open_local(n_nodes=120, n_workloads=24, replicas=6, seed_no=6)
    pl = simulator.plan(cluster, apps)
    c = compile_cluster(pl.nodes, pl.pods, pl.ctx, open_local=True, storage_classes=list(cluster.StorageClasss), local_devices=True)
    o = Oracle(c)
    out = o.schedule()[0]
    mv = _moves(out, c, 5000)
    loc = np.asarray(c.storage.class_local, np.uint8)
    cls = c.pods["pod_class"][np.minimum(mv[:, 0], len(out) - 1)]
    placed = (out[np.minimum(mv[:, 0], len(out) - 1)] >= 0) & (mv[:, 0] < len(out))
    for scope in (0, GPU | HARD):
        g, code, _ = checkers.moves_score(o, mv, out, scope, class_local=loc)
        sel = placed & (loc[cls] == 1) & (out[np.minimum(mv[:, 0], len(out) - 1)] != mv[:, 1])
        assert sel.sum() > 0 and (code[sel] == abi.MOVE_NOT_MOVABLE).all()
    # pinned (DaemonSet) classes of a mix cluster
    p, c2, o2, out2 = _state("mix", seed_no=103, n_nodes=95, n_workloads=40, max_replicas=7)
    mv2 = _moves(out2, c2, 20000)
    pinned = _needs(c2)[c2.pods["pod_class"][np.minimum(mv2[:, 0], len(out2) - 1)]] == -1
    g, code, _ = checkers.moves_score(o2, mv2, out2, GPU | HARD)
    g0, c0 = o2.moves_score(mv2, out2)
    assert pinned.sum() > 0
    np.testing.assert_array_equal(code[pinned], c0[pinned])


def _node(name, cores, zone=None, labels=None, gpus=None, taints=None):
    from simon_b200 import synth
    n = synth._node(name, cores, zone or "", "", 100, labels, taints)
    if zone is None:
        del n["metadata"]["labels"]["topology.kubernetes.io/zone"]
    if gpus:
        cnt, per = gpus
        for sect in ("allocatable", "capacity"):
            n["status"][sect]["alibabacloud.com/gpu-count"] = str(cnt)
            n["status"][sect]["alibabacloud.com/gpu-mem"] = f"{cnt * per}Gi"
    return n


def _pod(name, labels=None, node=None, gpu=None, spec_extra=None):
    spec = {"containers": [{"name": "c", "image": "registry.local/x:v1"}]}
    if node:
        spec["nodeName"] = node
    spec.update(spec_extra or {})
    meta = {"name": name, "namespace": "default", "labels": dict(labels or {})}
    if gpu:
        meta["annotations"] = {"alibabacloud.com/gpu-mem": f"{gpu[1]}Gi", "alibabacloud.com/gpu-count": str(gpu[0])}
    return {"apiVersion": "v1", "kind": "Pod", "metadata": meta, "spec": spec}


def _compile(nodes, pods):
    from simon_b200 import simulator
    from simon_b200.compiler import compile_cluster
    from simon_b200.objects import AppResource, ResourceTypes
    cluster = ResourceTypes()
    cluster.Nodes.extend(nodes)
    app = AppResource("app", ResourceTypes())
    app.Resource.Pods.extend(pods)
    pl = simulator.plan(cluster, [app])
    c = compile_cluster(pl.nodes, pl.pods, pl.ctx)
    return c, [x.name for x in pl.pods]


def _gpu_cluster():
    """Nodes: s (64 cores, 4 x 16 GiB), b (4 cores, 2 x 16 GiB), n (no GPU), t (1 x 48 GiB, tainted; only `big` tolerates it).
    g12 (1 GPU, 12 GiB) is pinned to b by a nodeSelector: AllocateGpuId puts it on device 0 (both free, first on ties), so b's
    free device memory is [4, 16] GiB.  The movers have no selector; s, emptier by far, outscores b, so they all run on s, and
    `big` (40 GiB) only fits t."""
    tol = [{"key": "big", "operator": "Exists", "effect": "NoSchedule"}]
    nodes = [_node("s", 64, "z", gpus=(4, 16)), _node("b", 4, "z", gpus=(2, 16)), _node("n", 4, "z"),
             _node("t", 64, "z", gpus=(1, 48), taints=[{"key": "big", "value": "1", "effect": "NoSchedule"}])]
    pods = [_pod("g12", gpu=(1, 12), spec_extra={"nodeSelector": {"kubernetes.io/hostname": "b"}}),
            _pod("m4", gpu=(1, 4)), _pod("m5", gpu=(1, 5)), _pod("d8", gpu=(2, 8)), _pod("d10", gpu=(2, 10)),
            _pod("big", gpu=(1, 40), spec_extra={"tolerations": tol})]
    return _compile(nodes, pods)


def test_gpu_share_known_answers():
    from oracle.binding import Oracle
    from simon_b200 import abi
    c, names = _gpu_cluster()
    o = Oracle(c)
    out = o.schedule()[0]
    S, B, NO, T = (c.node_names.index(x) for x in ("s", "b", "n", "t"))
    at = dict(zip(names, out.tolist()))
    assert at["g12"] == B and at["big"] == T
    assert all(at[m] == S for m in ("m4", "m5", "d8", "d10"))
    used = checkers.gpu_used(o)
    assert used[0, B] == 12 * GI and used[1, B] == 0
    pod = {nm: i for i, nm in enumerate(names)}
    mv = np.array([[pod[m], B] for m in ("m4", "m5", "d8", "d10", "big")] + [[pod["m4"], NO]], np.uint32)
    g0, c0 = o.moves_score(mv, out)
    assert (c0 == abi.MOVE_NOT_MOVABLE).all()                 # without the scope, GPU-share pods are not candidates
    g, code, slots = checkers.moves_score(o, mv, out, GPU)
    assert checkers.moves_score(o, mv, out, HARD)[1].tolist() == c0.tolist()
    want = [
        (0, 1),             # m4, 4 GiB: fits both devices (4, 16 free); the tightest is device 0, exactly full
        (0, 1 << 4),        # m5, 5 GiB: only device 1 holds it
        (0, 2 << 4),        # d8, 2 x 8 GiB: device 0 (4 free) is skipped, device 1 takes both slots
        (1 << SFC_GPU, 0),  # d10, 2 x 10 GiB: device 1 takes one (6 left < 10): fails with 20 GiB free in total
        (1 << SFC_GPU, 0),  # big, 40 GiB: b's total gpu-mem, 32 GiB, is below the request
        (1 << SFC_GPU, 0),  # m4 to a node without GPUs
    ]
    assert list(zip(code.tolist(), slots.tolist())) == want
    # a Python restatement of AllocateGpuId over the oracle's gpu_used gives the same slots
    for (m, (cd, sl)) in zip(mv.tolist(), want):
        assert _allocate(c, used, m[0], m[1]) == sl


def _allocate(c, used, pod, b):
    """AllocateGpuId (cache/gpunodeinfo.go:232-290) restated over the oracle's gpu_used -> 4-bit slots, 0 = none"""
    from simon_b200 import compiler as K
    cls = int(c.pods["pod_class"][pod])
    req, num = int(_class_word(c, K.SCW_GPU_MEM)[cls]), int(_class_word(c, K.SCW_GPU_COUNT)[cls])
    nd = int(c.snap["gpu_count"][b])
    avail = [int(c.snap["gpu_dev_mem"][b]) - int(used[d, b]) for d in range(nd)]
    if int(c.snap["gpu_total_mem"][b]) < req or nd == 0 or req <= 0 or num <= 0:
        return 0
    if num == 1:
        fits = [(a, d) for d, a in enumerate(avail) if a >= req]
        return 0 if not fits else 1 << (4 * min(fits)[1])
    out, got, d = [0] * 8, 0, 0
    while d < nd and got < num:
        if avail[d] >= req:
            avail[d] -= req
            out[d] += 1
            got += 1
        else:
            d += 1
    return sum(min(x, 15) << (4 * q) for q, x in enumerate(out)) if got == num else 0


def _spread_cluster():
    """Zones A (a1 with 64 cores, a2), B (b1), C (c1, c2), and n0 without the zone label; x1 (zone D) is outside the class's
    node selection (pool=other).  Pre-bound pods labelled app=s: one on b1, one on c1 and one on c2, and one on x1.  Then p
    (app=s, zone spread maxSkew 1 DoNotSchedule, nodeSelector pool=main) is scheduled: the registered zones are A, B and C (D has
    no node that passes p's selection, n0 has no zone), the counts 0, 1, 2 (x1's pod sits in the unregistered D), the minimum 0,
    so only A passes (0 + 1 - 0 = 1); a1, emptier by far, wins.  After it: A = 1 (p), B = 1, C = 2."""
    main = {"pool": "main"}
    nodes = [_node("a1", 64, "A", main), _node("a2", 4, "A", main), _node("b1", 4, "B", main), _node("c1", 4, "C", main),
             _node("c2", 4, "C", main), _node("n0", 4, None, main), _node("x1", 4, "D", {"pool": "other"})]
    s = {"app": "s"}
    tsc = {"topologySpreadConstraints": [{"maxSkew": 1, "topologyKey": "topology.kubernetes.io/zone",
                                          "whenUnsatisfiable": "DoNotSchedule", "labelSelector": {"matchLabels": s}}],
           "nodeSelector": main}
    pods = [_pod("r-b1", s, "b1"), _pod("r-c1", s, "c1"), _pod("r-c2", s, "c2"), _pod("r-x1", s, "x1"), _pod("p", s, spec_extra=tsc)]
    return _compile(nodes, pods)


def test_hard_spread_known_answers():
    from oracle.binding import Oracle
    from simon_b200 import abi
    c, names = _spread_cluster()
    o = Oracle(c)
    out = o.schedule()[0]
    A1, A2, B1, C1, N0, X1 = (c.node_names.index(x) for x in ("a1", "a2", "b1", "c1", "n0", "x1"))
    p = names.index("p")
    assert out[p] == A1
    mv = np.array([[p, B1], [p, A2], [p, N0], [p, C1], [p, X1]], np.uint32)
    assert (o.moves_score(mv, out)[1] == abi.MOVE_NOT_MOVABLE).all()
    g, code, _ = checkers.moves_score(o, mv, out, HARD)
    assert checkers.moves_score(o, mv, out, GPU)[1].tolist() == [abi.MOVE_NOT_MOVABLE] * 5
    assert code.tolist() == [
        1 << SFC_PTS_SKEW,      # b1: p leaves A, so A = 0 and the minimum drops to 0: 1 + 1 - 0 > 1 (without the removal: 1 + 1 - 1 = 1)
        0,                          # a2: A's count without p is 0: 0 + 1 - 0 = 1
        1 << SFC_PTS_MISSING,   # n0 has no zone label
        1 << SFC_PTS_SKEW,      # c1: 2 + 1 - 0 > 1
        1 << SFC_STATIC,        # x1 fails p's nodeSelector first
    ]


# object-level replay: every other running pod bound by spec.nodeName at its placement, the moved pod pending as the last pod
@pytest.mark.parametrize("kind,kw,seed", [
    ("mix", dict(seed_no=103, n_nodes=95, n_workloads=40, max_replicas=7), 1),
    ("mix", dict(seed_no=215, n_nodes=45, n_workloads=30, max_replicas=9), 2),
    ("c3", dict(n_nodes=200, n_workloads=60, replicas=8, n_apps=2, seed_no=21, gpu_pct=25), 3),
])
def test_scoped_moves_replay_on_objects(kind, kw, seed):
    import copy
    from oracle.binding import Oracle
    from simon_b200 import abi
    from simon_b200.compiler import compile_cluster
    p, c, o, out = _state(kind, **kw)
    need = _needs(c)
    mv = _moves(out, c, 20000, seed=seed)
    g, code, _ = checkers.moves_score(o, mv, out, HARD)
    cls = c.pods["pod_class"][np.minimum(mv[:, 0], len(out) - 1)]
    pre = np.array([bool(r.node_name) for r in p.pods])
    cand = np.nonzero((need[cls] == HARD) & (code < (1 << 24)) & ~pre[np.minimum(mv[:, 0], len(out) - 1)])[0]
    assert len(cand) > 20 and (code[cand] == 0).sum() > 5 and (code[cand] & (3 << SFC_PTS_MISSING)).sum() > 0
    pick = np.random.RandomState(seed).choice(cand, min(len(cand), 100), replace=False)
    for m in pick:
        pod, b = int(mv[m, 0]), int(mv[m, 1])
        recs = []
        for i, r in enumerate(p.pods):
            if i != pod and out[i] >= 0:
                r2 = copy.copy(r)
                r2.node_name = c.node_names[out[i]]
                recs.append(r2)
        recs.append(copy.copy(p.pods[pod]))
        c2 = compile_cluster(p.nodes, recs, p.ctx)
        o2 = Oracle(c2)
        o2.schedule()
        stage = int(o2.last_detail()[0][c2.node_names.index(c.node_names[b])])
        want = _stage_of(int(code[m]))
        assert (1 <= stage <= 4) if want < 0 else stage == want, (m, int(code[m]), stage)
        o2.close()


def _stage_of(code):
    """the oracle's per-node stage number (simon_oracle.c ST_FILTER) of a move code"""
    if code == 0:
        return 0
    if code & 1:
        return -1                   # static: stages 1..4, checked below
    for bits, st in ((1 << 1, 5), (0x3ffc, 6), (3 << SFC_PTS_MISSING, 14), (7 << 16, 15), (1 << SFC_GPU, 17)):
        if code & bits:
            return st
    raise AssertionError(code)


# ---------------------------------------------------------------------------------------------------------------- GPU ----

def _engine_vs_checker(c, o, out, mv, scope, class_local=None, static_cache=True):
    from simon_b200 import moves as M
    from simon_b200.engine import Engine
    gain, code, slots = checkers.moves_score(o, mv, out, scope, class_local=class_local)
    with Engine(c, device=0, static_cache=static_cache) as eng:
        np.testing.assert_array_equal(eng.schedule()[0], out)
        eng.moves_set_scope(scope)
        eng.moves_upload(mv, 0)
        r = eng.moves_run(k=32, want_arrays=True, want_per_pod=True, want_gpu_slots=bool(scope & GPU))
        half = len(mv) // 2
        eng.moves_upload(mv[half:], half)
        r2 = eng.moves_run(k=8, want_arrays=False)
    bad = np.nonzero(r["code"] != code)[0]
    assert len(bad) == 0, f"codes differ at moves {bad[:5]}: gpu {r['code'][bad[:5]]} checker {code[bad[:5]]}"
    np.testing.assert_array_equal(r["gain"], gain)
    if scope & GPU:
        np.testing.assert_array_equal(r["gpu_slots"], slots)
    feas = np.nonzero(code == 0)[0]
    keys = [M.pack_key(int(gain[m]), int(m)) for m in feas]
    assert r["best_key"] == (max(keys) if keys else 0) and r["n_feasible"] == len(feas)
    assert r["topk"] == sorted(((int(m), int(gain[m])) for m in feas), key=lambda mg: (-mg[1], mg[0]))[:32]
    feas2 = [m for m in feas if m >= half]
    assert r2["topk"] == sorted(((int(m), int(gain[m])) for m in feas2), key=lambda mg: (-mg[1], mg[0]))[:8]
    assert r2["best_key"] == (max(M.pack_key(int(gain[m]), int(m)) for m in feas2) if feas2 else 0)
    want = np.zeros(len(out), np.uint64)
    for m in feas:
        k = M.pack_key(int(gain[m]), int(m))
        if k > int(want[mv[m, 0]]):
            want[mv[m, 0]] = k
    np.testing.assert_array_equal(r["best_per_pod"][:len(out)], want)
    return code


@pytest.mark.gpu
@pytest.mark.parametrize("kind,kw,n", CASES + GPU_CASES)
def test_scoped_moves_gpu_match_checker(kind, kw, n):
    p, c, o, out = _state(kind, **kw)
    mv = _moves(out, c, n)
    for scope in (GPU, HARD, GPU | HARD):
        _engine_vs_checker(c, o, out, mv, scope)


@pytest.mark.gpu
def test_scoped_moves_gpu_known_answers():
    from oracle.binding import Oracle
    for c, names in (_gpu_cluster(), _spread_cluster()):
        o = Oracle(c)
        out = o.schedule()[0]
        mv = np.array([[i, b] for i in range(len(out)) for b in range(c.n_nodes)], np.uint32)
        _engine_vs_checker(c, o, out, mv, GPU | HARD)


@pytest.mark.gpu
def test_scoped_moves_gpu_open_local_stay_not_movable():
    from simon_b200 import abi, simulator, synth
    from simon_b200.compiler import compile_cluster
    cluster, apps = synth.make_open_local(n_nodes=120, n_workloads=24, replicas=6, seed_no=6)
    pl = simulator.plan(cluster, apps)
    c = compile_cluster(pl.nodes, pl.pods, pl.ctx, open_local=True, storage_classes=list(cluster.StorageClasss), local_devices=True)
    from simon_b200.engine import Engine
    loc = np.asarray(c.storage.class_local, np.uint8)
    with Engine(c, device=0) as eng:
        out = eng.schedule()[0]
        mv = _moves(out, c, 5000)
        eng.moves_set_scope(GPU | HARD)
        eng.moves_upload(mv, 0)
        r = eng.moves_run(k=0, want_arrays=True)
    pod = np.minimum(mv[:, 0], len(out) - 1)
    sel = (loc[c.pods["pod_class"][pod]] == 1) & (out[pod] >= 0) & (out[pod] != mv[:, 1].astype(np.int64))
    assert sel.sum() > 0 and (r["code"][sel] == abi.MOVE_NOT_MOVABLE).all()


@pytest.mark.gpu
def test_unscoped_run_after_scoped_and_placement_after_reset():
    from simon_b200.engine import Engine
    kind, kw, n = GPU_CASES[0]
    p, c, o, out = _state(kind, **kw)
    mv = _moves(out, c, n)
    g0, c0 = o.moves_score(mv, out)
    with Engine(c, device=0) as eng:
        np.testing.assert_array_equal(eng.schedule()[0], out)
        eng.moves_upload(mv, 0)
        eng.moves_set_scope(GPU | HARD)
        rs = eng.moves_run(k=4)
        eng.moves_set_scope(0)
        r = eng.moves_run(k=4)
        eng.reset()
        np.testing.assert_array_equal(eng.schedule()[0], out)
    assert rs["n_feasible"] > r["n_feasible"]
    np.testing.assert_array_equal(r["code"], c0)
    np.testing.assert_array_equal(r["gain"], g0)


@pytest.mark.gpu
def test_scope_abi_refusals():
    from simon_b200.engine import Engine, lib
    c, names = _gpu_cluster()
    m4, b = names.index("m4"), c.node_names.index("b")
    with Engine(c, device=0) as eng:
        eng.schedule()
        with pytest.raises(RuntimeError, match="error -1"):
            eng.moves_set_scope(4)
        eng.moves_upload(np.array([[m4, b]], np.uint32), 0)
        eng.moves_run(k=1)
        with pytest.raises(RuntimeError, match="error -3"):
            eng.moves_run(k=1, want_gpu_slots=True)             # the run's scope lacked GPU share
        eng.moves_set_scope(GPU)
        r = eng.moves_run(k=1, want_gpu_slots=True)
        assert r["code"].tolist() == [0] and r["gpu_slots"].tolist() == [1]           # m4 to b: device 0
        eng.moves_upload(np.array([[m4, b]], np.uint32), 0)
        slots = np.zeros(1, np.uint32)
        assert lib().simon_moves_gpu_slots_download(eng.h, 0, 1, slots.ctypes.data) == -3       # no run since the upload
