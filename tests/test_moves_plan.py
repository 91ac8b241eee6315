"""Migration plans (simon_moves_plan, rebalance.py): a sequence of applied moves, each chosen on the state the earlier ones leave.
CPU: the plan checker (tests/checkers.c) against a plan made by rebuilding the oracle from scratch before every step, and
the host-side helpers (candidate lists, MigrationPlan formatting).  GPU: the engine's plans against the checker, step by step and in
their end state, plus the live state left untouched, an independent rebuild of the end state, refusals and the session entry point."""
import copy

import numpy as np
import pytest

import checkers
from util import make_case

GPU, HARD = 1, 2
NO_MOVE, MAX_MOVES = 1, 2


def _oracle_state(c):
    from oracle.binding import Oracle
    o = Oracle(c)
    out = o.schedule()[0]
    return o, out


def _sampled(out, c, n, seed=11):
    from simon_b200 import moves as M
    return M.sample_moves(len(out), c.n_nodes, n, seed=seed, placement=out)


def _checker(c, mv, max_moves, min_gain=1, scope=0, class_local=None):
    o, out = _oracle_state(c)
    res = checkers.plan(o, mv, out, o.gpu_slot_words(), max_moves, min_gain, scope, class_local=class_local)
    o.close()
    res["live"] = out
    return res


# ---------------------------------------------------------------------------------------------------------------- CPU ----

def _rebuild_plan(p, c, out, mv, max_moves, min_gain, scope):
    """The same plan by a different mechanism: before every step the oracle is rebuilt from scratch with every running pod pre-bound
    at its current node (as synth.make_c5 builds a live snapshot), and the best qualifying move of the scoped scoring is taken."""
    from oracle.binding import Oracle
    from simon_b200.compiler import compile_cluster
    placement = np.array(out, np.int64)
    moved, steps = set(), []
    while len(steps) < max_moves:
        keep = np.nonzero(placement >= 0)[0]
        recs = []
        for i in keep.tolist():
            r = copy.copy(p.pods[i])
            r.node_name = c.node_names[placement[i]]
            recs.append(r)
        c2 = compile_cluster(p.nodes, recs, p.ctx)
        assert list(c2.node_names) == list(c.node_names)
        o2 = Oracle(c2)
        out2 = o2.schedule()[0]
        np.testing.assert_array_equal(out2, placement[keep])
        pos = np.full(len(placement), -1, np.int64)
        pos[keep] = np.arange(len(keep))
        sel = np.nonzero(pos[mv[:, 0]] >= 0)[0]
        mv2 = np.stack([pos[mv[sel, 0]], mv[sel, 1]], 1).astype(np.uint32)
        gain, code, _ = checkers.moves_score(o2, mv2, out2, scope)
        o2.close()
        ok = (code == 0) & np.array([int(mv[m, 0]) not in moved for m in sel], bool)
        if not ok.any():
            return steps, NO_MOVE
        g = np.where(ok, gain, -10 ** 6)
        j = int(np.argmax(g))               # first index of the maximum: the lowest move index among equal gains
        if g[j] < min_gain:
            return steps, NO_MOVE
        m = int(sel[j])
        pod, b = int(mv[m, 0]), int(mv[m, 1])
        steps.append((m, pod, int(placement[pod]), b, int(gain[j]), 0))
        placement[pod] = b
        moved.add(pod)
    return steps, MAX_MOVES


def _limits_case(name):
    from test_engine_limits import BUILDERS, compiled
    return compiled(*BUILDERS[name]())


REBUILD_CASES = [
    ("mix", lambda: make_case("mix", seed_no=103, n_nodes=95, n_workloads=40, max_replicas=7), 0, 6, 1),
    ("mix-2", lambda: make_case("mix", seed_no=215, n_nodes=45, n_workloads=30, max_replicas=9), 0, 40, 1),
    ("ports", lambda: _limits_case("entries32"), 0, 5, 1),
    ("scalars", lambda: _limits_case("scalars8"), 0, 5, 1),
    ("hard-spread", lambda: make_case("c3", n_nodes=120, n_workloads=30, replicas=6, n_apps=2, seed_no=21, gpu_pct=0), HARD, 6, 1),
    ("anti-affinity", lambda: make_case("mix", seed_no=104, n_nodes=60, n_workloads=30, max_replicas=6), HARD, 6, 2),
]


@pytest.mark.parametrize("name,build,scope,max_moves,min_gain", REBUILD_CASES, ids=[c[0] for c in REBUILD_CASES])
def test_checker_equals_rebuild_from_scratch(name, build, scope, max_moves, min_gain):
    from simon_b200 import rebalance
    from simon_b200.compiler import SCW_GPU_MEM
    p, c = build()
    o, out = _oracle_state(c)
    o.close()
    mv = rebalance.candidates(c, out)
    gpu_cls = np.array([int(c.pods["class_blob"][int(c.pods["class_off"][k]) + SCW_GPU_MEM]) > 0
                        for k in range(len(c.pods["class_off"]) - 1)])
    mv = mv[~gpu_cls[c.pods["pod_class"][mv[:, 0]]]]          # pre-bound GPU-share pods hold no device memory: leave them out
    res = _checker(c, mv, max_moves, min_gain, scope)
    want, stop = _rebuild_plan(p, c, out, mv, max_moves, min_gain, scope)
    assert len(want) > 0, name
    assert [tuple(int(x) for x in s) for s in res["steps"]] == want
    assert res["stop_reason"] == stop


def _tiny_compiled():
    from simon_b200 import simulator, synth
    from simon_b200.compiler import compile_cluster
    cluster, apps = synth.make_mix(seed_no=103, n_nodes=12, n_workloads=6, max_replicas=3)
    pl = simulator.plan(cluster, apps)
    return compile_cluster(pl.nodes, pl.pods, pl.ctx)


def test_candidates_order_and_cap():
    from simon_b200 import rebalance
    from simon_b200.scaledown import NodeOrder
    c = _tiny_compiled()
    o, out = _oracle_state(c)
    o.close()
    order = NodeOrder(c).remaining([]).tolist()
    mv = rebalance.candidates(c, out)
    want = [(q, g) for q in range(len(out)) if out[q] >= 0 for g in order if g != out[q]]
    assert [tuple(x) for x in mv.tolist()] == want
    src, tgt = [order[0], order[3]], [order[5], order[1], order[0]]
    mv = rebalance.candidates(c, out, sources=src, targets=tgt)
    tg = [g for g in order if g in tgt]
    want = [(q, g) for q in range(len(out)) if out[q] in src for g in tg if g != out[q]]
    assert [tuple(x) for x in mv.tolist()] == want and len(want) > 0
    with pytest.raises(ValueError, match=f"{len(want)} candidate moves exceed the cap of {len(want) - 1}"):
        rebalance.candidates(c, out, sources=src, targets=tgt, cap=len(want) - 1)
    assert len(rebalance.candidates(c, out, sources=src, targets=tgt, cap=len(want))) == len(want)


def test_migration_plan_from_raw_arrays():
    from simon_b200 import abi, rebalance
    from simon_b200.compiler import SCW_GPU_MEM
    c = _tiny_compiled()
    o, out = _oracle_state(c)
    o.close()
    cls = c.pods["pod_class"]
    gpu = np.array([int(c.pods["class_blob"][int(c.pods["class_off"][k]) + SCW_GPU_MEM]) > 0 for k in range(len(c.pods["class_off"]) - 1)])
    placed = np.nonzero(out >= 0)[0]
    q0 = int(placed[0])
    qg = [int(q) for q in placed if gpu[cls[q]]]
    q1 = qg[0] if qg else int(placed[1])
    steps = np.zeros(2, abi.PLAN_STEP_DTYPE)
    steps[0] = (7, q0, out[q0], (out[q0] + 1) % c.n_nodes, 12, 0)
    steps[1] = (3, q1, out[q1], (out[q1] + 2) % c.n_nodes, 5, (2 << 4) | (1 << 12))
    end = out.copy()
    end[q0], end[q1] = steps[0]["to"], steps[1]["to"]
    mp = rebalance.from_raw(c, steps, abi.PLAN_STOP_MAX_MOVES, 3, end, 1.5)
    assert mp.StopReason == "MaxMoves" and mp.Excluded == 3 and mp.KernelMs == 1.5
    m0, m1 = mp.Migrations
    assert m0.Pod is c.pod_recs[q0] and m1.Pod is c.pod_recs[q1]
    assert (m0.From, m0.To, m0.Gain, m0.GpuIndex) == (c.node_names[out[q0]], c.node_names[(out[q0] + 1) % c.n_nodes], 12, None)
    assert m1.GpuIndex == ("1-1-3" if gpu[cls[q1]] else None) and m1.Gain == 5
    assert sorted(sum(mp.NodePods.values(), [])) == sorted(c.pod_recs[q].name for q in placed)
    assert c.pod_recs[q0].name in mp.NodePods[m0.To]
    assert rebalance.from_raw(c, steps[:0], abi.PLAN_STOP_NO_MOVE, 0, out).StopReason == "NoMove"


def test_plan_session_refusal_without_a_device():
    from simon_b200 import simulator
    sim = simulator.NewSimulator()
    with pytest.raises(RuntimeError, match="RunCluster"):
        sim.PlanMigrations()


# ---------------------------------------------------------------------------------------------------------------- GPU ----

def _steps(r):
    s = r["steps"]
    return np.stack([s["move"], s["pod"], s["from"], s["to"], s["gain"], s["gpu_slots"]], 1).astype(np.int64) if len(s) else np.zeros((0, 6), np.int64)


def _engine_vs_checker(c, mv, max_moves, min_gain=1, scope=0, class_local=None, rebuild=False, static_cache=True):
    """The engine's plan equals the checker's, step by step and in the end state; the live state is untouched; with rebuild, the end
    placement resumed on a fresh context gives the plan's end state, and after NO_MOVE no unmoved pod has a qualifying move there."""
    from simon_b200.engine import Engine
    if class_local is None:
        ref = _checker(c, mv, max_moves, min_gain, scope)
    else:
        # the C oracle has no Open-Local: its state is the engine's placement, every placed pod pre-bound where the engine put it
        with Engine(c, device=0, static_cache=static_cache) as eng:
            live = eng.schedule()[0]
            assert not eng.gpu_slot_words().any()
        cf = copy.copy(c)
        cf.pods = dict(c.pods)
        cf.pods["pod_fixed_node"] = np.where(live >= 0, live, -2).astype(np.int32)
        from oracle.binding import Oracle
        o = Oracle(cf)
        o.schedule()
        ref = checkers.plan(o, mv, live, np.zeros(len(live), np.uint32), max_moves, min_gain, scope, class_local=class_local)
        o.close()
        ref["live"] = live
    with Engine(c, device=0, static_cache=static_cache) as eng:
        out = eng.schedule()[0]
        np.testing.assert_array_equal(out, ref["live"])
        eng.moves_set_scope(scope)
        eng.moves_upload(mv, 0)
        before = (eng.state(), eng.state_ext(), eng.gpu_slot_words(), eng.moves_run(k=8, want_arrays=True))
        r = eng.moves_plan(max_moves, min_gain)
        pl, sl = eng.moves_plan_download()
        st, ext = eng.moves_plan_state()
        after = (eng.state(), eng.state_ext(), eng.gpu_slot_words(), eng.moves_run(k=8, want_arrays=True))
    got = _steps(r)
    want = ref["steps"]
    n = min(len(got), len(want))
    bad = [i for i in range(n) if not np.array_equal(got[i], want[i])]
    assert not bad and len(got) == len(want), f"steps differ at {bad[:3]}: gpu {got[bad[:3]] if bad else got[n:n + 2]} checker {want[bad[:3]] if bad else want[n:n + 2]}"
    assert r["stop_reason"] == ref["stop_reason"] and r["excluded"] == ref["excluded"]
    np.testing.assert_array_equal(pl, ref["placement"])
    np.testing.assert_array_equal(sl, ref["slots"])
    for k in ref["state"]:
        np.testing.assert_array_equal(st[k], ref["state"][k], err_msg=k)
    for k in ref["state_ext"]:
        np.testing.assert_array_equal(ext[k], ref["state_ext"][k], err_msg=k)
    for x, y in zip(before[:2], after[:2]):
        for k in x:
            np.testing.assert_array_equal(x[k], y[k], err_msg=k)
    np.testing.assert_array_equal(before[2], after[2])
    for k in ("gain", "code"):
        np.testing.assert_array_equal(before[3][k], after[3][k])
    assert before[3]["topk"] == after[3]["topk"] and before[3]["best_key"] == after[3]["best_key"]
    if rebuild:
        _independent_rebuild(c, r, pl, st, ext, mv, min_gain, scope, static_cache)
    return r


def _independent_rebuild(c, r, pl, st, ext, mv, min_gain, scope, static_cache=True):
    from simon_b200.engine import Engine
    c2 = copy.copy(c)
    c2.pods = dict(c.pods)
    fixed = np.array(c.pods["pod_fixed_node"], np.int32)
    moved = _steps(r)[:, 1]
    fixed[moved] = np.where(fixed[moved] >= 0, pl[moved], fixed[moved])     # a moved pre-bound pod is bound to its new node
    c2.pods["pod_fixed_node"] = fixed
    with Engine(c2, device=0, static_cache=static_cache) as eng:
        eng.schedule_resume(pl)
        st2, ext2 = eng.state(), eng.state_ext()
        for k in st:
            np.testing.assert_array_equal(st2[k], st[k], err_msg=f"resume {k}")
        for k in ext:
            np.testing.assert_array_equal(ext2[k], ext[k], err_msg=f"resume {k}")
        if r["stop_reason"] == NO_MOVE:
            eng.moves_set_scope(scope)
            eng.moves_upload(mv, 0)
            rr = eng.moves_run(k=0, want_arrays=True)
            unmoved = ~np.isin(mv[:, 0], moved)
            assert not ((rr["code"] == 0) & (rr["gain"] >= min_gain) & unmoved).any()


def _moves_cases():
    return [
        ("mix", dict(seed_no=103, n_nodes=95, n_workloads=40, max_replicas=7), 30000, 0),
        ("mix", dict(seed_no=215, n_nodes=45, n_workloads=30, max_replicas=9), 20000, 0),
        ("c3", dict(n_nodes=1500, n_workloads=200, replicas=20, n_apps=4, seed_no=5), 200000, 0),
        ("c2", dict(n_nodes=300, n_workloads=30, replicas=30, seed_no=2), 50000, 0),
        ("c3", dict(n_nodes=400, n_workloads=80, replicas=10, n_apps=2, seed_no=21, gpu_pct=25), 40000, GPU),
        ("c3", dict(n_nodes=400, n_workloads=80, replicas=10, n_apps=2, seed_no=21, gpu_pct=25), 40000, HARD),
        ("c3", dict(n_nodes=400, n_workloads=80, replicas=10, n_apps=2, seed_no=21, gpu_pct=25), 40000, GPU | HARD),
    ]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,kw,n,scope", _moves_cases())
def test_plan_gpu_matches_checker(kind, kw, n, scope):
    from simon_b200 import rebalance
    p, c = make_case(kind, **kw)
    o, out = _oracle_state(c)
    o.close()
    mv = _sampled(out, c, n)
    r = _engine_vs_checker(c, mv, 25, 1, scope, rebuild=not (scope & GPU))
    assert len(r["steps"]) > 0
    if scope & GPU:
        assert (r["steps"]["gpu_slots"] != 0).any()
    # both stop reasons: a long plan on the small clusters ends with NO_MOVE; min_gain 200 plans nothing
    if kind == "mix":
        r2 = _engine_vs_checker(c, rebalance.candidates(c, out), 10 ** 6, 1, scope, rebuild=True)
        assert r2["stop_reason"] == NO_MOVE and len(r2["steps"]) > 0
    r3 = _engine_vs_checker(c, mv, 5, 200, scope)
    assert len(r3["steps"]) == 0 and r3["stop_reason"] == NO_MOVE


@pytest.mark.gpu
def test_plan_gpu_live_snapshot_c5():
    from simon_b200 import synth
    p, c = make_case("c3", n_nodes=500, n_workloads=50, replicas=10, n_apps=2, seed_no=3)
    live = synth.make_c5(c, 5000)
    o, out = _oracle_state(live)
    o.close()
    mv = _sampled(out, live, 300000)
    r = _engine_vs_checker(live, mv, 30, 1, 0, rebuild=True)
    assert r["stop_reason"] == MAX_MOVES and len(r["steps"]) == 30


@pytest.mark.gpu
def test_plan_gpu_20000_nodes():
    p, c = make_case("c3", n_nodes=20000, n_workloads=60, replicas=10, n_apps=2, seed_no=9)
    o, out = _oracle_state(c)
    o.close()
    mv = _sampled(out, c, 200000)
    r = _engine_vs_checker(c, mv, 12, 1, HARD, rebuild=True)
    assert len(r["steps"]) == 12


@pytest.mark.gpu
def test_plan_gpu_daemonsets_and_open_local_never_move():
    from simon_b200 import rebalance, simulator, synth
    from simon_b200.compiler import SCW_FLAGS, compile_cluster, CLS_PINNED
    cluster, apps = synth.make_open_local(n_nodes=120, n_workloads=24, replicas=6, seed_no=6)
    pl = simulator.plan(cluster, apps)
    c = compile_cluster(pl.nodes, pl.pods, pl.ctx, open_local=True, storage_classes=list(cluster.StorageClasss), local_devices=True)
    loc = np.asarray(c.storage.class_local, np.uint8)
    o, out = _oracle_state(c)
    o.close()
    mv = rebalance.candidates(c, out)
    r = _engine_vs_checker(c, mv, 40, 1, GPU | HARD, class_local=loc)
    cls = c.pods["pod_class"][r["steps"]["pod"]]
    assert len(cls) > 0 and not loc[cls].any()
    p2, c2 = make_case("mix", seed_no=103, n_nodes=95, n_workloads=40, max_replicas=7)
    o, out2 = _oracle_state(c2)
    o.close()
    flags = np.array([int(c2.pods["class_blob"][int(c2.pods["class_off"][k]) + SCW_FLAGS]) for k in range(len(c2.pods["class_off"]) - 1)])
    pinned = (flags & CLS_PINNED) != 0
    assert pinned[c2.pods["pod_class"][out2 >= 0]].any()
    r2 = _engine_vs_checker(c2, rebalance.candidates(c2, out2), 60, 1, GPU | HARD)
    assert len(r2["steps"]) > 0 and not pinned[c2.pods["pod_class"][r2["steps"]["pod"]]].any()


@pytest.mark.gpu
@pytest.mark.parametrize("name,scope", [("entries32", 0), ("commit_list_long", HARD), ("scalars8", 0), ("gpu8", GPU)])
def test_plan_gpu_engine_limits(name, scope):
    from simon_b200 import rebalance
    p, c = _limits_case(name)
    o, out = _oracle_state(c)
    o.close()
    if name == "commit_list_long":
        # the scheduler spreads this builder evenly (every feasible move gains 0): every other pod is pre-bound onto nodes 0-2
        # instead, so that moves gain and apply the long commit list
        q = np.arange(len(out))
        c = copy.copy(c)
        c.pods = dict(c.pods)
        c.pods["pod_fixed_node"] = np.where(out >= 0, np.where(q % 2 == 0, q % 3, out), -2).astype(np.int32)
        o, out = _oracle_state(c)
        o.close()
    mv = rebalance.candidates(c, out)
    if len(mv) > 400000:
        mv = mv[np.random.RandomState(3).choice(len(mv), 400000, replace=False)]
        mv = mv[np.lexsort((mv[:, 1], mv[:, 0]))]
    r = _engine_vs_checker(c, mv, 20, 1, scope, rebuild=not (scope & GPU))
    if name == "gpu8":
        assert r["excluded"] > 0                # the pod with more than 15 slots on one device stays where it is
    else:
        assert len(r["steps"]) > 0


@pytest.mark.gpu
def test_plan_keeps_drain_downloads_and_refusals():
    from simon_b200 import scaledown
    from simon_b200.engine import Engine, lib
    from simon_b200 import abi
    import ctypes as C
    p, c = make_case("mix", seed_no=215, n_nodes=45, n_workloads=30, max_replicas=9)
    o, out = _oracle_state(c)
    o.close()
    mv = _sampled(out, c, 5000)
    steps = np.zeros(4, abi.PLAN_STEP_DTYPE)
    res = abi.SimonMovesPlanResult()
    plan = lambda mx, mg: lib().simon_moves_plan(eng.h, mx, mg, steps.ctypes.data, C.byref(res))
    with Engine(c, device=0) as eng:
        eng.moves_upload(mv, 0)
        assert plan(2, 1) == -3 and "no placement" in lib().simon_last_error(eng.h).decode()       # nothing placed yet
        pl = np.zeros(max(len(out), 1), np.int32)
        assert lib().simon_moves_plan_download(eng.h, pl.ctypes.data, None) == -3                   # no plan yet
        eng.schedule()
        remain = scaledown.NodeOrder(c).remaining([0, 1])
        d0 = eng.drain_run(out, [remain], detail=True)[0]
        assert plan(0, 1) == -1 and "max_moves" in lib().simon_last_error(eng.h).decode()
        assert plan(2, 0) == -1 and plan(2, 201) == -1 and "min_gain" in lib().simon_last_error(eng.h).decode()
        eng.moves_upload(mv, 5)
        assert plan(2, 1) == -1 and "move_base" in lib().simon_last_error(eng.h).decode()
        eng.moves_upload(mv, 0)
        r = eng.moves_plan(3, 1)
        assert len(r["steps"]) == 3 and r["stop_reason"] == MAX_MOVES
        slots = np.zeros(1, np.uint32)
        assert lib().simon_moves_gpu_slots_download(eng.h, 0, 1, slots.ctypes.data) == -3
        # the drain's device outputs are still served after the plan
        ev =np.zeros(max(d0["n_evicted"], 1), np.uint32)
        node = np.zeros(max(d0["n_evicted"], 1), np.int32)
        assert lib().simon_drain_download(eng.h, 0, ev.ctypes.data, node.ctypes.data, None, None, None, None, None) == 0
        np.testing.assert_array_equal(ev[:d0["n_evicted"]], d0["evicted"])
        np.testing.assert_array_equal(node[:d0["n_evicted"]], d0["node"])
        eng.reset()
        assert plan(2, 1) == -3
    with Engine(c, device=0) as eng:
        eng.schedule()
        assert plan(2, 1) == -3 and "simon_moves_upload" in lib().simon_last_error(eng.h).decode()


@pytest.mark.gpu
def test_session_plan_migrations():
    from simon_b200 import rebalance, simulator, synth
    from simon_b200.engine import Engine
    cluster, apps = synth.make_c3(n_nodes=200, n_workloads=40, replicas=6, n_apps=2, seed_no=4)
    names = None
    with simulator.NewSimulator() as sim:
        sim.RunCluster(simulator.PrepareCluster(cluster))
        sim.ScheduleApp(apps[0])
        eng, c = sim._live()
        placements = sim.placements.copy()
        busy = np.argsort(-np.bincount(placements[placements >= 0], minlength=c.n_nodes), kind="stable")[:20]
        src = [c.node_names[g] for g in busy]
        mp = sim.PlanMigrations(sources=src, max_moves=15)
        assert len(mp.Migrations) > 0 and all(m.From in src for m in mp.Migrations)
        with Engine(c, device=0) as e2:
            e2.schedule_resume(placements)
            mv =rebalance.candidates(c, placements, [int(g) for g in busy])
            e2.moves_upload(mv, 0)
            r = e2.moves_plan(15, 1)
        assert [(m.Pod.name, m.From, m.To, m.Gain) for m in mp.Migrations] == \
            [(c.pod_recs[int(s["pod"])].name, c.node_names[int(s["from"])], c.node_names[int(s["to"])], int(s["gain"])) for s in r["steps"]]
        np.testing.assert_array_equal(sim.placements, placements)
        res = sim.ScheduleApp(apps[1])
        names = [(u.Pod.name if hasattr(u, "Pod") else str(u)) for u in res.UnscheduledPods], sim.placements.copy()
    with simulator.NewSimulator() as sim2:
        sim2.RunCluster(simulator.PrepareCluster(cluster))
        sim2.ScheduleApp(apps[0])
        res2 = sim2.ScheduleApp(apps[1])
        names2 = [(u.Pod.name if hasattr(u, "Pod") else str(u)) for u in res2.UnscheduledPods], sim2.placements.copy()
    assert names[0] == names2[0]
    np.testing.assert_array_equal(names[1], names2[1])
