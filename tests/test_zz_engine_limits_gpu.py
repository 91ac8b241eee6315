"""The device at the engine's fixed limits: every builder of test_engine_limits.py against the C oracle.

Per builder: a full single run at the engine's own geometry and with the large-cluster variant (node, recorded winning score,
failure records, state(), state_ext(), GPU-share slot words, the kernel that ran), a scenario batch on four node lists,
simon_schedule_resume from half of the pods, drains against the drain checker, and move scoring (sampled and hand-picked moves)
against the scoped checker, with the scope off and, where the builder has GPU-share or hard-spread classes, on.  Past the
limits the upload refuses a class of 33 entries, 9 hard or 9 soft spread constraints.
"""
import functools

import numpy as np
import pytest

from test_engine_limits import BUILDERS, compiled, entries32

GPU, HARD = 1, 2
SCOPED = {"soft_taints256", "topo8", "gpu8", "entries32", "commit_list_long", "big_record"}


@functools.lru_cache(maxsize=None)
def case(name):
    return compiled(*BUILDERS[name]())


@functools.lru_cache(maxsize=None)
def oracle_full(name):
    from oracle.binding import Oracle
    _p, c = case(name)
    o = Oracle(c)
    res = o.schedule() + (o.state(), o.state_ext(), o.gpu_slot_words())
    o.close()
    return res


def _engine(c, **kw):
    from simon_b200.engine import Engine
    return Engine(c, device=0, **kw)


def _assert_run(name, eng, out, score, fc, fp, what):
    ref, rscore, rfc, rfp, rst, rext, rslots = oracle_full(name)
    bad = np.nonzero(out != ref)[0]
    assert len(bad) == 0, f"{what}: {len(bad)} mismatches, first at pods {bad[:5]}: gpu {out[bad[:5]]} oracle {ref[bad[:5]]}"
    sched = ref >= 0
    np.testing.assert_array_equal(score[sched & (rscore > 0)], rscore[sched & (rscore > 0)], err_msg=what)
    np.testing.assert_array_equal(fp, rfp, err_msg=what)
    np.testing.assert_array_equal(fc, rfc, err_msg=what)
    st, ext = eng.state(), eng.state_ext()
    for k in rst:
        np.testing.assert_array_equal(st[k], rst[k], err_msg=f"{what}: {k}")
    for k in rext:
        np.testing.assert_array_equal(ext[k], rext[k], err_msg=f"{what}: {k}")
    np.testing.assert_array_equal(eng.gpu_slot_words(), rslots, err_msg=f"{what}: GPU slots")


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(BUILDERS))
def test_full_run_matches_oracle(name):
    _p, c = case(name)
    for big in (False, True):
        with _engine(c, record_scores=True, force_large=big) as eng:
            out, score, fc, fp = eng.schedule()
            li = eng.last_launch()
            assert li["kernel"].startswith("simon_place_kernel_") and li["large"] == big, li
            assert (li["kernel"] == "simon_place_kernel_big") == big, li
            _assert_run(name, eng, out, score, fc, fp, f"{name} large={big}")
    if name == "gpu8":
        slots, gu = oracle_full(name)[6], oracle_full(name)[5]["gpu_used"]
        nib = np.array([(slots >> np.uint32(4 * d)) & np.uint32(15) for d in range(8)])
        assert (nib == 15).any() and (gu == 16 << 30).any()      # a saturated slot word, a device full with 16 slots of 1 GiB


def _node_lists(n, seed):
    rng = np.random.default_rng(seed)
    return [np.arange(n), np.arange(0, n, 2), np.arange(n)[: (2 * n) // 3][::-1], rng.permutation(n)[: (4 * n) // 5]]


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(BUILDERS))
def test_scenario_batch_matches_oracle(name):
    from oracle.binding import Oracle
    _p, c = case(name)
    lists = _node_lists(c.n_nodes, 3)
    with _engine(c) as eng:
        res, nodes = eng.run_scenarios(lists, want_nodes=True)
        assert eng.last_launch()["n_scenarios"] == len(lists)
    o = Oracle(c)
    for i, act in enumerate(lists):
        o.set_active(act)
        o.reset()
        ref = o.schedule()[0]
        st = o.state()
        np.testing.assert_array_equal(nodes[i], ref, err_msg=f"{name} scenario {i}")
        assert res[i]["n_unscheduled"] == int((ref == -1).sum()), i
        assert (res[i]["req_mcpu"], res[i]["req_mem"]) == (int(st["req_mcpu"][act].sum()), int(st["req_mem"][act].sum())), i
    o.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(BUILDERS))
def test_resume_from_half_rebuilds_the_state(name):
    _p, c = case(name)
    ref, _s, _fc, _fp, rst, rext, rslots = oracle_full(name)
    with _engine(c) as eng:
        out = eng.schedule_resume(ref[: len(ref) // 2])[0]
        np.testing.assert_array_equal(out, ref)
        st, ext = eng.state(), eng.state_ext()
        for k in rst:
            np.testing.assert_array_equal(st[k], rst[k], err_msg=k)
        for k in rext:
            np.testing.assert_array_equal(ext[k], rext[k], err_msg=k)
        np.testing.assert_array_equal(eng.gpu_slot_words()[len(ref) // 2:], rslots[len(ref) // 2:])


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(BUILDERS))
def test_drains_match_checker(name):
    import checkers
    from oracle.binding import Oracle
    from simon_b200 import scaledown
    from test_drain import _assert_drain_equal
    _p, c = case(name)
    o = Oracle(c)
    placed = o.schedule()[0]
    rng = np.random.default_rng(7)
    order = scaledown.NodeOrder(c)
    drains = [[int(g)] for g in rng.choice(c.n_nodes, 4, replace=False)]
    drains += [rng.choice(c.n_nodes, int(rng.integers(2, max(3, c.n_nodes // 4))), replace=False).tolist() for _ in range(3)]
    remain = [order.remaining(d) for d in drains]
    with _engine(c, record_scores=True) as eng:
        got = eng.drain_run(placed, remain)
    for d, rl, g in zip(drains, remain, got):
        want = checkers.drain(o, placed, rl)
        _assert_drain_equal(g, want, f"{name} drain {d}")
        pos = g["node"] >= 0
        assert np.array_equal(g["score"][pos], want["score"][pos]), d
    o.close()


def _hand_picked(name, c, out):
    """Moves the sampler may miss: for entries32, every pod of A onto every node that holds a partner pod b<i> (NodePorts must
    refuse each); otherwise every pod of the first 8 classes onto 16 fixed nodes."""
    cls = c.pods["pod_class"]
    if name == "entries32":
        names = [r.tmpl.workload_name for r in c.pod_recs]
        a = [q for q in range(len(out)) if names[q] == "a" and out[q] >= 0]
        held = sorted({int(out[q]) for q in range(len(out)) if names[q].startswith("b") and out[q] >= 0})
        mv = [(q, g) for q in a for g in held if g != out[q]]
        assert len(mv) >= 20
        return np.array(mv, np.uint32)
    pods = [q for q in range(len(out)) if cls[q] < 8 and out[q] >= 0][:64]
    return np.array([(q, g) for q in pods for g in range(0, c.n_nodes, max(1, c.n_nodes // 16))], np.uint32).reshape(-1, 2)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(BUILDERS))
def test_moves_match_checker(name):
    from oracle.binding import Oracle
    from simon_b200 import moves as M
    from test_moves_scope import _engine_vs_checker
    _p, c = case(name)
    o = Oracle(c)
    out = o.schedule()[0]
    mv = M.sample_moves(len(out), c.n_nodes, 20000, seed=5, placement=out)
    hand = _hand_picked(name, c, out)
    mv = np.concatenate([hand, mv]).astype(np.uint32)
    n_feasible = 0
    for scope in ((0, GPU | HARD) if name in SCOPED else (0,)):
        code = _engine_vs_checker(c, o, out, mv, scope)
        assert (code[len(hand):] != 0).any(), scope
        n_feasible += int((code == 0).sum())
        if name == "entries32":
            assert (code[:len(hand)] == 1 << 1).all(), (scope, np.unique(code[:len(hand)]))   # SFC_PORTS on every hand-picked move
    assert n_feasible > 0
    o.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kw,what", [(dict(n_ports=33), "33 constraint/term entries"), (dict(n_hard=9, n_soft=8), "entries exceed"),
                                     (dict(n_hard=8, n_soft=9), "entries exceed")],
                         ids=["entries33", "hard9", "soft9"])
def test_upload_refuses_one_past_the_entry_limits(kw, what):
    """33 entries, 9 DoNotSchedule or 9 ScheduleAnyway constraints in one class: the upload refuses the cluster, never narrows."""
    _p, c = compiled(*entries32(**kw))
    with pytest.raises(RuntimeError, match=what):
        _engine(c)
