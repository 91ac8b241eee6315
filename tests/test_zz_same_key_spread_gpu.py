"""PodTopologySpread constraints of one kind that share a topology key, on the engine: against the object-level restatement
(oracle/pyref.py: node, winning total and failure histogram of every pod) and against the C oracle and the checkers built on it
(state, per-node detail, scenario batches, drains, resumed runs, move scoring and migration plans).

Such constraints share one summed counter per key, which a pod of a class that m of the key's selectors match increments m times;
a later ScheduleAnyway constraint on a non-hostname key has topology size 0 (see test_same_key_spread.py for the reference's
rules and the known answers).  The file sorts after the rest of the suite.
"""
import functools

import numpy as np
import pytest

import test_drain as TD
from test_same_key_spread import SEEDS, kat_case, oracle_run
from util import assert_matches_walk, make_case, pyref_walk

pytestmark = pytest.mark.gpu
HARD = 2


def _engine(c, cs=0, t=0, big=False, **kw):
    from simon_b200.engine import Engine
    return Engine(c, device=0, cluster_ctas=cs, threads_per_cta=t, force_large=big, **kw)


def _assert_state(eng, st, what):
    got = eng.state()
    for k in st:
        np.testing.assert_array_equal(got[k], st[k], err_msg=f"{what} {k}")


@pytest.mark.parametrize("seed", SEEDS)
def test_engine_matches_pyref_same_key(seed):
    """Every pod of the seeded clusters: node, winning total and failure histogram against a per-pod pyref walk, state() against
    the oracle's."""
    p, c = make_case("same_key", seed_no=seed)
    st = oracle_run(c)[4]
    with _engine(c, record_scores=True) as eng:
        out, score, fc, fp = eng.schedule()
        assert_matches_walk(pyref_walk(p, c), out, score, fc, fp, f"seed {seed}")
        _assert_state(eng, st, f"seed {seed}")


@functools.lru_cache(maxsize=None)
def large():
    """300 nodes and about 280 pods of the same-key generator, with its pyref walk and oracle run."""
    p, c = make_case("same_key", seed_no=31, n_nodes=300, n_workloads=60, max_replicas=8)
    return p, c, pyref_walk(p, c), oracle_run(c)


# kernel -> (CTAs, threads per CTA, large-cluster variant) for 300 nodes: one slot per thread, 5 slots (counted at run time), and
# the large-cluster variant
GEOMS = {"simon_place_kernel_256_1": (2, 160, False), "simon_place_kernel_256_0": (1, 64, False), "simon_place_kernel_big": (2, 160, True)}


@pytest.mark.parametrize("kernel", sorted(GEOMS))
def test_variant_matches_pyref_and_oracle_same_key(kernel):
    cs, t, big = GEOMS[kernel]
    p, c, walk, (_o, rscore, rfc, rfp, rst) = large()
    with _engine(c, cs, t, big, record_scores=True) as eng:
        out, score, fc, fp = eng.schedule()
        li = eng.last_launch()
        assert li["kernel"] == kernel and (li["cluster_ctas"], li["threads_per_cta"], li["large"]) == (cs, t, big), li
        assert_matches_walk(walk, out, score, fc, fp, kernel)
        np.testing.assert_array_equal(fc, rfc)
        np.testing.assert_array_equal(fp, rfp)
        _assert_state(eng, rst, kernel)
    assert (out == -1).any() and (out >= 0).sum() > len(out) // 2


@pytest.mark.parametrize("name", ["sum_blocks", "critical_path", "soft_zone_log2", "soft_hostname"])
def test_known_answers_on_the_engine(name):
    """The CPU suite's known-answer clusters: the engine's run equals the pyref walk, and the last pod's per-node totals and filter
    verdicts equal the oracle's."""
    p, c = kat_case(name)
    with _engine(c, record_scores=True) as eng:
        out, score, fc, fp = eng.schedule()
        assert_matches_walk(pyref_walk(p, c), out, score, fc, fp, name)
    last = len(p.pods) - 1
    _o, _s, _fc, _fp, _st, sc = oracle_run(c, dump_pod=last)
    with _engine(c) as eng:
        dout, tot, code = eng.dump_pod(last)
    np.testing.assert_array_equal(dout, out[:last + 1])
    feas = code == 0
    ref_tot = np.array([int(x[8]) for x in sc], np.int64)
    if feas.sum() > 1:
        np.testing.assert_array_equal(tot[feas], ref_tot[feas], err_msg=name)


def test_dumped_pods_match_oracle_detail():
    """dump_pod of a few pods of the 300-node cluster with same-key constraints of each kind: per-node totals (where more than one
    node is feasible) and the feasible set against the oracle's per-node detail."""
    from oracle.binding import Oracle
    p, c, walk, _ref = large()
    kinds = []
    for i, r in enumerate(p.pods):
        tsc = r.tmpl.pod["spec"].get("topologySpreadConstraints") or []
        keys = [t["topologyKey"] for t in tsc]
        if r.node_name or len(keys) == len(set(keys)):
            continue
        kinds.append((frozenset(t["whenUnsatisfiable"] for t in tsc), i))
    chosen = {}
    for k, i in kinds:
        chosen.setdefault(k, []).append(i)
    pods = sorted({v[len(v) // 2] for v in chosen.values()} | {kinds[-1][1]})
    assert len(pods) >= 3
    for pod in pods:
        o = Oracle(c)
        o.enable_dump()
        ref_out = o.schedule(0, pod + 1)[0]
        ref_code, sc = o.last_detail()
        o.close()
        with _engine(c) as eng:
            out, tot, code = eng.dump_pod(pod)
        np.testing.assert_array_equal(out, ref_out)
        np.testing.assert_array_equal(code == 0, np.asarray(ref_code) == 0, err_msg=f"pod {pod}")
        feas = np.asarray(ref_code) == 0
        if feas.sum() > 1:
            np.testing.assert_array_equal(tot[feas], np.array([int(x[8]) for x in sc], np.int64)[feas], err_msg=f"pod {pod}")


def test_scenario_batch_matches_oracle_same_key():
    """All nodes, every other node, a reversed prefix and a random subset in one batch, each against the oracle on that list."""
    from oracle.binding import Oracle
    _p, c, _walk, _ref = large()
    n = c.n_nodes
    rng = np.random.default_rng(3)
    lists = [np.arange(n), np.arange(0, n, 2), np.arange(n)[: (2 * n) // 3][::-1], rng.permutation(n)[: (4 * n) // 5]]
    with _engine(c) as eng:
        res, nodes = eng.run_scenarios(lists, want_nodes=True)
    o = Oracle(c)
    for i, act in enumerate(lists):
        o.set_active(act)
        o.reset()
        ref = o.schedule()[0]
        np.testing.assert_array_equal(nodes[i], ref, err_msg=f"scenario {i}")
        assert res[i]["n_unscheduled"] == int((ref == -1).sum()), i
    o.close()


@pytest.mark.parametrize("kernel", ["simon_drain_kernel_256", "simon_drain_kernel_big"])
def test_drain_batch_matches_checker_same_key(kernel):
    """Drains take each evicted pod's counter increments out of the live state (as many as its class's multiplicity) before
    placing it again: against the drain checker, which rebuilds every drain's state from empty."""
    import checkers
    from simon_b200 import scaledown
    cs, t, big = TD.DRAIN_VARIANTS[kernel]
    rng = np.random.default_rng(5)
    for seed in (2, 5):
        _p, c = make_case("same_key", seed_no=seed, n_nodes=40, n_workloads=20)
        o, placed = TD._live(c)
        order = scaledown.NodeOrder(c)
        drains = TD._drains(c, rng, n_single=15)
        remain = [order.remaining(d) for d in drains]
        with _engine(c, cs, t, big, record_scores=True) as eng:
            got = eng.drain_run(placed, remain)
            assert eng.last_launch()["kernel"] == kernel
        n_evicted = 0
        for d, rl, g in zip(drains, remain, got):
            want = checkers.drain(o, placed, rl)
            TD._assert_drain_equal(g, want, f"{kernel} seed {seed} drain {d}")
            n_evicted += g["n_evicted"]
        assert n_evicted > 0
        o.close()


def test_resume_from_half_matches_pyref_same_key():
    """schedule_resume rebuilds the first half's counters (with their multiplicity) at the nodes of the pyref walk, then places the
    rest: the same nodes and state as the oracle's full run."""
    _p, c, walk, (ref, _s, _fc, _fp, rst) = large()
    P = len(ref)
    np.testing.assert_array_equal(walk[0], ref)
    with _engine(c) as eng:
        out = eng.schedule_resume(walk[0][: P // 2])[0]
        np.testing.assert_array_equal(out, ref)
        _assert_state(eng, rst, "resume")


def _own_count_cluster():
    """Zones A (a1, a2), B (b1) and C (c1), equal nodes.  Running: a=x on b1, b=y on c1.  p (a=x, b=y) has DoNotSchedule zone
    constraints a=x and b=y, maxSkew 1: summed counts A 0, B 1, C 1, so p goes to A (a1).  Then A holds p's count of 2.  Moved
    with p taken off (counts 0, 1, 1, min 0): to a2 passes (0 + 1 - 0), to b1 and c1 fails on skew (1 + 1 - 0 = 2 > 1).  Taking off
    only 1 would leave A at 1 and the minimum at 1, and let p onto b1 and c1."""
    from test_moves_scope import _compile, _node, _pod
    nodes = [_node("a1", 4, "A"), _node("a2", 4, "A"), _node("b1", 4, "B"), _node("c1", 4, "C")]
    cons = [{"maxSkew": 1, "topologyKey": "topology.kubernetes.io/zone", "whenUnsatisfiable": "DoNotSchedule",
             "labelSelector": {"matchLabels": sel}} for sel in ({"a": "x"}, {"b": "y"})]
    pods = [_pod("rb", {"a": "x"}, "b1"), _pod("rc", {"b": "y"}, "c1"), _pod("p", {"a": "x", "b": "y"}, spec_extra={"topologySpreadConstraints": cons})]
    return _compile(nodes, pods)


def test_hard_spread_moves_take_out_the_own_count():
    """Moves of a pod that two same-key selectors match remove its count of 2 at its source: hand-picked moves and every move of the
    seeded clusters, at scope HARD_SPREAD, against the scoped checker."""
    from oracle.binding import Oracle
    from simon_b200.abi import SFC_PTS_SKEW
    from test_moves_scope import _engine_vs_checker, _moves
    c, names = _own_count_cluster()
    o = Oracle(c)
    out = o.schedule()[0]
    n = {x: c.node_names.index(x) for x in ("a1", "a2", "b1", "c1")}
    q = names.index("p")
    assert out[q] == n["a1"]
    mv = np.array([(q, n["a2"]), (q, n["b1"]), (q, n["c1"])], np.uint32)
    code = _engine_vs_checker(c, o, out, mv, HARD)
    assert code[0] == 0 and code[1] == code[2] == 1 << SFC_PTS_SKEW, code.tolist()
    o.close()
    for seed in SEEDS[:4]:
        _p, c = make_case("same_key", seed_no=seed)
        o = Oracle(c)
        out = o.schedule()[0]
        mv = _moves(out, c, 20000, seed=seed)
        code = _engine_vs_checker(c, o, out, mv, HARD)
        assert (code == 0).any() and (code == 1 << SFC_PTS_SKEW).any(), seed
        o.close()


def test_migration_plan_matches_checker_same_key():
    """A short migration plan with hard-spread classes admitted, step by step and in its end state against the plan checker, and
    its end placement resumed on a fresh context."""
    from simon_b200 import rebalance
    from test_moves_plan import _engine_vs_checker, _oracle_state
    steps = 0
    for seed in (1, 3, 6):
        _p, c = make_case("same_key", seed_no=seed)
        o, out = _oracle_state(c)
        o.close()
        mv = rebalance.candidates(c, out)
        r = _engine_vs_checker(c, mv, 12, 1, HARD, rebuild=True)
        steps += len(r["steps"])
    assert steps > 0
