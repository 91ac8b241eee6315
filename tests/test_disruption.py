"""PodDisruptionBudgets (simon_b200/disruption.py, simon_pdbs_upload): membership, desired counts and refusals of the compiler; the plan
checker with a PDB table against the PDB-less checker run one step at a time.  GPU: identity without a table (or
with an unconstraining one), `allowed` on the device, drains against an object-level restatement of filterPodsWithPDBViolation, move
scoring, plans against the checker, scale, refusals and the session option."""
import ctypes as C
import re

import numpy as np
import pytest

import checkers
from util import make_case

NO_MOVE, MAX_MOVES = 1, 2
GPU, HARD = 1, 2


def pdb(name, ns="default", selector=None, **spec):
    o = {"apiVersion": "policy/v1beta1", "kind": "PodDisruptionBudget", "metadata": {"name": name, "namespace": ns}, "spec": dict(spec)}
    if selector is not None:
        o["spec"]["selector"] = selector
    return o


# ---- the object-level restatement: filterPodsWithPDBViolation's membership and count over dict labels (independent of the CSR) ----

def _sel_matches(sel, labels):
    if sel is None:
        return False
    ml, me = sel.get("matchLabels") or {}, sel.get("matchExpressions") or []
    if not ml and not me:
        return False                      # an empty selector matches nothing here
    for k, v in ml.items():
        if labels.get(k) != str(v):
            return False
    for e in me:
        k, op, vals = e["key"], e["operator"], [str(x) for x in e.get("values") or []]
        ok = {"In": k in labels and labels[k] in vals, "NotIn": k not in labels or labels[k] not in vals,
              "Exists": k in labels, "DoesNotExist": k not in labels}[op]
        if not ok:
            return False
    return True


def members_ref(pdbs, recs):
    """Per PDB: the pod indices of its members."""
    out = []
    for o in pdbs:
        ns = o["metadata"].get("namespace") or "default"
        sel = o["spec"].get("selector")
        out.append([q for q, r in enumerate(recs) if (r.tmpl.namespace or "default") == ns and _sel_matches(sel, r.tmpl.labels)])
    return out


def violations_ref(pdbs, recs, evicted, allowed):
    """filterPodsWithPDBViolation(evicted, PDBs with DisruptionsAllowed = allowed): {pdb: evicted members} over the violated PDBs."""
    mem = [set(m) for m in members_ref(pdbs, recs)]
    cnt = {}
    for q in evicted:
        for j, m in enumerate(mem):
            if q in m:
                cnt[j] = cnt.get(j, 0) + 1
    return {j: n for j, n in cnt.items() if n > allowed[j]}


def app_pairs(c):
    """(namespace, app label) of the pods of workloads (outside kube-system)."""
    return sorted({(r.tmpl.namespace or "default", r.tmpl.labels["app"]) for r in c.pod_recs
                   if r.tmpl.labels.get("app") and r.tmpl.namespace != "kube-system"})


def mixed_pdbs(c, seed=0):
    """PDBs of every spec form over the compiled pod list: one per (namespace, app label) of the workloads (random forms), tier selectors
    by matchExpressions in every such namespace (overlapping the app PDBs: pods in two PDBs), a kube-system one, an empty and a nil
    selector and one without members."""
    rng = np.random.RandomState(seed)
    apps = app_pairs(c)
    forms = [dict(maxUnavailable=1), dict(minAvailable=2), dict(minAvailable="50%"), dict(maxUnavailable="25%"), dict(minAvailable=0),
             dict(maxUnavailable=0)]
    out = [pdb(f"app-{a}", ns=ns, selector={"matchLabels": {"app": a}}, **forms[int(rng.randint(len(forms)))]) for ns, a in apps]
    for ns in sorted({ns for ns, _ in apps}):
        out.append(pdb("tier-web", ns=ns, selector={"matchExpressions": [{"key": "tier", "operator": "In", "values": ["web"]}]},
                       maxUnavailable="30%"))
        out.append(pdb("tier-not-db", ns=ns, selector={"matchExpressions": [{"key": "tier", "operator": "Exists"},
                                                                             {"key": "tier", "operator": "NotIn", "values": ["db"]}]},
                       minAvailable="60%"))
    out.append(pdb("sys", ns="kube-system", selector={"matchExpressions": [{"key": "app", "operator": "Exists"}]}, maxUnavailable=2))
    out.append(pdb("empty", selector={}, maxUnavailable=0))
    out.append(pdb("nil", minAvailable=1))
    out.append(pdb("nobody", selector={"matchLabels": {"app": "no-such-app"}}, maxUnavailable=1))
    return out


# ---------------------------------------------------------------------------------------------------------------- CPU ----

@pytest.mark.parametrize("seed", [0, 1, 2])
def test_membership_equals_object_restatement(seed):
    from simon_b200 import disruption
    p, c = make_case("mix", seed_no=103 + seed, n_nodes=40, n_workloads=20, max_replicas=6)
    pdbs = mixed_pdbs(c, seed)
    t = disruption.compile_pdbs(pdbs, c)
    ref = members_ref(pdbs, c.pod_recs)
    got = [[] for _ in pdbs]
    for q in range(len(c.pod_recs)):
        ids = t.pdbs_of(q).tolist()
        assert ids == sorted(set(ids))
        for j in ids:
            got[j].append(q)
    assert got == ref
    assert t.expected.tolist() == [len(m) for m in ref]
    names = [o["metadata"]["name"] for o in pdbs]
    for nm in ("empty", "nil", "nobody"):
        assert ref[names.index(nm)] == []
    assert any(len(t.pdbs_of(q)) >= 2 for q in range(len(c.pod_recs)))      # pods in several PDBs
    assert sum(1 for m in ref if m) >= 4


def test_desired_every_spec_form():
    from simon_b200.disruption import desired_of
    assert desired_of({"minAvailable": 3}, 10) == 3
    assert desired_of({"minAvailable": 12}, 10) == 12                   # above expected: nothing is allowed
    assert desired_of({"minAvailable": "50%"}, 7) == 4                  # ceil(3.5)
    assert desired_of({"minAvailable": "33%"}, 10) == 4                 # ceil(3.3)
    assert desired_of({"minAvailable": "0%"}, 10) == 0
    assert desired_of({"maxUnavailable": 1}, 10) == 9
    assert desired_of({"maxUnavailable": 15}, 10) == 0                  # above expected
    assert desired_of({"maxUnavailable": "25%"}, 10) == 7               # 10 - ceil(2.5)
    assert desired_of({"maxUnavailable": "25%"}, 1) == 0                # 1 - ceil(0.25)
    assert desired_of({"maxUnavailable": "100%"}, 6) == 0
    assert desired_of({"minAvailable": "100%"}, 0) == 0


@pytest.mark.parametrize("spec,msg", [
    (dict(minAvailable=1, maxUnavailable=1), "both are"),
    (dict(), "neither is"),
    (dict(minAvailable="3"), "without '%'"),
    (dict(maxUnavailable=-1), "negative"),
    (dict(minAvailable="-5%"), "not a non-negative"),
    (dict(minAvailable=1.5), "neither an integer"),
])
def test_compile_refusals(spec, msg):
    from simon_b200 import disruption
    from simon_b200.compiler import CompileError
    p, c = make_case("mix", seed_no=103, n_nodes=12, n_workloads=6, max_replicas=3)
    with pytest.raises(CompileError, match=re.escape(msg)):
        disruption.compile_pdbs([pdb("x", selector={"matchLabels": {"app": "wl-001"}}, **spec)], c)


def test_compile_refuses_bad_selector():
    from simon_b200 import disruption
    from simon_b200.compiler import CompileError
    p, c = make_case("mix", seed_no=103, n_nodes=12, n_workloads=6, max_replicas=3)
    for sel in ({"matchExpressions": [{"key": "a", "operator": "In", "values": []}]},
                {"matchExpressions": [{"key": "a", "operator": "Gt", "values": ["1"]}]}):
        with pytest.raises(CompileError, match="selector"):
            disruption.compile_pdbs([pdb("x", selector=sel, maxUnavailable=1)], c)


def _plan_case(seed=0):
    from simon_b200 import rebalance
    from oracle.binding import Oracle
    p, c = make_case("mix", seed_no=215 + seed, n_nodes=45, n_workloads=30, max_replicas=9)
    o = Oracle(c)
    out = o.schedule()[0]
    o.close()
    return p, c, out, rebalance.candidates(c, out)


@pytest.mark.parametrize("seed", [0, 1])
def test_pdb_checker_equals_stepwise_pdb_less_checker(seed):
    """The checker with a PDB table equals the PDB-less checker run one step at a time on one oracle state, each step given the move
    list without the moves of pods that moved or belong to a PDB whose budget is spent (an explicit exclusion list)."""
    from simon_b200 import disruption
    from oracle.binding import Oracle
    p, c, out, mv = _plan_case(seed)
    t = disruption.compile_pdbs(mixed_pdbs(c, seed), c)
    allowed = t.allowed(out)
    max_moves = 40
    o = Oracle(c)
    o.schedule()
    ref = checkers.plan_pdb(o, mv, out, o.gpu_slot_words(), max_moves, 1, 0, t.pod_off, t.pod_pdb, allowed)
    o.close()
    # the second mechanism
    o = Oracle(c)
    o.schedule()
    placement, slots = out.copy(), o.gpu_slot_words()
    remaining = allowed.astype(np.int64).copy()
    moved, steps, stop = set(), [], NO_MOVE
    while len(steps) < max_moves:
        excluded = set(moved)
        for q in range(len(out)):
            if (remaining[t.pdbs_of(q)] <= 0).any():
                excluded.add(q)
        keep = np.array([int(m[0]) not in excluded for m in mv], bool)
        idx = np.nonzero(keep)[0]
        r = checkers.plan(o, mv[idx], placement, slots, 1, 1, 0)
        if not len(r["steps"]):
            stop = r["stop_reason"]
            break
        s = r["steps"][0].copy()
        s[0] = idx[s[0]]
        steps.append(tuple(int(x) for x in s))
        placement, slots = r["placement"], r["slots"]
        moved.add(int(s[1]))
        remaining[t.pdbs_of(int(s[1]))] -= 1
    else:
        stop = MAX_MOVES
    o.close()
    assert [tuple(int(x) for x in s) for s in ref["steps"]] == steps
    assert ref["stop_reason"] == stop
    np.testing.assert_array_equal(ref["placement"], placement)
    spent = np.zeros(t.n_pdbs, np.int64)
    for s in steps:
        spent[t.pdbs_of(s[1])] += 1
    assert (spent <= allowed).all() and len(steps) > 0
    assert ref["pdb_blocked"] == sum(1 for q in range(len(out)) if out[q] >= 0 and (allowed[t.pdbs_of(q)] <= 0).any()
                                     and not _pinned(c)[c.pods["pod_class"][q]])


def _pinned(c):
    from simon_b200.compiler import CLS_PINNED, SCW_FLAGS
    off, blob = c.pods["class_off"], c.pods["class_blob"]
    return np.array([(int(blob[int(off[k]) + SCW_FLAGS]) & CLS_PINNED) != 0 for k in range(len(off) - 1)])


# ---------------------------------------------------------------------------------------------------------------- GPU ----

def _upload_raw(eng, n_pdbs, n_pods, off, ids, desired):
    from simon_b200 import abi
    from simon_b200.engine import lib
    keep = [np.ascontiguousarray(off, np.uint32), np.ascontiguousarray(ids if len(ids) else [0], np.uint32),
            np.ascontiguousarray(desired if len(desired) else [0], np.int32)]
    s = abi.SimonPdbs(n_pdbs, n_pods, *[a.ctypes.data for a in keep])
    rc = lib().simon_pdbs_upload(eng.h, C.byref(s))
    return rc, lib().simon_last_error(eng.h).decode()


def _generous(c):
    """One PDB per pod plus one over all pods, none binding: each allows at least every pod to go."""
    from simon_b200.disruption import PdbTables
    P = len(c.pod_recs)
    off = np.arange(P + 1, dtype=np.uint32) * 2
    ids = np.stack([np.zeros(P, np.uint32), np.arange(1, P + 1, dtype=np.uint32)], 1).reshape(-1)
    return PdbTables(names=["all"] + [f"p{q}" for q in range(P)], pod_off=off, pod_pdb=ids, desired=np.zeros(P + 1, np.int32))


def _run_all(eng, c, out, mv, remain, table):
    """Move runs (both scopes), drains and a plan on the engine; -> (outputs, launch count deltas)."""
    from simon_b200.disruption import PdbTables
    if table == "none":
        pass
    elif table == "empty":
        eng.pdbs_upload(PdbTables(names=[], pod_off=np.zeros(len(out) + 1, np.uint32), pod_pdb=np.zeros(0, np.uint32),
                                  desired=np.zeros(0, np.int32)))
    else:
        eng.pdbs_upload(table)
    res, launches = [], []
    for scope in (0, GPU | HARD):
        eng.moves_set_scope(scope)
        eng.moves_upload(mv, 0)
        n0 = eng.launch_count()
        r = eng.moves_run(k=16, want_arrays=True, want_per_pod=True)
        launches.append(eng.launch_count() - n0)
        res.append((r["gain"].tolist(), r["code"].tolist(), r["topk"], r["best_key"], r["best_per_pod"].tolist()))
    n0 = eng.launch_count()
    d = eng.drain_run(out, remain, detail=True)
    launches.append(eng.launch_count() - n0)
    res.append([{k: (v.tolist() if hasattr(v, "tolist") else v) for k, v in x.items() if k not in ("n_pdb_violated", "pdb_violated", "pdb_evicted")}
                for x in d])
    assert all(x["n_pdb_violated"] == 0 for x in d)
    eng.moves_set_scope(0)
    eng.moves_upload(mv, 0)
    n0 = eng.launch_count()
    r = eng.moves_plan(25, 1)
    launches.append(eng.launch_count() - n0)
    pl, sl = eng.moves_plan_download()
    st = eng.moves_plan_state()
    res.append((r["steps"].tolist(), r["stop_reason"], r["excluded"], pl.tolist(), sl.tolist(), {k: v.tolist() for k, v in st[0].items()}))
    return res, launches, len(r["steps"]) + 0


@pytest.mark.gpu
def test_identity_without_a_binding_table():
    from simon_b200 import moves as M, scaledown
    from simon_b200.engine import Engine
    p, c = make_case("c3", n_nodes=300, n_workloads=60, replicas=8, n_apps=2, seed_no=21, gpu_pct=20)
    runs = {}
    order = scaledown.NodeOrder(c)
    for table in ("none", "empty", "generous"):
        with Engine(c, device=0) as eng:
            out = eng.schedule()[0]
            mv = M.sample_moves(len(out), c.n_nodes, 40000, seed=5, placement=out)
            remain = [order.remaining([g]) for g in range(0, c.n_nodes, 7)]
            runs[table] = _run_all(eng, c, out, mv, remain, _generous(c) if table == "generous" else table)
    assert runs["none"][0] == runs["empty"][0] and runs["none"][1] == runs["empty"][1]
    assert runs["none"][0] == runs["generous"][0]
    ln, lg, steps = runs["none"][1], runs["generous"][1], runs["generous"][2]
    assert steps > 0
    # documented additions with a table: 3 per move run (count, allowed, mark), 2 per drain batch (count, allowed), and in a plan
    # 3 at the setup plus 2 per enqueued step (at least one per recorded step)
    assert lg[0] == ln[0] + 3 and lg[1] == ln[1] + 3 and lg[2] == ln[2] + 2
    extra = lg[3] - ln[3]
    assert extra >= 3 + 2 * steps and (extra - 3) % 2 == 0


@pytest.mark.gpu
def test_allowed_after_schedule_resume_and_drain():
    from simon_b200 import disruption, scaledown
    from simon_b200.engine import Engine
    p, c = make_case("mix", seed_no=215, n_nodes=45, n_workloads=30, max_replicas=9)
    pdbs = mixed_pdbs(c, 3)
    t = disruption.compile_pdbs(pdbs, c)
    with Engine(c, device=0) as eng:
        eng.pdbs_upload(t)
        with pytest.raises(RuntimeError, match="no placement"):
            eng.pdbs_allowed()
        out = eng.schedule()[0]
        np.testing.assert_array_equal(eng.pdbs_allowed(), t.allowed(out))
        ref_healthy = np.array([sum(1 for q in m if out[q] >= 0) for m in members_ref(pdbs, c.pod_recs)])
        np.testing.assert_array_equal(t.allowed(out), np.maximum(0, ref_healthy - t.desired))
        eng.schedule_resume(out[:len(out) // 2])
        np.testing.assert_array_equal(eng.pdbs_allowed(), t.allowed(eng.results()))
        # a drain's rebuild leaves `placed`, with some pods unplaced
        placed = out.copy()
        movable = np.nonzero((placed >= 0) & (c.pods["pod_fixed_node"] < 0) & ~_pinned(c)[c.pods["pod_class"]])[0]
        placed[movable[::3]] = -1
        eng.drain_run(placed, [scaledown.NodeOrder(c).remaining([0])], detail=False)
        np.testing.assert_array_equal(eng.pdbs_allowed(), t.allowed(placed))
        assert (t.allowed(placed) != t.allowed(out)).any()


@pytest.mark.gpu
def test_drain_sweep_pdb_violations():
    from simon_b200 import disruption, scaledown
    from simon_b200.engine import Engine
    p, c = make_case("mix", seed_no=104, n_nodes=60, n_workloads=40, max_replicas=8)
    pdbs = mixed_pdbs(c, 4)
    t = disruption.compile_pdbs(pdbs, c)
    order = scaledown.NodeOrder(c)
    remain = [order.remaining([g]) for g in range(c.n_nodes)]
    with Engine(c, device=0) as eng:
        out = eng.schedule()[0]
        base = eng.drain_run(out, remain, detail=True)
        eng.pdbs_upload(t)
        res = eng.drain_run(out, remain, detail=True)
        allowed = eng.pdbs_allowed()
    n_viol = 0
    for g, (r, b) in enumerate(zip(res, base)):
        for k in ("n_evicted", "n_placed", "n_unscheduled", "n_blocked", "n_vanished", "req_mcpu", "req_mem"):
            assert r[k] == b[k], (g, k)
        np.testing.assert_array_equal(r["node"], b["node"])
        want = violations_ref(pdbs, c.pod_recs, r["evicted"].tolist(), allowed)
        assert r["n_pdb_violated"] == len(want)
        assert dict(zip(r["pdb_violated"].tolist(), r["pdb_evicted"].tolist())) == want
        assert r["pdb_violated"].tolist() == sorted(want)
        n_viol += bool(want)
    assert 0 < n_viol < c.n_nodes
    # 8 sampled drains: the same restatement on the CPU drain checker's evicted lists
    from oracle.binding import Oracle
    o = Oracle(c)
    np.testing.assert_array_equal(o.schedule()[0], out)
    rng = np.random.RandomState(1)
    for g in rng.choice(c.n_nodes, 8, replace=False).tolist():
        ev = checkers.drain(o, out, remain[g])["evicted"]
        want = violations_ref(pdbs, c.pod_recs, [int(q) for q in ev], allowed)
        assert dict(zip(res[g]["pdb_violated"].tolist(), res[g]["pdb_evicted"].tolist())) == want
    o.close()


@pytest.mark.gpu
def test_move_scoring_marks_pdb_blocked_pods():
    from simon_b200 import disruption, moves as M
    from simon_b200.engine import Engine
    p, c = make_case("c3", n_nodes=400, n_workloads=80, replicas=10, n_apps=2, seed_no=21, gpu_pct=25)
    pdbs = mixed_pdbs(c, 5) + [pdb(f"tight-{a}", ns=ns, selector={"matchLabels": {"app": a}}, maxUnavailable=0) for ns, a in app_pairs(c)[::4]]
    t = disruption.compile_pdbs(pdbs, c)
    with Engine(c, device=0) as eng:
        out = eng.schedule()[0]
        mv = M.sample_moves(len(out), c.n_nodes, 100000, seed=3, placement=out)
        for scope in (0, GPU | HARD):
            eng.pdbs_upload(None)
            eng.moves_set_scope(scope)
            eng.moves_upload(mv, 0)
            a = eng.moves_run(k=0)
            eng.pdbs_upload(t)
            b = eng.moves_run(k=0)
            blocked = disruption.blocked_pods(t, t.allowed(out))[mv[:, 0]]
            assert blocked.any()
            NM = 1 << 26
            was = a["code"] == NM
            live = (a["code"] & ((1 << 25) | (1 << 24) | (1 << 27))) == 0      # placed, not a no-op, index in range
            want_nm = was | (blocked & live)
            np.testing.assert_array_equal(b["code"] == NM, want_nm)
            keep = ~want_nm
            np.testing.assert_array_equal(b["code"][keep], a["code"][keep])
            np.testing.assert_array_equal(b["gain"][keep], a["gain"][keep])


def _engine_plan(c, mv, t, max_moves, scope=0, min_gain=1, static_cache=True):
    from simon_b200.engine import Engine
    with Engine(c, device=0, static_cache=static_cache) as eng:
        out = eng.schedule()[0]
        eng.moves_set_scope(scope)
        eng.moves_upload(mv, 0)
        if t is not None:
            eng.pdbs_upload(t)
        allowed = eng.pdbs_allowed() if t is not None else None
        r = eng.moves_plan(max_moves, min_gain)
        pl, sl = eng.moves_plan_download()
        st = eng.moves_plan_state()
    return out, allowed, r, pl, sl, st


def _steps(r):
    s = r["steps"]
    return np.stack([s["move"], s["pod"], s["from"], s["to"], s["gain"], s["gpu_slots"]], 1).astype(np.int64) if len(s) else np.zeros((0, 6), np.int64)


def _plan_vs_checker(c, mv, t, max_moves, scope=0, rebuild=True, static_cache=True):
    from oracle.binding import Oracle
    from simon_b200.engine import Engine
    out, allowed, r, pl, sl, st = _engine_plan(c, mv, t, max_moves, scope, static_cache=static_cache)
    np.testing.assert_array_equal(allowed, t.allowed(out))
    o = Oracle(c)
    assert np.array_equal(o.schedule()[0], out)
    ref = checkers.plan_pdb(o, mv, out, o.gpu_slot_words(), max_moves, 1, scope, t.pod_off, t.pod_pdb, allowed)
    o.close()
    got = _steps(r)
    assert got.tolist() == ref["steps"].tolist()
    assert r["stop_reason"] == ref["stop_reason"] and r["excluded"] == ref["excluded"] and r["pdb_blocked"] == ref["pdb_blocked"]
    np.testing.assert_array_equal(pl, ref["placement"])
    np.testing.assert_array_equal(sl, ref["slots"])
    for k in ref["state"]:
        np.testing.assert_array_equal(st[0][k], ref["state"][k], err_msg=k)
    spent = np.zeros(t.n_pdbs, np.int64)
    for q in r["steps"]["pod"]:
        spent[t.pdbs_of(int(q))] += 1
    assert (spent <= allowed).all()
    if rebuild and not (scope & GPU):
        import copy
        c2 = copy.copy(c)
        c2.pods = dict(c.pods)
        fixed = np.array(c.pods["pod_fixed_node"], np.int32)
        moved = got[:, 1]
        fixed[moved] = np.where(fixed[moved] >= 0, pl[moved], fixed[moved])
        c2.pods["pod_fixed_node"] = fixed
        with Engine(c2, device=0, static_cache=static_cache) as eng:
            eng.schedule_resume(pl)
            s2 = eng.state()
        for k in s2:
            np.testing.assert_array_equal(s2[k], st[0][k], err_msg=f"resume {k}")
    return out, allowed, r


@pytest.mark.gpu
@pytest.mark.parametrize("kind,kw,scope", [
    ("mix", dict(seed_no=215, n_nodes=45, n_workloads=30, max_replicas=9), 0),
    ("mix", dict(seed_no=103, n_nodes=95, n_workloads=40, max_replicas=7), 0),
    ("c3", dict(n_nodes=400, n_workloads=80, replicas=10, n_apps=2, seed_no=21, gpu_pct=25), GPU),
    ("c3", dict(n_nodes=400, n_workloads=80, replicas=10, n_apps=2, seed_no=21, gpu_pct=25), HARD),
])
def test_plan_equals_pdb_checker(kind, kw, scope):
    from simon_b200 import disruption, rebalance
    p, c = make_case(kind, **kw)
    t = disruption.compile_pdbs(mixed_pdbs(c, 7), c)
    out0 = _engine_plan(c, np.zeros((0, 2), np.uint32), None, 1)[0]
    mv = rebalance.candidates(c, out0)
    if len(mv) > 300000:
        mv = mv[np.random.RandomState(3).choice(len(mv), 300000, replace=False)]
        mv = mv[np.lexsort((mv[:, 1], mv[:, 0]))]
    out, allowed, r = _plan_vs_checker(c, mv, t, 60, scope)
    assert len(r["steps"]) > 0
    # the plan departs from the PDB-less plan exactly at the first step whose unconstrained winner is blocked
    r0 = _engine_plan(c, mv, None, 60, scope)[2]
    a, b = _steps(r0), _steps(r)
    n = 0
    while n < min(len(a), len(b)) and (a[n] == b[n]).all():
        n += 1
    if n < len(a):
        remaining = allowed.astype(np.int64).copy()
        for q in b[:n, 1]:
            remaining[t.pdbs_of(int(q))] -= 1
        assert (remaining[t.pdbs_of(int(a[n, 1]))] <= 0).any()
    else:
        assert n == len(b)


def _table(lists, desired):
    from simon_b200.disruption import PdbTables
    off = np.r_[0, np.cumsum([len(l) for l in lists])].astype(np.uint32)
    ids = np.array([j for l in lists for j in l], np.uint32)
    return PdbTables(names=[str(j) for j in range(len(desired))], pod_off=off, pod_pdb=ids, desired=np.array(desired, np.int32))


def _live_c5(n_nodes, n_running):
    from simon_b200 import synth
    p, c = make_case("c3", n_nodes=n_nodes, n_workloads=50, replicas=4, n_apps=2, seed_no=9)
    live = synth.make_c5(c, n_running)
    return live, live.pods["pod_class"], len(live.pods["pod_class"])


@pytest.mark.gpu
def test_plan_c5_snapshot_and_two_pdbs_per_pod():
    """A live C5 snapshot: one PDB per pod class (maxUnavailable 1) and one over every pod (2 % may go): every pod is in two PDBs."""
    from simon_b200 import moves as M
    live, cls, P = _live_c5(500, 5000)
    n_cls = int(cls.max()) + 1
    cnt = np.bincount(cls, minlength=n_cls)
    t = _table([[int(cls[q]), n_cls] for q in range(P)], np.r_[np.maximum(0, cnt - 1), P - (2 * P + 99) // 100].tolist())
    out0 = _engine_plan(live, np.zeros((0, 2), np.uint32), None, 1)[0]
    mv = M.sample_moves(P, live.n_nodes, 300000, seed=11, placement=out0)
    out, allowed, r = _plan_vs_checker(live, mv, t, 40)
    assert len(r["steps"]) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("what", ["big_pdb", "many_pdbs", "pod_in_64"])
def test_plan_scale(what):
    """A PDB with over 100,000 members used up mid-plan; 100,000 PDBs; pods in 64 PDBs."""
    from simon_b200 import moves as M
    live, cls, P = _live_c5(2500, 160000)
    assert P > 100000
    if what == "big_pdb":
        lists, desired = [[0]] * P, [P - 3]                              # 3 moves, then its members stop
    elif what == "many_pdbs":
        lists = [[q % 100000] for q in range(P)]
        desired = np.maximum(0, np.bincount(np.arange(P) % 100000, minlength=100000) - 1).tolist()     # each allows one
    else:
        lists = [list(range(64)) if q % 7 == 0 else [64 + q % 5] for q in range(P)]
        desired = [len(range(0, P, 7)) - 4] * 64 + [0, 0, 0, 10 ** 6, 10 ** 6]
    t = _table(lists, desired)
    out0 = _engine_plan(live, np.zeros((0, 2), np.uint32), None, 1)[0]
    mv = M.sample_moves(P, live.n_nodes, 400000, seed=2, placement=out0)
    mv = mv[mv[:, 0] < 30000]
    out, allowed, r = _plan_vs_checker(live, mv, t, 12, rebuild=False)
    assert len(r["steps"]) > 0
    if what == "big_pdb":
        assert len(r["steps"]) == 3


@pytest.mark.gpu
def test_pdb_upload_refusals_and_drop():
    from simon_b200 import disruption, moves as M
    from simon_b200.engine import Engine, lib
    p, c = make_case("mix", seed_no=215, n_nodes=45, n_workloads=30, max_replicas=9)
    P = len(c.pod_recs)
    t = disruption.compile_pdbs(mixed_pdbs(c, 2) + [pdb("zero", selector={"matchLabels": {"tier": "web"}}, maxUnavailable=0)], c)
    with Engine(c, device=0) as eng:
        off = np.zeros(P + 1, np.uint32)
        bad = [
            ((2, P + 1, off, [], [0, 0]), "n_pods"),
            ((2, P, np.r_[off[:-1], 0], [], [0, 0]), None),
            ((2, P, np.r_[1, np.ones(P, np.uint32)], [0], [0, 0]), "pod_off[0]"),
            ((2, P, np.r_[0, 2, np.ones(P - 1, np.uint32)], [0, 1], [0, 0]), "not monotone"),
            ((2, P, np.r_[0, np.ones(P, np.uint32)], [2], [0, 0]), "names PDB 2 of 2"),
            ((2, P, np.r_[0, np.full(P, 2, np.uint32)], [1, 1], [0, 0]), "not ascending"),
            ((2, P, np.r_[0, np.full(P, 2, np.uint32)], [1, 0], [0, 0]), "not ascending"),
            ((2, P, off, [], [0, -1]), "desired -1"),
        ]
        for args, msg in bad:
            rc, err = _upload_raw(eng, *args)
            if msg is None:
                assert rc == 0
                continue
            assert rc == -1 and msg in err, (msg, err)
        out = eng.schedule()[0]
        mv = M.sample_moves(len(out), c.n_nodes, 20000, seed=1, placement=out)
        eng.moves_upload(mv, 0)
        a = eng.moves_run(k=4)
        eng.pdbs_upload(t)
        b = eng.moves_run(k=4)
        assert (a["code"] != b["code"]).any()
        # a new pod upload drops the table: behaviour equals no table
        rc = lib().simon_pods_upload(eng.h, C.byref(eng.pods))
        assert rc == 0
        eng.schedule()
        eng.moves_upload(mv, 0)
        d = eng.moves_run(k=4)
        np.testing.assert_array_equal(d["code"], a["code"])
        np.testing.assert_array_equal(d["gain"], a["gain"])
        assert eng.pdbs_allowed() is not None and lib().simon_pdbs_allowed(eng.h, None) == 0     # no table: nothing written
    with Engine(c, device=0) as eng:
        assert lib().simon_pdbs_allowed(eng.h, None) == -3 and "no placement" in lib().simon_last_error(eng.h).decode()


@pytest.mark.gpu
def test_session_honours_cluster_and_app_pdbs():
    from simon_b200 import rebalance, simulator, synth
    cluster, apps = synth.make_c3(n_nodes=200, n_workloads=40, replicas=6, n_apps=2, seed_no=4)
    with simulator.NewSimulator() as sim:
        sim.RunCluster(simulator.PrepareCluster(cluster))
        sim.ScheduleApp(apps[0])
        eng, c = sim._live()
        base_drain = sim.DrainNodes([[c.node_names[g]] for g in range(0, c.n_nodes, 5)])
        base_sd = sim.PlanScaleDown(max_remove=8)
        base_mp = sim.PlanMigrations(max_moves=20)
    # the app's workloads, half protected by PDBs of the cluster, half by PDBs of the app
    pairs = app_pairs(c)
    import copy
    cluster2 = copy.deepcopy(cluster)
    cluster2.PodDisruptionBudgets = [pdb(f"c-{a}", ns=ns, selector={"matchLabels": {"app": a}}, maxUnavailable=0) for ns, a in pairs[::2]]
    app0 = copy.deepcopy(apps[0])
    app0.Resource.PodDisruptionBudgets = [pdb(f"a-{a}", ns=ns, selector={"matchLabels": {"app": a}}, maxUnavailable=0) for ns, a in pairs[1::2]]
    # without the option: the same results as the current session
    with simulator.NewSimulator() as sim:
        sim.RunCluster(simulator.PrepareCluster(cluster2))
        sim.ScheduleApp(app0)
        d = sim.DrainNodes([[c.node_names[g]] for g in range(0, c.n_nodes, 5)])
        assert [(x.Drainable, len(x.EvictedPods)) for x in d] == [(x.Drainable, len(x.EvictedPods)) for x in base_drain]
        assert sim.PlanScaleDown(max_remove=8).RemovedNodes == base_sd.RemovedNodes
        assert [(m.Pod.name, m.To) for m in sim.PlanMigrations(max_moves=20).Migrations] == [(m.Pod.name, m.To) for m in base_mp.Migrations]
    with simulator.NewSimulator(simulator.WithPodDisruptionBudgets()) as sim:
        sim.RunCluster(simulator.PrepareCluster(cluster2))
        sim.ScheduleApp(app0)
        t = sim.pdb_tables
        assert t.n_pdbs == len(cluster2.PodDisruptionBudgets) + len(app0.Resource.PodDisruptionBudgets)
        d = sim.DrainNodes([[c.node_names[g]] for g in range(0, c.n_nodes, 5)])
        viol = [x for x in d if x.PdbViolations]
        assert viol and all(not x.Drainable for x in viol)
        names = {v.Name for x in viol for v in x.PdbViolations}
        assert any(n.split("/")[1].startswith("c-") for n in names) and any(n.split("/")[1].startswith("a-") for n in names)
        for x in d:
            for v in x.PdbViolations:
                assert v.Allowed == 0 and v.Evicted > 0
        sd = sim.PlanScaleDown(max_remove=8)
        # the sweep drops the nodes whose drain violates a PDB from the order; every prefix of the plan is PDB-clean
        swept = {w.Node: w for w in sd.Sweep}
        assert set(sd.Order) <= set(base_sd.Order)
        assert all(swept[nm].PdbViolated == 0 for nm in sd.Order) and any(w.PdbViolated for w in sd.Sweep)
        assert all(p["n_pdb_violated"] == 0 for p in sd.Prefixes if p["ok"])
        assert len(sd.RemovedNodes) == sum(1 for p in sd.Prefixes if p["ok"])
        mp = sim.PlanMigrations(max_moves=20)
        blocked = {c.pod_recs[q].name for q in range(len(c.pod_recs)) if len(t.pdbs_of(q))}
        assert not any(m.Pod.name in blocked for m in mp.Migrations)
        assert mp.PdbBlocked > 0
