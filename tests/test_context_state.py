"""Context lifetime (simon_api.cu, Validity::drop): which downloads an upload or a run leaves valid, a refused upload that leaves the
context as it was, and data derived from two uploads that a re-upload rebuilds instead of accumulating."""
import ctypes as C
import dataclasses
import os

import numpy as np
import pytest

from util import make_case

HERE = os.path.dirname(os.path.abspath(__file__))
EXAMPLE = os.path.join(HERE, "golden", "reference", "example")
ERR_STATE = -3


def _local_case():
    """demo_1 with the simple and open_local applications: LVM volumes and an HDD device per annotated node, local and ordinary
    classes."""
    from simon_b200.compiler import compile_cluster
    from simon_b200.objects import AppResource, create_cluster_resource_from_cluster_config, get_object_from_yaml_content, \
        get_yaml_content_from_directory
    from simon_b200.simulator import plan
    cluster = create_cluster_resource_from_cluster_config(os.path.join(EXAMPLE, "cluster", "demo_1"))
    apps = [AppResource(a, get_object_from_yaml_content(get_yaml_content_from_directory(os.path.join(EXAMPLE, "application", a))))
            for a in ("simple", "open_local")]
    p = plan(cluster, apps)
    return compile_cluster(p.nodes, p.pods, p.ctx, open_local=True, storage_classes=list(cluster.StorageClasss), local_devices=True)


def _all_pods_pdb(n_pods):
    """One PDB over every pod that allows every disruption (desired 0)."""
    from simon_b200.disruption import PdbTables
    return PdbTables(names=["all"], pod_off=np.arange(n_pods + 1, dtype=np.uint32), pod_pdb=np.zeros(n_pods, np.uint32),
                     desired=np.zeros(1, np.int32))


def _moves(c, out):
    """Every placed pod onto every node."""
    return np.array([(q, g) for q in range(len(out)) if out[q] >= 0 for g in range(c.n_nodes)], np.uint32).reshape(-1, 2)


def _downloads(eng):
    """name -> (return code, arrays written) of every download of the context, each into fresh sentinel-filled arrays."""
    from simon_b200.engine import lib
    L, h, c = lib(), eng.h, eng.c
    P, N, V = len(c.pod_recs), c.n_nodes, c.storage.n_vgs
    K = max(int(c.snap_dims["n_scalars"]), 1)

    def call(fn, *shapes):
        arrs = [np.full(n, 77, t) for n, t in shapes]
        rc = fn(*[a.ctypes.data for a in arrs])
        return rc, arrs

    i64, i32, u32 = np.int64, np.int32, np.uint32
    node6 = [(N, i64)] * 5 + [(N, i32)]
    return {
        "results": call(lambda a: L.simon_results_download(h, 0, P, a, None), (P, i32)),
        "state": call(lambda *a: L.simon_state_download(h, *a), *node6),
        "storage_state": call(lambda a: L.simon_storage_state_download(h, a), (max(V * N, 1), i64)),
        "devices_state": call(lambda a: L.simon_devices_state_download(h, a), (N, u32)),
        "pdbs_allowed": call(lambda a: L.simon_pdbs_allowed(h, a), (1, i32)),
        "scenario_storage": call(lambda a, b: L.simon_scenarios_storage_download(h, 0, a, b), (max(V * N, 1), i64), (N, u32)),
        "drain": call(lambda *a: L.simon_drain_download(h, 0, *a), (P, u32), (P, i32), (P, u32), (P, i64), (P, u32),
                      (P * 24, u32), (P, u32)),
        "drain_pdb": call(lambda a, b: L.simon_drain_pdb_download(h, 0, a, b), (1, u32), (1, u32)),
        "plan": call(lambda a, b: L.simon_moves_plan_download(h, a, b), (P, i32), (P, u32)),
        "plan_state": call(lambda *a: L.simon_moves_plan_state_download(h, *a), *node6, (K * N, i64), (8 * N, i64)),
        "move_slots": call(lambda a: L.simon_moves_gpu_slots_download(h, 0, len(eng._moves_keep), a), (len(eng._moves_keep), u32)),
    }


def _prime(c):
    """An engine holding every kind of data: a placement, a PDB table, a drain batch, a storage batch, a move list, a plan and a
    move run with GPU share in its scope.  -> (engine, placement, drain node lists)."""
    from simon_b200 import abi
    from simon_b200.engine import Engine
    eng = Engine(c, device=0)
    out = eng.schedule()[0]
    eng.pdbs_upload(_all_pods_pdb(len(out)))
    remain = [np.arange(1, c.n_nodes, dtype=np.uint32)]
    eng.drain_run(out, remain)
    eng.run_scenarios_local([np.arange(c.n_nodes, dtype=np.uint32)])
    eng.moves_upload(_moves(c, out))
    eng.moves_plan(8)
    eng.moves_set_scope(abi.MOVES_SCOPE_GPU_SHARE)
    eng.moves_run(want_gpu_slots=True)
    return eng, out, remain


def _upload(eng, fn, struct):
    from simon_b200.engine import lib
    eng._check(getattr(lib(), fn)(eng.h, C.byref(struct)))


# the single-scenario pool's downloads: an event that clears or rebuilds the live state changes what they return
LIVE_STATE = {"results", "state", "storage_state", "devices_state"}
ALL = {"results", "state", "storage_state", "devices_state", "pdbs_allowed", "scenario_storage", "drain", "drain_pdb", "plan",
       "plan_state", "move_slots"}

# event -> (what it does to a primed engine, downloads that answer SIMON_ERR_STATE after it, downloads whose contents it changes)
EVENTS = {
    "snapshot_upload": (lambda e, out, remain: _upload(e, "simon_snapshot_upload", e.snap), ALL, set()),
    "pods_upload": (lambda e, out, remain: _upload(e, "simon_pods_upload", e.pods),
                    ALL - {"results", "state"}, {"results", "state"}),
    "storage_upload": (lambda e, out, remain: _upload(e, "simon_storage_upload", e.storage),
                       {"devices_state", "scenario_storage", "pdbs_allowed"}, LIVE_STATE),
    "devices_upload": (lambda e, out, remain: _upload(e, "simon_devices_upload", e.devices),
                       {"scenario_storage", "pdbs_allowed"}, LIVE_STATE),
    "state_reset": (lambda e, out, remain: e.reset(), {"pdbs_allowed"}, LIVE_STATE),
    "drain_run": (lambda e, out, remain: e.drain_run(out, remain), {"scenario_storage"}, LIVE_STATE),
    "scenarios_run_local": (lambda e, out, remain: e.run_scenarios_local([np.arange(e.c.n_nodes, dtype=np.uint32)]), set(), set()),
    "moves_upload": (lambda e, out, remain: e.moves_upload(e._moves_keep), {"move_slots"}, set()),
    "moves_replay": (lambda e, out, remain: e.moves_replay(2), {"move_slots"}, set()),
    "moves_plan": (lambda e, out, remain: e.moves_plan(8), {"move_slots"}, set()),
    "pdbs_upload": (lambda e, out, remain: e.pdbs_upload(_all_pods_pdb(len(out))), set(), set()),
}


@pytest.mark.gpu
@pytest.mark.parametrize("event", list(EVENTS))
def test_each_event_drops_exactly_its_table_row(event):
    """After each event, every download whose data it dropped answers SIMON_ERR_STATE; every other one answers 0 with the arrays it
    gave before (or, for the live-state downloads of an event that clears or rebuilds the live state, answers 0).  simon_moves_run
    answers SIMON_ERR_STATE exactly when the event dropped the move list."""
    from simon_b200 import abi
    from simon_b200.engine import lib
    c = _local_case()
    assert c.storage.devices and c.storage.class_local.any() and not c.storage.class_local.all()
    eng, out, remain = _prime(c)
    try:
        before = _downloads(eng)
        assert all(rc == 0 for rc, _ in before.values()), {k: rc for k, (rc, _) in before.items()}
        act, dropped, changed = EVENTS[event]
        act(eng, out, remain)
        after = _downloads(eng)
        for name, (rc, arrs) in after.items():
            if name in dropped:
                assert rc == ERR_STATE, f"{event}: {name} answers {rc}, not SIMON_ERR_STATE"
                continue
            assert rc == 0, f"{event}: {name} answers {rc}: {lib().simon_last_error(eng.h).decode()}"
            if name not in changed:
                for a, b in zip(arrs, before[name][1]):
                    np.testing.assert_array_equal(a, b, err_msg=f"{event}: {name} changed")
        res = abi.SimonMovesResult()
        rc = lib().simon_moves_run(eng.h, 0, None, None, None, None, C.byref(res))
        assert rc == (ERR_STATE if event in ("snapshot_upload", "pods_upload") else 0), f"{event}: simon_moves_run answers {rc}"
        if event == "pods_upload":
            # the PDB table went with the pod set: with a new placement there is nothing to count
            eng.schedule()
            a = np.full(1, 77, np.int32)
            assert lib().simon_pdbs_allowed(eng.h, a.ctypes.data) == 0 and a[0] == 77
    finally:
        eng.close()


def _batch_kinds(c, out):
    """kind -> a batch of that kind on an engine whose live placement is `out` (of _local_case()), returning its results: drains and
    waves remove node 0; the joining wave starts from a base without the last node (no pod is bound to it) and joins it."""
    from simon_b200 import scaledown
    P, N = len(out), c.n_nodes
    remain, every = [np.arange(1, N, dtype=np.uint32)], [np.arange(N, dtype=np.uint32)]
    absent = N - 1
    assert not (np.asarray(c.pods["pod_fixed_node"]) == absent).any()
    local = np.asarray(c.storage.class_local)[np.asarray(c.pods["pod_class"])]
    guard, fixed = scaledown.pod_guard(c), np.asarray(c.pods["pod_fixed_node"])
    probe = next(q for q in range(P) if fixed[q] == -1 and guard[q] == -1 and not local[q] and out[q] >= 0)

    def wave(e, joins):
        if joins is None:
            e.wave_begin(out)
        else:
            e.wave_begin(np.where(out == absent, -1, out), np.arange(N) != absent)
        return e.wave_run(remain, joins)
    return {
        "drain_run": lambda e: e.drain_run(out, remain),
        "drain_run_local": lambda e: e.drain_run(out, remain, local=True),
        "wave_run": lambda e: wave(e, None),
        "wave_run_join": lambda e: wave(e, [np.array([absent], np.uint32)]),
        "probe_run": lambda e: e.probe_run(out, [(probe, 2)]),
        "grow_run": lambda e: e.grow_run(out, P // 2, every),
        "scenarios_run_local": lambda e: e.run_scenarios_local(every),
    }


# batch kind -> the downloads its batch serves, and the code each answers right after it (None: simon_wave_commit's own refusals of
# the batch's first scenario)
BATCH_SERVES = {
    "drain_run": {"drain": 0, "drain_pdb": 0},
    "drain_run_local": {"drain": 0, "drain_pdb": 0, "scenario_storage": 0},
    "wave_run": {"drain": 0, "drain_pdb": 0, "wave_join": 0, "wave_commit": None},
    "wave_run_join": {"drain": 0, "drain_pdb": 0, "wave_join": 0, "wave_commit": -1},       # it joined a node: commit_retire only
    "probe_run": {"probe": 0, "scenario_storage": 0},
    "grow_run": {"grow": 0, "scenario_storage": 0},
    "scenarios_run_local": {"scenario_storage": 0},
}
# what a later batch of a kind leaves of an earlier one: a storage batch keeps the drain, probe and grow batches (not a wave batch,
# whose slots it overwrote); every other kind replaces them all
BATCH_KEEPS = {"scenarios_run_local": {"drain", "drain_pdb", "probe", "grow"}}
# batch kind -> its *_times entry point
BATCH_TIMES = {"drain_run": "drain", "drain_run_local": "drain", "wave_run": "drain", "wave_run_join": "drain", "probe_run": "probe",
               "grow_run": "grow"}


def _batch_answers(eng):
    """download -> return code of every batch download of scenario 0, and simon_wave_commit last (a commit that succeeds ends the
    wave batch)."""
    from simon_b200.engine import lib
    L, h = lib(), eng.h
    return {
        "drain": L.simon_drain_download(h, 0, *[None] * 7),
        "drain_pdb": L.simon_drain_pdb_download(h, 0, None, None),
        "wave_join": L.simon_wave_join_download(h, 0, *[None] * 6),
        "probe": L.simon_probe_download(h, 0, *[None] * 4),
        "grow": L.simon_grow_download(h, 0, *[None] * 5),
        "scenario_storage": L.simon_scenarios_storage_download(h, 0, None, None),
        "wave_commit": L.simon_wave_commit(h, 0),
    }


def _batch_times(eng):
    from simon_b200.engine import lib
    out = {}
    for name in ("drain", "probe", "grow"):
        su, pm = C.c_float(0), C.c_float(0)
        eng._check(getattr(lib(), f"simon_{name}_times")(eng.h, C.byref(su), C.byref(pm)))
        out[name] = (su.value, pm.value)
    return out


@pytest.mark.gpu
def test_batch_downloads_and_times_after_each_pair_of_batch_kinds():
    """For every ordered pair of batch kinds, a batch of the first then one of the second: each batch download answers as the second
    batch leaves it (BATCH_SERVES, BATCH_KEEPS, SIMON_ERR_STATE otherwise), and the *_times entry points of the kinds the second
    batch is not keep the values the first batch left."""
    from simon_b200.engine import Engine
    c = _local_case()
    wrong = []
    with Engine(c, device=0) as eng:
        out = eng.schedule()[0]
    kinds = _batch_kinds(c, out)

    def served(kind, res, d):
        code = BATCH_SERVES[kind][d]
        if code is None:
            r = res[0]
            code = 0 if r["n_unscheduled"] == r["n_blocked"] == r["n_pdb_violated"] == 0 else -1
        return code
    for first in kinds:
        for second in kinds:
            with Engine(c, device=0) as eng:
                eng.schedule()
                res1 = kinds[first](eng)
                t1 = _batch_times(eng)
                res2 = kinds[second](eng)
                t2 = _batch_times(eng)
                got = _batch_answers(eng)
            for d, rc in got.items():
                if d in BATCH_SERVES[second]:
                    want = served(second, res2, d)
                elif d in BATCH_SERVES[first] and d in BATCH_KEEPS.get(second, ()):
                    want = served(first, res1, d)
                else:
                    want = ERR_STATE
                if rc != want:
                    wrong.append(f"{first} then {second}: {d} answers {rc}, not {want}")
            for name in t1:
                if name != BATCH_TIMES.get(second) and t2[name] != t1[name]:
                    wrong.append(f"{first} then {second}: simon_{name}_times changed from {t1[name]} to {t2[name]}")
    assert not wrong, "\n".join(wrong)


GPU_CASE = ("c3", dict(n_nodes=400, n_workloads=80, replicas=10, n_apps=2, seed_no=21, gpu_pct=25))


@pytest.mark.gpu
def test_a_new_upload_of_the_same_cluster_drops_the_move_list():
    """Same snapshot and pod set uploaded again after a move run with GPU share: the move list is gone (simon_moves_run and
    simon_moves_gpu_slots_download answer SIMON_ERR_STATE) until the next simon_moves_upload, which then scores as a fresh context."""
    from simon_b200 import abi
    from simon_b200.engine import Engine, lib
    _p, c = make_case(GPU_CASE[0], **GPU_CASE[1])

    def scored(eng, mv):
        eng.moves_upload(mv)
        eng.moves_set_scope(abi.MOVES_SCOPE_GPU_SHARE)
        return eng.moves_run(k=16, want_per_pod=True, want_gpu_slots=True)

    with Engine(c, device=0) as eng, Engine(c, device=0) as fresh:
        out = eng.schedule()[0]
        from simon_b200 import moves as M
        mv = M.sample_moves(len(out), c.n_nodes, 20000, seed=3, placement=out)
        scored(eng, mv)
        _upload(eng, "simon_snapshot_upload", eng.snap)
        _upload(eng, "simon_pods_upload", eng.pods)
        eng.schedule()
        res = abi.SimonMovesResult()
        assert lib().simon_moves_run(eng.h, 0, None, None, None, None, C.byref(res)) == ERR_STATE
        slots = np.zeros(len(mv), np.uint32)
        assert lib().simon_moves_gpu_slots_download(eng.h, 0, len(mv), slots.ctypes.data) == ERR_STATE
        got = scored(eng, mv)
        fresh.schedule()
        want = scored(fresh, mv)
        assert want["gpu_slots"].any()
        for key in ("gain", "code", "best_per_pod", "gpu_slots"):
            np.testing.assert_array_equal(got[key], want[key], err_msg=key)
        assert (got["best_key"], got["n_feasible"], got["topk"]) == (want["best_key"], want["n_feasible"], want["topk"])


@pytest.mark.gpu
def test_a_refused_pod_upload_leaves_the_context_unchanged():
    """A pod set past the entry limit is refused with SIMON_ERR_LIMIT before anything changes: the earlier pod set still schedules,
    scores moves and downloads its state exactly as a fresh context of it does."""
    from simon_b200 import abi
    from simon_b200.engine import Engine, lib
    from test_engine_limits import compiled, entries32
    _p, c = compiled(*entries32())
    _p, bad = compiled(*entries32(n_ports=33))
    _snap, bad_pods, bad_keep = abi.marshal(bad)

    def run(eng):
        out = eng.schedule()
        eng.moves_upload(_moves(c, out[0]))
        return out, eng.moves_run(k=8, want_per_pod=True), eng.state()

    with Engine(c, device=0) as eng, Engine(c, device=0) as fresh:
        run(eng)
        assert lib().simon_pods_upload(eng.h, C.byref(bad_pods)) == -4
        assert "entries exceed" in lib().simon_last_error(eng.h).decode()
        # the move list and the live state of the earlier pod set, then a new placement of it from the empty state
        moves, state = eng.moves_run(k=8, want_per_pod=True), eng.state()
        eng.reset()
        got, want = (eng.schedule(), moves, state), run(fresh)
        for a, b in zip(got[0], want[0]):
            np.testing.assert_array_equal(a, b)
        for key in ("gain", "code", "best_per_pod"):
            np.testing.assert_array_equal(got[1][key], want[1][key], err_msg=key)
        for key in want[2]:
            np.testing.assert_array_equal(got[2][key], want[2][key], err_msg=key)


@pytest.mark.gpu
def test_a_storage_reupload_replaces_the_local_classes():
    """A storage table that flags one more (ordinary, movable) class as local, then the original table again: the class's moves get
    the codes and gains of a fresh context with the original table, and placements are the fresh context's."""
    from simon_b200 import abi
    from simon_b200.engine import Engine
    c = _local_case()
    with Engine(c, device=0) as fresh:
        out = fresh.schedule()[0]
        mv = _moves(c, out)
        fresh.moves_upload(mv)
        want = fresh.moves_run()
    pod_class = np.asarray(c.pods["pod_class"])
    movable = [k for k in np.unique(pod_class[mv[:, 0]]) if not c.storage.class_local[k]
               and not (want["code"][pod_class[mv[:, 0]] == k] & abi.MOVE_NOT_MOVABLE).all()]
    assert movable, "the case needs an ordinary class with movable pods"
    k = int(movable[0])
    flagged = dataclasses.replace(c.storage, class_local=c.storage.class_local.copy())
    flagged.class_local[k] = 1
    st, keep = abi.marshal_storage(flagged)
    with Engine(c, device=0) as eng:
        for table, devices in ((st, eng.devices), (eng.storage, eng.devices)):
            _upload(eng, "simon_storage_upload", table)
            _upload(eng, "simon_devices_upload", devices)
        got_out = eng.schedule()
        eng.moves_upload(mv)
        got = eng.moves_run()
    with Engine(c, device=0) as fresh:
        want_out = fresh.schedule()
    sel = pod_class[mv[:, 0]] == k
    np.testing.assert_array_equal(got["code"][sel], want["code"][sel])
    np.testing.assert_array_equal(got["gain"][sel], want["gain"][sel])
    np.testing.assert_array_equal(got["code"], want["code"])
    np.testing.assert_array_equal(got["gain"], want["gain"])
    for a, b in zip(got_out, want_out):
        np.testing.assert_array_equal(a, b)
