"""Drain and headroom-probe kernels at several node slots per thread, and the phase-timer variants, against the CPU checkers.

The drain and probe kernels (simon_drain_kernel_*, simon_drain_local_kernel_*, simon_probe_kernel_*, simon_probe_local_kernel_*) run
their node-slot loops with run-time slot counts.  Their variant tests use 40- and 120-node clusters, where a thread holds at most one
node, but production batches on 10,000 nodes run at 2 to 4 slots per thread.  Here each of them, the
large-cluster ones included, runs at two forced geometries of 2 or more slots on the 1,200-node dense mix
(test_zz_kernel_variants_gpu._dense) or on a 1,000-node Open-Local mixed cluster with devices (test_open_local_oracle.make_mixed_local),
and every drain and probe is compared with the drain and probe checkers (tests/checkers.c).  The 256-thread and large-cluster kernels
also run at 16 or more slots on one CTA.  The 320-thread kernels run at 4 slots on one CTA, and the 384-thread ones at 3 on one CTA
(Open-Local) or 2 on two (dense: one CTA's shared memory does not hold 1,200 nodes at 352 threads).  8 slots at 257 or more threads
would need more than 2,000 node slots in one CTA.  The checkers' answers do not depend on the geometry, so each family's are computed once.

A 10,000-node C3 batch runs in the engine's own geometry, with more scenarios than the device holds at once, and a sample of it is
compared with the checkers.

The phase-timer variants (simon_prof_kernel_*, SIMON_PROFILE=1, which launch() reads once per process) run in a child process, each
at the family and geometry of test_zz_kernel_variants_gpu.VARIANTS for the same threads and slots, compared with the oracle as
assert_matches_oracle compares.  The child also runs two launches no timer variant exists for: a 5,600-node C3 in its natural
384-thread geometry and an Open-Local placement.  These must fall back to the variants without timers.  The file sorts after the
rest of the suite."""
import functools
import json
import os
import subprocess
import sys
import time

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if __name__ == "__main__":                      # the phase-timer child (see _prof_child): the paths conftest.py gives the suite
    ROOT = os.path.dirname(HERE)
    for p in (os.path.join(ROOT, "open-simulator_b200"), ROOT, HERE):
        if p not in sys.path:
            sys.path.insert(0, p)

from simon_b200 import abi, headroom, scaledown  # noqa: E402
from util import compiled_kernels  # noqa: E402

THREADS = min(16, len(os.sched_getaffinity(0)))

# kernel -> (cluster family, [(CTAs per scenario, threads per CTA, force_large, node slots per thread)]).  Slots: ceil(nodes / (CTAs x
# threads)), nodes = the most nodes a scenario keeps (drains: N - 1, probes: N) on 1,200 (dense) or 1,000 (local) nodes.
SLOT_GEOMETRIES = {
    "simon_drain_kernel_256": ("dense", [(2, 160, False, 4), (1, 64, False, 19)]),
    "simon_drain_kernel_320": ("dense", [(2, 288, False, 3), (1, 320, False, 4)]),
    "simon_drain_kernel_384": ("dense", [(2, 352, False, 2), (2, 384, False, 2)]),
    "simon_drain_kernel_big": ("dense", [(2, 160, True, 4), (1, 64, True, 19)]),
    "simon_probe_kernel_256": ("dense", [(2, 160, False, 4), (1, 64, False, 19)]),
    "simon_probe_kernel_320": ("dense", [(2, 288, False, 3), (1, 320, False, 4)]),
    "simon_probe_kernel_384": ("dense", [(2, 352, False, 2), (2, 384, False, 2)]),
    "simon_probe_kernel_big": ("dense", [(2, 160, True, 4), (1, 64, True, 19)]),
    "simon_drain_local_kernel_256": ("local", [(2, 128, False, 4), (1, 64, False, 16)]),
    "simon_drain_local_kernel_320": ("local", [(2, 288, False, 2), (1, 288, False, 4)]),
    "simon_drain_local_kernel_384": ("local", [(2, 352, False, 2), (1, 352, False, 3)]),
    "simon_drain_local_kernel_big": ("local", [(2, 160, True, 4), (1, 64, True, 16)]),
    "simon_probe_local_kernel_256": ("local", [(2, 128, False, 4), (1, 64, False, 16)]),
    "simon_probe_local_kernel_320": ("local", [(2, 288, False, 2), (1, 288, False, 4)]),
    "simon_probe_local_kernel_384": ("local", [(2, 352, False, 2), (1, 352, False, 3)]),
    "simon_probe_local_kernel_big": ("local", [(2, 160, True, 4), (1, 64, True, 16)]),
}
# one geometry per family and batch kind also runs without the static-verdict cache
NO_STATIC_CACHE = {("simon_drain_kernel_256", 1, 64), ("simon_probe_kernel_256", 1, 64),
                   ("simon_drain_local_kernel_320", 1, 288), ("simon_probe_local_kernel_320", 1, 288)}
ENTRIES = [(k, fam, cs, t, big, slots, sc) for k, (fam, geoms) in SLOT_GEOMETRIES.items() for cs, t, big, slots in geoms
           for sc in ((True, False) if (k, cs, t) in NO_STATIC_CACHE else (True,))]


def _ids(entries):
    return [f"{k[6:]}-{cs}x{t}" + ("" if sc else "-no_static_cache") for k, _fam, cs, t, _big, _slots, sc in entries]


DRAIN_ENTRIES = [e for e in ENTRIES if "_drain_" in e[0]]
PROBE_ENTRIES = [e for e in ENTRIES if "_probe_" in e[0]]


def _prof_variants():
    """Timer variant -> (family, [(CTAs, threads, force_large)]) of the default variant of the same threads and slots in
    test_zz_kernel_variants_gpu.VARIANTS: simon_prof_kernel_<t>_<s> runs where simon_place_kernel_<t>_<s> is checked."""
    from test_zz_kernel_variants_gpu import VARIANTS
    return {"simon_prof_kernel_" + k[len("simon_place_kernel_"):]: VARIANTS[k] for k in VARIANTS
            if k.startswith(("simon_place_kernel_256_", "simon_place_kernel_320_"))}


# ---- CPU ----------------------------------------------------------------------------------------------------------------------

def test_slot_table_names_every_drain_and_probe_kernel():
    names = set()
    for prefix in ("simon_drain_kernel_", "simon_drain_local_kernel_", "simon_probe_kernel_", "simon_probe_local_kernel_"):
        names |= compiled_kernels(prefix)
    assert len(names) == 16 and set(SLOT_GEOMETRIES) == names, sorted(names ^ set(SLOT_GEOMETRIES))
    for k, (_fam, geoms) in SLOT_GEOMETRIES.items():
        assert len({(cs, t) for cs, t, *_ in geoms}) >= 2 and all(s >= 2 for *_, s in geoms), k
        if k.endswith(("_256", "_big")):
            assert max(s for *_, s in geoms) >= 8, k


def test_timer_table_names_every_timer_variant():
    """Fails when simon_kernel.cu gains a phase-timer variant whose (threads, slots) no default variant of VARIANTS covers."""
    prof = _prof_variants()
    assert set(prof) == compiled_kernels("simon_prof_kernel_"), sorted(set(prof) ^ compiled_kernels("simon_prof_kernel_"))
    assert len(prof) == 10


# ---- cluster families and the checkers' answers -----------------------------------------------------------------------------

@functools.lru_cache(maxsize=None)
def family(name):
    if name == "dense":
        from test_zz_kernel_variants_gpu import family as kv_family
        return kv_family("dense")
    if name == "local":
        from test_open_local_oracle import make_mixed_local
        return make_mixed_local(71, n_nodes=1000, n_workloads=200, max_replicas=8)[1]
    raise KeyError(name)


def _oracle(c):
    from oracle.binding import Oracle
    return Oracle(c, threads=THREADS, open_local=getattr(c, "storage", None) is not None)


def _drain_set(c, placed, rng, n_single, n_multi):
    """Single-node drains of n_single nodes that hold scheduler-placed pods (GPU-share nodes among them), and n_multi multi-node
    drains whose removed nodes lie inside the node order, so that every later node moves to another slot: a run of 40 from the
    middle, every fifth node of the first half, a random set of the first two thirds, two neighbours near the front, every node with
    GPU-share devices in the first 90 % of the order (GPU-share pods then find no node), and random sets."""
    n = c.n_nodes
    free = c.pods["pod_fixed_node"] == -1
    used = np.unique(placed[free & (placed >= 0)])
    gpu = np.intersect1d(used, np.nonzero(c.snap["gpu_count"] > 0)[0])
    k_gpu = min(len(gpu), n_single // 4)
    single = rng.choice(gpu, k_gpu, replace=False).tolist() + \
        rng.choice(np.setdiff1d(used, gpu), n_single - k_gpu, replace=False).tolist()
    gpu_front = np.nonzero(c.snap["gpu_count"][: (9 * n) // 10] > 0)[0].tolist()
    multi = [list(range(n // 3, n // 3 + 40)), list(range(0, n // 2, 5)), rng.choice((2 * n) // 3, 60, replace=False).tolist(),
             [1, 2], gpu_front]
    while len(multi) < n_multi:
        lo = int(rng.integers(0, n // 2))
        multi.append(rng.choice(np.arange(lo, lo + n // 3), int(rng.integers(2, 30)), replace=False).tolist())
    return [[int(g)] for g in single] + [[int(g) for g in m] for m in multi[:n_multi]]


def _occupancy(c, st, rl):
    idx = np.asarray(rl, dtype=np.int64)
    return dict(req_mcpu=int(st["req_mcpu"][idx].sum()), req_mem=int(st["req_mem"][idx].sum()),
                alloc_mcpu=int(c.snap["alloc_mcpu"][idx].sum()), alloc_mem=int(c.snap["alloc_mem"][idx].sum()))


def _vg_sums(c, vg, rl):
    st = c.storage
    req = cap = 0
    for x in rl:
        nv = int(st.node_n_vg[x])
        if nv >= 0:
            req += int(vg[:nv, x].sum())
            cap += int(st.vg_capacity[:nv, x].sum())
    return req, cap


def checker_drains(c, placed, drains):
    """The drain checker on a fresh oracle: per drain the checker's result, its occupancy sums and, with Open-Local, the VG sums
    and the VG and device state; -> (remaining-node lists, answers, the live VG and device state)."""
    import checkers
    local = getattr(c, "storage", None) is not None
    order = scaledown.NodeOrder(c)
    remain = [order.remaining(d) for d in drains]
    o = _oracle(c)
    try:
        np.testing.assert_array_equal(o.schedule()[0], placed)
        live = o.storage_state() if local else None
        wants = []
        for rl in remain:
            w = checkers.drain(o, placed, rl)
            w.update(_occupancy(c, o.state(), rl))
            if local:
                vg, dev = o.storage_state()
                w["vg_requested"], w["vg_capacity"] = _vg_sums(c, vg, rl)
                w["vg_state"], w["dev_state"] = vg, dev
            wants.append(w)
    finally:
        o.close()
    return remain, wants, live


def checker_probes(c, placed, probes):
    """The probe checker on a fresh oracle: per probe the checker's result, the request sums over every node and, with Open-Local,
    the VG sum and the VG and device state."""
    import checkers
    local = getattr(c, "storage", None) is not None
    o = _oracle(c)
    try:
        np.testing.assert_array_equal(o.schedule()[0], placed)
        wants = []
        for q, r in probes:
            w = checkers.probe(o, placed, q, r)
            st = o.state()
            w.update(req_mcpu=int(st["req_mcpu"].sum()), req_mem=int(st["req_mem"].sum()))
            if local:
                vg, dev = o.storage_state()
                w["vg_requested"] = _vg_sums(c, vg, range(c.n_nodes))[0]
                w["vg_state"], w["dev_state"] = vg, dev
            wants.append(w)
    finally:
        o.close()
    return wants


def _probe_set(c, placed, rng, n_few, n_capped, n_local=0):
    """n_few probes of 1-11 replicas and n_capped probes capped at the free pod slots (the session's default cap, which no probe of
    these families reaches).  With n_local: that many of the few-replica probes of classes with Open-Local volumes, the rest without."""
    from test_zz_headroom_gpu import _probe_pods
    free = headroom.free_pod_slots(c, placed)
    qs = _probe_pods(c, rng, 400)
    if n_local:
        loc = c.storage.class_local[c.pods["pod_class"][qs]].astype(bool)
        few = [q for q, x in zip(qs, loc) if x][:n_local] + [q for q, x in zip(qs, loc) if not x][:n_few - n_local]
    else:
        few = qs[:n_few]
    capped = [q for q in qs if q not in few][:n_capped]
    return [(q, int(rng.integers(1, 12))) for q in few] + [(q, free) for q in capped], len(few)


@functools.lru_cache(maxsize=None)
def checked(name):
    """The family's live placement (the oracle's), its drains and probes, and the checkers' answers for them."""
    c = family(name)
    from test_zz_kernel_variants_gpu import oracle_run
    t0 = time.perf_counter()
    if name == "dense":
        placed = oracle_run("dense")[0]
    else:
        o = _oracle(c)
        placed = o.schedule()[0]
        o.close()
    rng = np.random.default_rng(29)
    drains = _drain_set(c, placed, rng, n_single=24, n_multi=8)
    remain, dwants, live = checker_drains(c, placed, drains)
    probes, n_few = _probe_set(c, placed, rng, 10, 4, n_local=6 if name == "local" else 0)
    pwants = checker_probes(c, placed, probes)
    print(f"{name}: {c.n_nodes} nodes, {len(placed)} pods, checker answers for {len(drains)} drains and {len(probes)} probes in "
          f"{time.perf_counter() - t0:.1f} s")
    return dict(c=c, placed=placed, drains=drains, remain=remain, dwants=dwants, live=live, probes=probes, n_few=n_few, pwants=pwants)


def _engine(c, **kw):
    from simon_b200.engine import Engine
    return Engine(c, device=0, **kw)


# kernel -> the (CTAs, threads, node slots) it ran at, for the summary test at the end
_RAN = {}


def _assert_launch(li, kernel, cs, t, big, slots, n):
    assert (li["kernel"], li["cluster_ctas"], li["threads_per_cta"], li["large"], li["node_slots"], li["n_scenarios"]) == \
        (kernel, cs, t, big, slots, n), li
    assert li["node_slots"] >= 2, li
    _RAN.setdefault(kernel, set()).add((cs, t, li["node_slots"]))


# ---- GPU: forced multi-slot geometries ----------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("kernel,fam,cs,t,big,slots,static_cache", DRAIN_ENTRIES, ids=_ids(DRAIN_ENTRIES))
def test_drain_kernel_at_several_slots_matches_checker(kernel, fam, cs, t, big, slots, static_cache):
    from test_drain import _assert_drain_equal
    k = checked(fam)
    c, placed, drains, remain = k["c"], k["placed"], k["drains"], k["remain"]
    local = fam == "local"
    with _engine(c, record_scores=True, cluster_ctas=cs, threads_per_cta=t, force_large=big, static_cache=static_cache) as eng:
        got = eng.drain_run(placed, remain, local=local)
        assert eng.last_drain["chunks"] == 1
        _assert_launch(eng.last_launch(), kernel, cs, t, big, slots, len(drains))
        states = [eng.scenario_storage_state(i) for i in range(len(drains))] if local else None
    moved = 0
    for j, (d, rl, g, w) in enumerate(zip(drains, remain, got, k["dwants"])):
        what = f"{kernel} {cs}x{t} static_cache={static_cache} drain {d if len(d) < 6 else f'of {len(d)} nodes'}"
        _assert_drain_equal(g, w, what)
        np.testing.assert_array_equal(g["score"], w["score"], err_msg=f"{what}: scores")
        for key in ("req_mcpu", "req_mem", "alloc_mcpu", "alloc_mem"):
            assert g[key] == w[key], (what, key, g[key], w[key])
        if local:
            assert (g["vg_requested"], g["vg_capacity"]) == (w["vg_requested"], w["vg_capacity"]), what
            rl = np.asarray(rl)
            gone = np.setdiff1d(np.arange(c.n_nodes), rl)
            bvg, bdev = states[j]
            np.testing.assert_array_equal(bvg[:, rl], w["vg_state"][:, rl], err_msg=f"{what}: VG state")
            np.testing.assert_array_equal(bdev[rl], w["dev_state"][rl], err_msg=f"{what}: device state")
            np.testing.assert_array_equal(bvg[:, gone], k["live"][0][:, gone], err_msg=f"{what}: removed nodes' VG state")
            np.testing.assert_array_equal(bdev[gone], k["live"][1][gone], err_msg=f"{what}: removed nodes' device state")
            moved += sum(1 for q in g["evicted"].tolist() if c.storage.class_local[int(c.pods["pod_class"][q])])
    # the batch moved pods, some of them with GPU share (and Open-Local volumes), and some found no node
    assert sum(g["n_placed"] for g in got) > 100 and any(g["n_unscheduled"] for g in got)
    assert any((g["gpu_slots"] != 0).any() for g in got)
    assert not local or moved > 0


@pytest.mark.gpu
@pytest.mark.parametrize("kernel,fam,cs,t,big,slots,static_cache", PROBE_ENTRIES, ids=_ids(PROBE_ENTRIES))
def test_probe_kernel_at_several_slots_matches_checker(kernel, fam, cs, t, big, slots, static_cache):
    from test_zz_headroom_gpu import _assert_probe_equal
    k = checked(fam)
    c, placed, probes = k["c"], k["placed"], k["probes"]
    local = fam == "local"
    with _engine(c, record_scores=True, cluster_ctas=cs, threads_per_cta=t, force_large=big, static_cache=static_cache) as eng:
        got = eng.probe_run(placed, probes)
        assert eng.last_probe["chunks"] == 1
        _assert_launch(eng.last_launch(), kernel, cs, t, big, slots, len(probes))
        states = [eng.scenario_storage_state(i) for i in range(len(probes))] if local else None
    for j, ((q, r), g, w) in enumerate(zip(probes, got, k["pwants"])):
        what = f"{kernel} {cs}x{t} static_cache={static_cache} probe {q} x {r}"
        _assert_probe_equal(g, w, what)
        assert (g["req_mcpu"], g["req_mem"]) == (w["req_mcpu"], w["req_mem"]), what
        if j >= k["n_few"]:                                           # capped at the free pod slots: stopped by a replica that failed
            assert g["stop_reason"] == abi.PROBE_STOP_UNSCHEDULABLE and g["fail_counts"].sum() > 0, what
        if local:
            assert g["vg_requested"] == w["vg_requested"], what
            np.testing.assert_array_equal(states[j][0], w["vg_state"], err_msg=f"{what}: VG state")
            np.testing.assert_array_equal(states[j][1], w["dev_state"], err_msg=f"{what}: device state")
    assert {g["stop_reason"] for g in got} == {abi.PROBE_STOP_UNSCHEDULABLE, abi.PROBE_STOP_MAX_REPLICAS}
    assert any((g["gpu_slots"] != 0).any() for g in got)
    if local:
        cls_local = c.storage.class_local[c.pods["pod_class"]]
        assert any(cls_local[q] and g["n_placed"] for (q, _r), g in zip(probes, got))
        assert any(not cls_local[q] and g["n_placed"] for (q, _r), g in zip(probes, got))


@pytest.mark.gpu
def test_zz_every_drain_and_probe_kernel_ran_at_multi_slot_geometries():
    """Runs after the two matrices above: every kernel of the table ran at two or more geometries of 2 or more slots, and the
    256-thread and large-cluster ones at 8 or more."""
    if set(_RAN) != set(SLOT_GEOMETRIES):
        pytest.skip("runs after the whole matrix of this module")
    for kernel, geoms in sorted(_RAN.items()):
        assert len(geoms) >= 2 and min(s for *_, s in geoms) >= 2, (kernel, geoms)
        if kernel.endswith(("_256", "_big")):
            assert max(s for *_, s in geoms) >= 8, (kernel, geoms)
        print(f"{kernel}: {sorted(geoms)} (CTAs, threads, node slots)")


# ---- GPU: the engine's own geometry at production size ------------------------------------------------------------------------

@pytest.mark.gpu
def test_production_batches_10000_nodes_in_the_engines_geometry():
    """C3 on 10,000 nodes with GPU share on a quarter of them (test_zz_kernel_variants_gpu's c3_10000_batch): 64 drains and 32
    probes of up to 64 replicas, each batch in one launch of the geometry the engine picks for it.  That geometry holds each
    scenario in 2 or more node slots per thread, and the batch has more CTAs than the device has SMs (one CTA per SM at this shared
    memory), so its scenarios run in several waves.  12 drains and 8 probes are compared with the checkers."""
    import checkers
    import torch
    from test_drain import _assert_drain_equal
    from test_zz_headroom_gpu import _assert_probe_equal, _probe_pods
    from test_zz_kernel_variants_gpu import family as kv_family, oracle_run
    c = kv_family("c3_10000_batch")
    t0 = time.perf_counter()
    placed = oracle_run("c3_10000_batch")[0]
    t_live = time.perf_counter() - t0
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    rng = np.random.default_rng(37)
    drains = _drain_set(c, placed, rng, n_single=58, n_multi=6)
    order = scaledown.NodeOrder(c)
    remain = [order.remaining(d) for d in drains]
    qs = _probe_pods(c, rng, 32)
    probes = [(q, int(rng.integers(1, 65))) for q in qs]
    with _engine(c, record_scores=True) as eng:
        got = eng.drain_run(placed, remain)
        dli = eng.last_launch()
        assert eng.last_drain["chunks"] == 1 and len(drains) == 64
        gotp = eng.probe_run(placed, probes)
        pli = eng.last_launch()
        assert eng.last_probe["chunks"] == 1 and len(probes) == 32
    for li, n in ((dli, len(drains)), (pli, len(probes))):
        assert not li["large"] and li["node_slots"] >= 2 and li["n_scenarios"] == n, li
        assert li["n_scenarios"] * li["cluster_ctas"] > n_sms, (li, n_sms)
    assert dli["kernel"].startswith("simon_drain_kernel_") and pli["kernel"].startswith("simon_probe_kernel_")
    sample = list(range(0, 58, 6)) + [58, 62]                        # 10 single-node drains, 2 multi-node ones
    o = _oracle(c)
    t0 = time.perf_counter()
    try:
        for j in sample:
            w = checkers.drain(o, placed, remain[j])
            _assert_drain_equal(got[j], w, f"drain {j}")
            np.testing.assert_array_equal(got[j]["score"], w["score"], err_msg=f"drain {j}: scores")
            occ = _occupancy(c, o.state(), remain[j])
            assert all(got[j][key] == v for key, v in occ.items()), (j, occ)
    finally:
        o.close()
    t_drains = time.perf_counter() - t0
    o = _oracle(c)
    t0 = time.perf_counter()
    try:
        for j in range(0, 32, 4):
            q, r = probes[j]
            _assert_probe_equal(gotp[j], checkers.probe(o, placed, q, r), f"probe {q} x {r}")
    finally:
        o.close()
    t_probes = time.perf_counter() - t0
    assert sum(got[j]["n_evicted"] for j in sample) > 0 and any((g["gpu_slots"] != 0).any() for g in got)
    assert sum(gotp[j]["n_placed"] for j in range(0, 32, 4)) > 8
    print(f"10,000 nodes: drains {dli['kernel']} {dli['cluster_ctas']} CTAs x {dli['threads_per_cta']} threads x "
          f"{dli['node_slots']} slots x {dli['n_scenarios']} scenarios; probes {pli['kernel']} {pli['cluster_ctas']} x "
          f"{pli['threads_per_cta']} x {pli['node_slots']} x {pli['n_scenarios']}; {n_sms} SMs.  CPU: live placement {t_live:.1f} s, "
          f"{len(sample)} checker drains {t_drains:.1f} s, 8 checker probes {t_probes:.1f} s ({THREADS} oracle threads)")


# ---- GPU: the phase-timer variants, in a child process with SIMON_PROFILE=1 ---------------------------------------------------

def _prof_child(names=None):
    """The child's work: every timer variant at its VARIANTS family and geometry, and the two launches without a timer variant,
    each compared with the oracle (names: only those runs).  -> one record per run: kernel launched, whether timers ran, and the
    first mismatch or error."""
    import traceback
    from test_zz_kernel_variants_gpu import assert_matches_oracle, family as kv_family
    from test_zz_kernel_variants_gpu import _engine as kv_engine
    out = []

    def run(name, fn):
        if names and name not in names:
            return
        rec = dict(name=name, kernel=None, timed=False, error=None)
        try:
            fn(rec)
        except Exception as e:  # noqa: BLE001 - reported to the parent, which fails on it
            rec["error"] = f"{type(e).__name__}: {e}\n{traceback.format_exc(limit=3)}"
        out.append(rec)

    for kernel, (fam, geoms) in sorted(_prof_variants().items()):
        for cs, t, big in geoms:
            def one(rec, kernel=kernel, fam=fam, cs=cs, t=t, big=big):
                with kv_engine(kv_family(fam), cs, t, big, record_scores=True) as eng:
                    out_, score, fc, fp = eng.schedule()
                    rec["kernel"] = eng.last_launch()["kernel"]
                    rec["timed"] = sum(eng.stats()["cycles"].values()) > 0
                    assert_matches_oracle(fam, out_, score, fc, fp, eng, f"{kernel} {fam} {cs}x{t}")
            run(kernel, one)

    def natural_384(rec):                                 # the single run's own geometry: 16 CTAs x 384 threads x 1 slot
        with kv_engine(kv_family("c3_5600"), 0, 0, False, record_scores=True) as eng:
            out_, score, fc, fp = eng.schedule()
            rec["kernel"] = eng.last_launch()["kernel"]
            rec["timed"] = sum(eng.stats()["cycles"].values()) > 0
            assert_matches_oracle("c3_5600", out_, score, fc, fp, eng, "c3_5600 natural geometry")
    run("c3_5600", natural_384)

    def open_local(rec):
        from test_zz_open_local_oracle_gpu import assert_engine_matches, cluster, oracle_full
        with kv_engine(cluster(300, 300), 2, 128, False, record_scores=True) as eng:
            out_, score, fc, fp = eng.schedule()
            rec["kernel"] = eng.last_launch()["kernel"]
            rec["timed"] = sum(eng.stats()["cycles"].values()) > 0
            assert_engine_matches(oracle_full(300, 300), eng, out_, score, fc, fp, "open-local 300 2x128")
    run("open_local_300", open_local)
    return out


@pytest.mark.gpu
def test_timer_variants_match_oracle_in_a_profiling_process():
    """SIMON_PROFILE=1 in a child process (the variable is read once per process): each simon_prof_kernel_* launched and matched
    the oracle with its timers running.  A geometry of 384 threads (the 5,600-node C3's own) and an Open-Local placement have no
    timer variant; they run the variants without timers, which last_launch() names, and match the oracle too."""
    env = dict(os.environ, SIMON_PROFILE="1")
    t0 = time.perf_counter()
    p = subprocess.run([sys.executable, os.path.abspath(__file__)], env=env, cwd=os.path.dirname(HERE), capture_output=True,
                       text=True, timeout=1500)
    assert p.returncode == 0, p.stderr[-4000:]
    recs = {r["name"]: r for r in json.loads(p.stdout.strip().splitlines()[-1])}
    prof = _prof_variants()
    assert set(recs) == set(prof) | {"c3_5600", "open_local_300"}
    for name, r in sorted(recs.items()):
        assert r["error"] is None, f"{name}: {r['error']}"
    for kernel in prof:
        assert recs[kernel]["kernel"] == kernel and recs[kernel]["timed"], recs[kernel]
    assert (recs["c3_5600"]["kernel"], recs["c3_5600"]["timed"]) == ("simon_place_kernel_384_1", False), recs["c3_5600"]
    assert (recs["open_local_300"]["kernel"], recs["open_local_300"]["timed"]) == ("simon_local_kernel_256", False), \
        recs["open_local_300"]
    print(f"timer variants: {len(prof)} compared with the oracle in {time.perf_counter() - t0:.0f} s (child process)")


if __name__ == "__main__":
    print(json.dumps(_prof_child(sys.argv[1:])))
