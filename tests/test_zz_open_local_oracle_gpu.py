"""Every Open-Local kernel path against the CPU oracle with Open-Local (Oracle(c, open_local=True)) on clusters that mix it with
every other plugin (test_open_local_oracle.make_mixed_local): placement with each simon_local_kernel_* variant, the per-node totals
and verdicts of sampled pods, scenario batches (simon_scenarios_run_local), resumed runs (simon_schedule_resume) and drains with
each simon_drain_local_kernel_* variant (simon_drain_run_local, against the drain checker on the storage oracle)."""
import functools
import os

import numpy as np
import pytest

from simon_b200 import scaledown
from test_drain_local import DRAIN_LOCAL_VARIANTS, _drains
from test_open_local_oracle import coverage, make_mixed_local
from test_zz_kernel_variants_gpu import VARIANTS
from util import compiled_kernels

pytestmark = pytest.mark.gpu
THREADS = min(16, len(os.sched_getaffinity(0)))

# kernel -> geometries, and the node count of the cluster family the geometry was chosen for (test_zz_kernel_variants_gpu.py)
LOCAL_ENTRIES = [(k, int(fam.split("_")[1]), cs, t, big) for k, (fam, geoms) in VARIANTS.items()
                 if fam.startswith("local_") for cs, t, big in geoms]
_LAUNCHED = {"place": set(), "drain": set()}
_DECISIONS = []


@functools.lru_cache(maxsize=None)
def cluster(n_nodes, seed):
    return make_mixed_local(seed, n_nodes=n_nodes, n_workloads=max(24, n_nodes // 5), max_replicas=8)[1]


def _oracle(c):
    from oracle.binding import Oracle
    return Oracle(c, threads=THREADS, open_local=True)


@functools.lru_cache(maxsize=None)
def oracle_full(n_nodes, seed):
    """The oracle's full run: (out, score, fail_counts, fail_pod, state, state_ext, slot words, VG state, device state)."""
    o = _oracle(cluster(n_nodes, seed))
    try:
        return o.schedule() + (o.state(), o.state_ext(), o.gpu_slot_words()) + o.storage_state()
    finally:
        o.close()


def _engine(c, **kw):
    from simon_b200.engine import Engine
    return Engine(c, device=0, **kw)


def assert_engine_matches(ref, eng, out, score, fc, fp, what, first=0):
    """A run of pods [first, P) against the oracle's full run ref: nodes, recorded winning scores, failures, the node state, the
    GPU slot words, the VG state and the device masks."""
    rout, rscore, rfc, rfp, rst, rext, rslots, rvg, rdev = ref
    bad = np.nonzero(out[first:] != rout[first:])[0] + first
    assert len(bad) == 0, f"{what}: {len(bad)} placements differ, first pods {bad[:6]}: gpu {out[bad[:6]]} oracle {rout[bad[:6]]}"
    np.testing.assert_array_equal(score[first:], rscore[first:], err_msg=f"{what}: scores")
    keep = rfp >= first
    np.testing.assert_array_equal(fp, rfp[keep], err_msg=f"{what}: failing pods")
    np.testing.assert_array_equal(fc, rfc[keep], err_msg=f"{what}: failure histograms")
    st, ext = eng.state(), eng.state_ext()
    for k in rst:
        np.testing.assert_array_equal(st[k], rst[k], err_msg=f"{what}: {k}")
    for k in rext:
        np.testing.assert_array_equal(ext[k], rext[k], err_msg=f"{what}: {k}")
    np.testing.assert_array_equal(eng.gpu_slot_words(), rslots, err_msg=f"{what}: GPU slots")
    np.testing.assert_array_equal(eng.storage_state(), rvg, err_msg=f"{what}: VG state")
    np.testing.assert_array_equal(eng.device_state(), rdev, err_msg=f"{what}: device state")
    _DECISIONS.append(int((eng.c.pods["pod_fixed_node"][first:] == -1).sum()))


# ---- placement: every local placement kernel ----

@pytest.mark.parametrize("kernel,n_nodes,cs,t,big", LOCAL_ENTRIES, ids=[f"{e[0][6:]}-{e[2]}x{e[3]}" for e in LOCAL_ENTRIES])
def test_local_kernel_matches_storage_oracle(kernel, n_nodes, cs, t, big):
    """Each simon_local_kernel_* at a geometry that launches it, with the pinned fast path on and off and the static-verdict cache
    off, against the oracle with Open-Local: everything a run leaves, compared exactly."""
    c = cluster(n_nodes, n_nodes)
    ref = oracle_full(n_nodes, n_nodes)
    for opts in (dict(pin_fast=True), dict(pin_fast=False), dict(static_cache=False)):
        with _engine(c, record_scores=True, cluster_ctas=cs, threads_per_cta=t, force_large=big, **opts) as eng:
            out, score, fc, fp = eng.schedule()
            li = eng.last_launch()
            assert li["kernel"] == kernel and li["local"] and li["large"] == big, li
            _LAUNCHED["place"].add(li["kernel"])
            assert_engine_matches(ref, eng, out, score, fc, fp, f"{kernel} {cs}x{t} {opts}")
    assert (ref[0] == -1).any()
    assert (ref[7] != c.storage.vg_requested.reshape(ref[7].shape)).any()     # some pods bound volumes


# ---- per-node detail ----

def test_per_node_totals_and_verdicts_of_local_pods():
    """For sampled pods with volumes and several feasible nodes, the engine's per-node verdicts and totals (the normalised
    Open-Local term included, on every node, not only the winner) against the oracle's per-node detail."""
    c = cluster(300, 11)
    P = c.pods_dims["n_pods"]
    local = c.storage.class_local[c.pods["pod_class"]].astype(bool) & (c.pods["pod_fixed_node"] == -1)
    o = _oracle(c)
    o.enable_dump()
    picked = []
    try:
        for i in range(P):
            o.schedule(i, 1)
            if local[i]:
                code, sc = o.last_detail()
                if (code == 0).sum() > 1 and len(set(sc[code == 0, 9].tolist())) > 1:
                    picked.append((i, code.copy(), sc[:, 8].copy()))
    finally:
        o.close()
    assert len(picked) >= 4
    for i, code, tot_ref in picked[::max(1, len(picked) // 6)]:
        with _engine(c) as eng:
            _out, tot, gcode = eng.dump_pod(i)
        feas = code == 0
        np.testing.assert_array_equal(gcode == 0, feas, err_msg=f"pod {i}: feasible sets")
        bad = np.nonzero(feas & (tot != tot_ref))[0]
        assert len(bad) == 0, f"pod {i}: totals differ on nodes {bad[:8]}: gpu {tot[bad[:8]]} oracle {tot_ref[bad[:8]]}"


# ---- scenario batches ----

def test_scenario_batches_match_storage_oracle():
    """simon_scenarios_run_local: each scenario against the oracle reset and restricted to its nodes: nodes, result sums, the VG
    sums over its annotated nodes and its final VG and device state (inactive nodes keep the uploaded state)."""
    c = cluster(300, 21)
    st = c.storage
    rng = np.random.default_rng(5)
    N = c.n_nodes
    scen = [np.arange(N, dtype=np.uint32)]
    for k in (N - 1, N - 20, N // 2, N // 3):
        scen.append(np.sort(rng.choice(N, size=k, replace=False)).astype(np.uint32))
    scen.append(rng.permutation(N)[: N - 5].astype(np.uint32))
    with _engine(c) as eng:
        res, nodes = eng.run_scenarios_local(scen, want_nodes=True)
        states = [eng.scenario_storage_state(i) for i in range(len(scen))]
        assert eng.last_launch()["local"]
    o = _oracle(c)
    try:
        for i, sn in enumerate(scen):
            o.reset()
            o.set_active(sn)
            out = o.schedule()[0]
            np.testing.assert_array_equal(nodes[i], out, err_msg=f"scenario {i}")
            assert res[i]["n_unscheduled"] == int((out == -1).sum()), i
            s = o.state()
            assert res[i]["req_mcpu"] == int(s["req_mcpu"][sn].sum()) and res[i]["req_mem"] == int(s["req_mem"][sn].sum()), i
            vg, dev = o.storage_state()
            req = cap = 0
            for g in sn.tolist():
                nv = int(st.node_n_vg[g])
                if nv >= 0:
                    req += int(vg[:nv, g].sum())
                    cap += int(st.vg_capacity[:nv, g].sum())
            assert (res[i]["vg_requested"], res[i]["vg_capacity"]) == (req, cap), i
            bvg, bdev = states[i]
            np.testing.assert_array_equal(bvg[:, sn], vg[:, sn], err_msg=f"scenario {i}: VG state")
            np.testing.assert_array_equal(bdev[sn], dev[sn], err_msg=f"scenario {i}: device state")
            off = np.setdiff1d(np.arange(N), sn)
            np.testing.assert_array_equal(bvg[:, off], st.vg_requested[:, off])
            np.testing.assert_array_equal(bdev[off], st.dev_alloc[off])
    finally:
        o.close()


# ---- resumed runs ----

@pytest.mark.parametrize("n_nodes,seed", [(300, 31), (700, 32)])
def test_resume_from_the_oracle_prefix(n_nodes, seed):
    """simon_schedule_resume from the oracle's first half (the Bind replay of the prefix's volumes) and from an empty prefix: the
    rest's nodes, scores and failures, the node state, GPU slots, VG state and device masks."""
    c = cluster(n_nodes, seed)
    ref = oracle_full(n_nodes, seed)
    P = c.pods_dims["n_pods"]
    with _engine(c, record_scores=True) as eng:
        for h in (P // 2, 0):
            out, score, fc, fp = eng.schedule_resume(ref[0][:h])
            assert eng.last_launch()["local"]
            assert_engine_matches(ref, eng, out, score, fc, fp, f"resume from {h}", first=h)


# ---- drains ----

@pytest.mark.parametrize("kernel", sorted(DRAIN_LOCAL_VARIANTS))
def test_drain_local_kernel_matches_storage_oracle(kernel):
    """simon_drain_run_local with each drain-local kernel, from the oracle's full placement (the engine's own), against
    The drain checker on the oracle with Open-Local (local volumes move, so class_local is not passed): the evicted pods, their
    nodes, scores, GPU slots and failures, the VG sums over the remaining annotated nodes, and each drain's VG and device state
    (remaining nodes: the drain oracle's; removed nodes: the live state)."""
    import checkers
    cs, t, big = DRAIN_LOCAL_VARIANTS[kernel]
    n_nodes, seed = 120, 41 + sorted(DRAIN_LOCAL_VARIANTS).index(kernel)
    c = cluster(n_nodes, seed)
    st = c.storage
    ref = oracle_full(n_nodes, seed)
    placed = ref[0]
    with _engine(c) as eng:
        np.testing.assert_array_equal(eng.schedule()[0], placed)
    order = scaledown.NodeOrder(c)
    drains = _drains(c, np.random.default_rng(seed), n_single=12, n_multi=4)
    remain = [order.remaining(d) for d in drains]
    with _engine(c, record_scores=True, cluster_ctas=cs, threads_per_cta=t, force_large=big) as eng:
        got = eng.drain_run(placed, remain, local=True)
        li = eng.last_launch()
        assert li["kernel"] == kernel and li["local"] and li["large"] == big, li
        _LAUNCHED["drain"].add(li["kernel"])
        states = [eng.scenario_storage_state(i) for i in range(len(drains))]
    live_vg, live_dev = ref[7], ref[8]
    o = _oracle(c)
    moved = 0
    try:
        for j, (d, rl, g) in enumerate(zip(drains, remain, got)):
            r = checkers.drain(o, placed, rl)
            for k in ("n_evicted", "n_placed", "n_unscheduled", "n_blocked", "n_vanished"):
                assert g[k] == r[k], (d, k)
            for k in ("evicted", "node", "score", "gpu_slots", "blocked", "fail_pod", "fail_counts"):
                np.testing.assert_array_equal(g[k], r[k], err_msg=f"drain {d}: {k}")
            vg, dev = o.storage_state()
            req = cap = 0
            for x in rl:
                nv = int(st.node_n_vg[x])
                if nv >= 0:
                    req += int(vg[:nv, x].sum())
                    cap += int(st.vg_capacity[:nv, x].sum())
            assert (g["vg_requested"], g["vg_capacity"]) == (req, cap), d
            bvg, bdev = states[j]
            rl = np.asarray(rl)
            gone = np.setdiff1d(np.arange(c.n_nodes), rl)
            np.testing.assert_array_equal(bvg[:, rl], vg[:, rl], err_msg=f"drain {d}: VG state")
            np.testing.assert_array_equal(bdev[rl], dev[rl], err_msg=f"drain {d}: device state")
            np.testing.assert_array_equal(bvg[:, gone], live_vg[:, gone], err_msg=f"drain {d}: removed nodes' VG state")
            np.testing.assert_array_equal(bdev[gone], live_dev[gone], err_msg=f"drain {d}: removed nodes' device state")
            moved += sum(1 for q in g["evicted"].tolist() if st.class_local[int(c.pods["pod_class"][q])])
    finally:
        o.close()
    assert moved > 0


# ---- what ran ----

def test_zz_every_local_kernel_launched_and_the_coverage():
    """Runs after the tests above: every local placement kernel and every drain-local kernel was launched and compared, and the
    interactions of test_open_local_oracle.coverage occur on the clusters compared here."""
    if not _LAUNCHED["place"] or not _LAUNCHED["drain"]:
        pytest.skip("runs after the placement and drain tests of this module")
    assert _LAUNCHED["place"] == compiled_kernels("simon_local_kernel_"), _LAUNCHED
    assert _LAUNCHED["drain"] == compiled_kernels("simon_drain_local_kernel_"), _LAUNCHED
    tot = {}
    for n_nodes in sorted({e[1] for e in LOCAL_ENTRIES}):
        for k, v in coverage(cluster(n_nodes, n_nodes), threads=THREADS).items():
            tot[k] = tot.get(k, 0) + v
    print(f"\nlocal placement kernels: {sorted(_LAUNCHED['place'])}\ndrain-local kernels: {sorted(_LAUNCHED['drain'])}\n"
          f"engine runs compared: {len(_DECISIONS)}, decisions compared: {sum(_DECISIONS)}\ncoverage: {tot}")
    for k, v in tot.items():
        assert v > 0, (k, tot)
