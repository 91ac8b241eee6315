"""Every placement kernel variant against the CPU oracle.

simon_api.cu:kernel_variant() picks one of the compiled instantiations of simon_place_body for a launch: unrolled node-slot loops
per (threads, slots per thread), run-time slot counts, the large-cluster variant (per-node arrays in global memory) and the
Open-Local variants.  Each is its own compilation with its own register allocation, so each one is checked here: VARIANTS names
the cluster family and the explicit geometry that reaches it, every test asserts the kernel it launched (Engine.last_launch), and
the CPU test below fails when simon_kernel.cu gains a variant the table does not name.

What is compared with the oracle: the node of every pod, the recorded winning score of every scheduled pod with a positive
score, the failure records, every state() column, state_ext() (extended resources and per-device GPU-share memory) and the
GPU-share device slots of every pod.  The families are crowded enough that pods fail and feasibility flips, and carry GPU-share
pods, DaemonSet (pinned) pods, host ports, spread and affinity constraints.  The file sorts after the rest of the suite.
"""
import functools
import os

import numpy as np
import pytest

from simon_b200 import simulator, synth
from simon_b200.compiler import compile_cluster
from test_daemonset_pins import _ds
from util import compiled_kernels

# kernel -> (cluster family, [(CTAs per scenario, threads per CTA, force_large)]); the families are built below
VARIANTS = {
    "simon_place_kernel_256_1": ("dense", [(8, 160, False)]),
    "simon_place_kernel_256_2": ("dense", [(3, 256, False)]),
    "simon_place_kernel_256_3": ("dense", [(2, 224, False)]),
    "simon_place_kernel_256_4": ("dense", [(2, 160, False)]),
    "simon_place_kernel_256_0": ("dense", [(2, 96, False)]),
    "simon_place_kernel_320_1": ("dense", [(4, 320, False)]),
    "simon_place_kernel_320_2": ("dense", [(2, 320, False)]),
    "simon_place_kernel_320_3": ("dense", [(2, 288, False)]),
    "simon_place_kernel_384_1": ("dense", [(4, 352, False)]),
    "simon_place_kernel_384_2": ("dense", [(2, 352, False)]),
    "simon_place_kernel_384_3": ("c3_1000", [(1, 352, False)]),
    "simon_place_kernel_320_4": ("c3_2000", [(2, 320, False)]),
    "simon_place_kernel_320_0": ("c2_1400", [(1, 288, False)]),
    "simon_place_kernel_384_0": ("c2_1400", [(1, 352, False)]),
    "simon_place_kernel_big": ("dense", [(16, 320, True), (2, 160, True), (1, 256, True)]),
    "simon_local_kernel_256": ("local_300", [(2, 128, False)]),
    "simon_local_kernel_320": ("local_500", [(1, 320, False)]),
    "simon_local_kernel_384": ("local_700", [(1, 352, False)]),
    "simon_local_kernel_big": ("local_400", [(1, 192, True)]),
}
ENTRIES = [(k, fam, cs, t, big) for k, (fam, geoms) in VARIANTS.items() for cs, t, big in geoms]


def compiled_kernel_variants():
    """The placement kernels simon_kernel.cu defines, without the per-phase timer variants (simon_prof_kernel_*)."""
    return compiled_kernels("simon_place_kernel_") | compiled_kernels("simon_local_kernel_")


def test_variant_table_names_every_placement_kernel_of_the_variant_list():
    names = compiled_kernel_variants()
    assert len(names) >= 19 and "simon_place_kernel_big" in names and "simon_local_kernel_big" in names
    assert set(VARIANTS) == names, f"kernels without a test: {sorted(names - set(VARIANTS))}, unknown: {sorted(set(VARIANTS) - names)}"


@pytest.mark.parametrize("seed", [101, 206, 223])
def test_oracle_ext_state_is_the_sum_over_its_placements(seed):
    """The oracle's exported extended-resource and GPU-share state, which the GPU tests compare with, agrees with its own
    placements: req_scalar sums the scalar requests of every placed pod (pre-bound ones included); gpu_used sums, per device, the
    slots each scheduled pod's word names times its per-slot memory; every GPU-share pod the scheduler placed holds exactly its
    GPU count of slots, and every other pod none."""
    from oracle.binding import Oracle
    from simon_b200.compiler import SCW_GPU_COUNT, SCW_GPU_MEM, SCW_OFF_SCALARS
    cluster, apps = synth.make_mix(seed_no=seed, n_nodes=80, n_workloads=60, max_replicas=8)
    c = _compile(cluster, apps)
    o = Oracle(c)
    out = o.schedule()[0]
    ext, slots = o.state_ext(), o.gpu_slot_words()
    o.close()
    K, N = int(c.snap_dims["n_scalars"]), c.n_nodes
    blob, off, cls, fixed = c.pods["class_blob"], c.pods["class_off"], c.pods["pod_class"], c.pods["pod_fixed_node"]
    rs, gu = np.zeros((K, N), np.int64), np.zeros((8, N), np.int64)
    n_gpu = 0
    for i, n in enumerate(out.tolist()):
        w = blob[int(off[cls[i]]):]
        counts = [(int(slots[i]) >> (4 * d)) & 15 for d in range(8)]
        if n < 0:
            assert slots[i] == 0
            continue
        rs[:, n] += w[int(w[SCW_OFF_SCALARS]):int(w[SCW_OFF_SCALARS]) + K]
        if fixed[i] >= 0 or w[SCW_GPU_MEM] <= 0:
            assert slots[i] == 0, i
            continue
        assert sum(counts) == w[SCW_GPU_COUNT], i
        n_gpu += 1
        for d in range(8):
            gu[d, n] += counts[d] * w[SCW_GPU_MEM]
    np.testing.assert_array_equal(ext["req_scalar"], rs)
    np.testing.assert_array_equal(ext["gpu_used"], gu)
    assert n_gpu > 0 and K > 0


# ---- cluster families ----------------------------------------------------------------------------------------------------------

def _compile(cluster, apps):
    p = simulator.plan(cluster, apps)
    return compile_cluster(p.nodes, p.pods, p.ctx)


def _dense():
    """make_mix (GPU share, host ports, extended resources, hard spread, required (anti-)affinity, DaemonSets, pre-bound pods) at
    1,200 nodes with many more workloads than its own tests use, plus two DaemonSets: one everywhere with a host port, one large
    enough not to fit some nodes."""
    cluster, apps = synth.make_mix(seed_no=100, n_nodes=1200, n_workloads=150, max_replicas=12)
    cluster.DaemonSets.append(_ds("agent", cpu="50m", port=9300, tolerations=[{"operator": "Exists"}]))
    cluster.DaemonSets.append(_ds("hog", cpu="1500m"))
    return _compile(cluster, apps)


def _c3(n_nodes, n_workloads=60, replicas=10, seed_no=41, daemonsets=True):
    """C3-shaped (prefilled, pre-bound pods, anti-affinity, spread) with GPU-share devices on a quarter of the nodes and two
    DaemonSets, one of them in an app."""
    cluster, apps = synth.make_c3(n_nodes=n_nodes, n_workloads=n_workloads, replicas=replicas, n_apps=2, seed_no=seed_no, gpu_pct=25)
    if daemonsets:
        cluster.DaemonSets.append(_ds("agent", cpu="50m", port=9300, tolerations=[{"operator": "Exists"}]))
        apps[1].Resource.DaemonSets.append(_ds("hog", cpu="2"))
    return _compile(cluster, apps)


def _c2(n_nodes):
    cluster, apps = synth.make_c2(n_nodes=n_nodes, n_workloads=40, replicas=20, seed_no=43)
    cluster.DaemonSets.append(_ds("agent", cpu="50m", port=9300, tolerations=[{"operator": "Exists"}]))
    apps[0].Resource.DaemonSets.append(_ds("hog", cpu="2"))
    return _compile(cluster, apps)


def _local(n_nodes):
    from test_open_local import _oracle_cluster
    nodes, pods, scs = _oracle_cluster(np.random.default_rng(n_nodes), n_nodes, 250)
    return compile_cluster(nodes, pods, open_local=True, storage_classes=scs)


FAMILIES = {
    "dense": _dense,
    "c3_1000": lambda: _c3(1000),
    "c3_2000": lambda: _c3(2000),
    "c2_1400": lambda: _c2(1400),
    "local_300": lambda: _local(300),
    "local_400": lambda: _local(400),
    "local_500": lambda: _local(500),
    "local_700": lambda: _local(700),
    "c3_5600": lambda: _c3(5600, replicas=8),
    "c3_7000": lambda: _c3(7000, replicas=8),
    "c3_11000": lambda: _c3(11000, replicas=8),
    "c3_10000_batch": lambda: _c3(10000, n_workloads=40, replicas=5, daemonsets=False),
}


@functools.lru_cache(maxsize=None)
def family(name):
    return FAMILIES[name]()


@functools.lru_cache(maxsize=None)
def oracle_run(name):
    """(out, score, fail_counts, fail_pod, state, state_ext, slot words) of the oracle on the whole pod list of a family."""
    from oracle.binding import Oracle
    c = family(name)
    o = Oracle(c, threads=min(16, len(os.sched_getaffinity(0))))
    res = o.schedule() + (o.state(), o.state_ext(), o.gpu_slot_words())
    o.close()
    return res


def assert_matches_oracle(name, out, score, fc, fp, eng, what=""):
    ref, rscore, rfc, rfp, rst, rext, rslots = oracle_run(name)
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


def _engine(c, cs, t, big, **kw):
    from simon_b200.engine import Engine
    return Engine(c, device=0, cluster_ctas=cs, threads_per_cta=t, force_large=big, **kw)


# per kernel: the stats of its runs, and what the matrix as a whole must have exercised
_SEEN = {}


@pytest.mark.gpu
@pytest.mark.parametrize("kernel,fam,cs,t,big", [e for e in ENTRIES if not e[1].startswith("local")],
                         ids=[f"{k[6:]}-{cs}x{t}" for k, fam, cs, t, big in ENTRIES if not fam.startswith("local")])
def test_variant_matches_oracle(kernel, fam, cs, t, big):
    c = family(fam)
    ref = oracle_run(fam)[0]
    for pin_fast in (True, False):
        with _engine(c, cs, t, big, record_scores=True, pin_fast=pin_fast) as eng:
            out, score, fc, fp = eng.schedule()
            li = eng.last_launch()
            assert li["kernel"] == kernel, li
            assert (li["cluster_ctas"], li["threads_per_cta"], li["large"]) == (cs, t, big), li
            assert_matches_oracle(fam, out, score, fc, fp, eng, f"{kernel} {cs}x{t} pin_fast={pin_fast}")
            _SEEN.setdefault(kernel, []).append(eng.stats())
    pinned = c.pods["pod_pin_node"] >= 0
    assert (ref == -1).any() and (ref[pinned] >= 0).any()             # pods failed, pinned pods were placed
    if fam != "c2_1400":                                              # C2 has no GPU share
        assert (oracle_run(fam)[6] != 0).any()                        # GPU-share pods were placed


@pytest.mark.gpu
def test_variant_matrix_exercised_the_flip_paths():
    """Across the matrix the kernels rebuilt feasible-set summaries, redid decisions after a feasibility flip and took the
    single-node flip fast path, so those paths ran on several variants."""
    want = {k for k, fam, *_ in ENTRIES if not fam.startswith("local")}
    if not want <= set(_SEEN):
        pytest.skip("runs after the whole matrix of test_variant_matches_oracle")
    for key in ("summary_rebuilds", "redone", "single_flip_fast"):
        assert sum(s[key] for runs in _SEEN.values() for s in runs) > 0, key
        assert sum(1 for runs in _SEEN.values() if any(s[key] for s in runs)) >= 3, key


@pytest.mark.gpu
@pytest.mark.parametrize("kernel,fam,cs,t,big", [e for e in ENTRIES if e[1].startswith("local")],
                         ids=[f"{k[6:]}-{cs}x{t}" for k, fam, cs, t, big in ENTRIES if fam.startswith("local")])
def test_open_local_variant_matches_restated_composition(kernel, fam, cs, t, big):
    """The storage-less CPU oracle plus storage.py's Filter, ScoreLVM, NormalizeScore and Bind, pod by pod
    (test_open_local.check_restated_open_local), at a geometry that launches the variant: a check independent of the oracle's own
    Open-Local, which test_zz_open_local_oracle_gpu.py compares every variant with on mixed clusters."""
    from test_open_local import check_restated_open_local
    c = family(fam)
    with _engine(c, cs, t, big, record_scores=True) as eng:
        out, score, _fc, _fp = eng.schedule()
        final = eng.storage_state()
        li = eng.last_launch()
    assert li["kernel"] == kernel and li["local"] and li["large"] == big, li
    assert check_restated_open_local(c, out, score, final) > 0
    assert (out >= 0).sum() > len(out) // 2


@pytest.mark.gpu
@pytest.mark.parametrize("fam,kernel,slots", [("c3_5600", "simon_place_kernel_384_1", 1), ("c3_7000", "simon_place_kernel_256_2", 2),
                                              ("c3_11000", "simon_place_kernel_384_2", 2)])
def test_natural_geometry_at_production_sizes(fam, kernel, slots):
    """The geometry the engine picks by itself for a single run of these sizes (16 CTAs, the fewest node slots per thread)."""
    c = family(fam)
    with _engine(c, 0, 0, False, record_scores=True) as eng:
        out, score, fc, fp = eng.schedule()
        li = eng.last_launch()
        assert (li["kernel"], li["cluster_ctas"], li["node_slots"], li["n_nodes"]) == (kernel, 16, slots, c.n_nodes), li
        assert_matches_oracle(fam, out, score, fc, fp, eng, kernel)


def _node_lists(n, seed):
    rng = np.random.default_rng(seed)
    sub = rng.permutation(n)[: (4 * n) // 5]
    return [np.arange(n), np.arange(0, n, 2), np.arange(n)[: (2 * n) // 3][::-1], sub]


@pytest.mark.gpu
@pytest.mark.parametrize("fam,kernel,cs,t,big", [("c3_10000_batch", "simon_place_kernel_320_4", 8, 320, False),
                                                 ("dense", "simon_place_kernel_384_2", 2, 352, False),
                                                 ("dense", "simon_place_kernel_256_2", 3, 256, False),
                                                 ("dense", "simon_place_kernel_big", 2, 160, True)])
def test_scenario_batch_variant_matches_oracle(fam, kernel, cs, t, big):
    """Scenario batches (one cluster per scenario, one launch): all nodes (no node list), every other node, a reversed subset and
    a random subset, each against the oracle restricted to the same node list.  The first row is the benchmark's batch shape
    (C3, 8 CTAs x 320 threads x 4 node slots on the full node list) with fewer pods."""
    from oracle.binding import Oracle
    c = family(fam)
    lists = _node_lists(c.n_nodes, 7)
    with _engine(c, cs, t, big) as eng:
        res, nodes = eng.run_scenarios(lists, want_nodes=True)
        li = eng.last_launch()
    assert (li["kernel"], li["n_scenarios"], li["large"]) == (kernel, len(lists), big), li
    o = Oracle(c, threads=min(16, len(os.sched_getaffinity(0))))
    for i, act in enumerate(lists):
        o.set_active(act)
        o.reset()
        ref = o.schedule()[0]
        st = o.state()
        np.testing.assert_array_equal(nodes[i], ref, err_msg=f"scenario {i}")
        assert res[i]["n_unscheduled"] == int((ref == -1).sum()), i
        assert (res[i]["req_mcpu"], res[i]["req_mem"]) == (int(st["req_mcpu"][act].sum()), int(st["req_mem"][act].sum())), i
        assert (res[i]["alloc_mcpu"], res[i]["alloc_mem"]) == (int(c.snap["alloc_mcpu"][act].sum()), int(c.snap["alloc_mem"][act].sum())), i
    o.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kernel,cs,t,big", [("simon_place_kernel_256_4", 2, 160, False), ("simon_place_kernel_384_2", 2, 352, False),
                                             ("simon_place_kernel_big", 2, 160, True)])
def test_resume_variant_rebuilds_the_state(kernel, cs, t, big):
    """simon_schedule_resume on the dense mix: the first half of the pods rebuilt at the nodes a full run gave them (GPU-share
    device memory replayed per node), the rest placed again - the same placements, state and device slots."""
    c = family("dense")
    with _engine(c, cs, t, big) as eng:
        out = eng.schedule()[0]
        st, ext, slots = eng.state(), eng.state_ext(), eng.gpu_slot_words()
        P = len(out)
        out2 = eng.schedule_resume(out[: P // 2])[0]
        assert eng.last_launch()["kernel"] == kernel
        np.testing.assert_array_equal(out2, out)
        st2, ext2 = eng.state(), eng.state_ext()
        for k in st:
            np.testing.assert_array_equal(st2[k], st[k], err_msg=k)
        for k in ext:
            np.testing.assert_array_equal(ext2[k], ext[k], err_msg=k)
        np.testing.assert_array_equal(eng.gpu_slot_words(), slots)
    np.testing.assert_array_equal(out, oracle_run("dense")[0])
