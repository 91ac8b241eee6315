"""Explained placement decisions on the GPU (simon_explain_set / Engine.explanations) against the CPU checker
(tests/explain_oracle.py), exactly.

Every simon_explain_kernel_* is launched at a geometry with several node slots per thread: VARIANTS names the cluster family
(test_zz_kernel_variants_gpu's) and the geometry, and each test asserts the kernel it launched.  The families mix spread, pod
(anti-)affinity, taints, GPU share, host ports, extended resources, DaemonSets and pre-bound pods, and Open-Local on the local ones; on
them every pod is explained.  With the set on, the placements, scores, failure records, node state and GPU slots are those of the same
run without it, and an unschedulable pod's histogram is its failure record."""
import numpy as np
import pytest

from explain_oracle import assert_records_equal, expected
from simon_b200 import abi
from test_zz_kernel_variants_gpu import _c3, _engine, family

# kernel -> (family, CTAs per scenario, threads per CTA, force_large): node slots per thread in the comment
VARIANTS = {
    "simon_explain_kernel_256": ("dense", 2, 160, False),           # 1,200 nodes: 4 slots
    "simon_explain_kernel_320": ("dense", 2, 288, False),           # 3 slots
    "simon_explain_kernel_384": ("dense", 2, 352, False),           # 2 slots
    "simon_explain_kernel_big": ("dense", 2, 160, True),            # 4 slots
    "simon_explain_local_kernel_256": ("local_300", 1, 128, False), # 3 slots
    "simon_explain_local_kernel_320": ("local_500", 1, 288, False), # 2 slots
    "simon_explain_local_kernel_384": ("local_700", 1, 352, False), # 2 slots
    "simon_explain_local_kernel_big": ("local_400", 1, 192, True),  # 3 slots
}
TOP_K = 3
_EXPECTED = {}


def _expected(fam, pods, top_k=TOP_K):
    key = (fam, top_k, len(pods), int(pods[0]), int(pods[-1]))
    if key not in _EXPECTED:
        _EXPECTED[key] = expected(family(fam), pods, top_k, open_local=fam.startswith("local"), threads=8)
    return _EXPECTED[key]


def _run(eng, **kw):
    out, score, fc, fp = eng.schedule(**kw)
    return out, score, fc, fp, eng.state(), eng.state_ext(), eng.gpu_slot_words()


def _assert_same_run(a, b, what):
    for x, y, name in zip(a, b, ("out", "score", "fail_counts", "fail_pod")):
        np.testing.assert_array_equal(x, y, err_msg=f"{what}: {name}")
    for d, e in ((a[4], b[4]), (a[5], b[5])):
        for k in d:
            np.testing.assert_array_equal(d[k], e[k], err_msg=f"{what}: {k}")
    np.testing.assert_array_equal(a[6], b[6], err_msg=f"{what}: GPU slots")


def _assert_rejected_is_fail_record(rec, pods, fc, fp):
    row = dict(zip(fp.tolist(), fc))
    n = 0
    for r, q in zip(rec, pods):
        if int(r["node"]) == -1:
            np.testing.assert_array_equal(r["rejected"], row[int(q)], err_msg=f"pod {q}")
            n += 1
    return n


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", list(VARIANTS))
def test_explain_variant_matches_checker(kernel):
    fam, cs, t, big = VARIANTS[kernel]
    c = family(fam)
    P = c.pods_dims["n_pods"]
    pods = np.arange(P, dtype=np.uint32)
    with _engine(c, cs, t, big, record_scores=True) as eng:
        plain = _run(eng)
        plain_kernel = eng.last_launch()["kernel"]
        eng.reset()
        got = _run(eng, explain=pods, top_k=TOP_K)
        li = eng.last_launch()
        rec, nodes = eng.explanations()
    assert li["kernel"] == kernel and not plain_kernel.startswith("simon_explain"), (li, plain_kernel)
    assert (li["cluster_ctas"], li["threads_per_cta"], li["large"]) == (cs, t, big), li
    assert li["node_slots"] >= 2, li
    _assert_same_run(got, plain, kernel)
    assert_records_equal(rec, nodes, _expected(fam, pods), pods, kernel)
    n_failed = _assert_rejected_is_fail_record(rec, pods, got[2], got[3])
    assert n_failed > 0 or fam.startswith("local")
    assert (rec["n_top"] == TOP_K).sum() >= 50
    sched = got[0] >= 0
    np.testing.assert_array_equal(nodes[sched & (rec["n_top"] > 0), 0]["words"][:, 8],
                                  np.where(rec[sched & (rec["n_top"] > 0)]["feasible"] > 1, got[1][sched & (rec["n_top"] > 0)], 0))


@pytest.mark.gpu
def test_explain_subset_split_calls_and_resume():
    """Every 7th pod explained (pinned runs of DaemonSet pods are cut by explained pods and resumed after them), top_k 8: one call,
    three split calls, and a resume from the middle, whose prefix records stay SIMON_EXPLAIN_NOT_RUN."""
    fam = "dense"
    c = family(fam)
    P = c.pods_dims["n_pods"]
    pods = np.arange(3, P, 7, dtype=np.uint32)
    want = _expected(fam, pods, 8)
    pinned = c.pods["pod_pin_node"] >= 0
    assert pinned[pods].any() and pinned.sum() > 100
    with _engine(c, 2, 160, False, record_scores=True) as eng:
        plain = _run(eng)
        eng.reset()
        got = _run(eng, explain=pods, top_k=8)
        _assert_same_run(got, plain, "subset")
        rec, nodes = eng.explanations()
        assert_records_equal(rec, nodes, want, pods, "subset")
        eng.reset()
        cuts = [0, P // 3, P // 3 + 1, (2 * P) // 3, P]
        for a, b in zip(cuts, cuts[1:]):
            eng.schedule(a, b - a)
        rec2, nodes2 = eng.explanations()
        assert_records_equal(rec2, nodes2, want, pods, "split")
        half = P // 2
        out3 = eng.schedule_resume(plain[0][:half])[0]
        np.testing.assert_array_equal(out3, plain[0])
        rec3, nodes3 = eng.explanations()
        pre = pods < half
        assert (rec3["node"][pre] == abi.EXPLAIN_NOT_RUN).all() and pre.any()
        assert_records_equal(rec3[~pre], nodes3[~pre], [w for w, p in zip(want, pre) if not p], pods[~pre], "resume")
        eng.explain_set([])
        eng.reset()
        eng.schedule()
        assert not eng.last_launch()["kernel"].startswith("simon_explain")


@pytest.mark.gpu
def test_explain_set_refusals():
    c = family("local_300")
    with _engine(c, 0, 0, False) as eng:
        P = c.pods_dims["n_pods"]
        eng.explain_set([1, 2], 2)
        for bad, k, msg in (([3, 3], 3, "ascending"), ([2, 1], 3, "ascending"), ([P], 3, "out of range"), ([0], 0, "top_k"),
                            ([0], abi.EXPLAIN_MAX_TOP + 1, "top_k")):
            with pytest.raises(RuntimeError, match=msg):
                eng.explain_set(bad, k)
        rec, _ = eng.explanations()             # the refused calls left the set of [1, 2] as it was
        assert list(rec["node"]) == [abi.EXPLAIN_NOT_RUN] * 2


@pytest.mark.gpu
def test_explain_c3_10000_every_pod():
    """A 10,000-node C3 with GPU share in the engine's own geometry, every pod explained at top_k 3: the placements of the run without
    the set, and 200 sampled records equal to the checker's."""
    c = _c3(10000, replicas=8)
    P = c.pods_dims["n_pods"]
    with _engine(c, 0, 0, False, record_scores=True) as eng:
        plain = _run(eng)
        eng.reset()
        got = _run(eng, explain=np.arange(P, dtype=np.uint32), top_k=3)
        li = eng.last_launch()
        rec, nodes = eng.explanations()
    assert li["kernel"].startswith("simon_explain_kernel_") and li["n_nodes"] == 10000, li
    _assert_same_run(got, plain, "c3 10000")
    reached = np.nonzero(c.pods["pod_fixed_node"] == -1)[0]
    sample = np.sort(np.random.default_rng(5).choice(reached, 200, replace=False)).astype(np.uint32)
    want = expected(c, sample, 3, threads=8)
    assert_records_equal(rec[sample], nodes[sample], want, sample, "c3 10000")


@pytest.mark.gpu
def test_explain_static_row_parts():
    """A cluster with container images, preferAvoidPods annotations and a host-side extra score plugin, every pod explained at 2 node
    slots per thread: the records equal the checker's, word 7 varies across the listed nodes, and explain.build splits it into parts
    that sum to the device word."""
    from explain_oracle import static_mix
    from simon_b200 import explain
    _p, c, plugins = static_mix()
    P = c.pods_dims["n_pods"]
    pods = np.arange(P, dtype=np.uint32)
    with _engine(c, 1, 64, False, record_scores=True) as eng:
        plain = _run(eng)
        eng.reset()
        got = _run(eng, explain=pods, top_k=4)
        li = eng.last_launch()
        rec, nodes = eng.explanations()
    assert li["kernel"] == "simon_explain_kernel_256" and li["node_slots"] == 2, li
    _assert_same_run(got, plain, "static row")
    assert_records_equal(rec, nodes, expected(c, pods, 4, threads=8), pods, "static row")
    listed = nodes[rec["n_top"] > 1]
    assert len({int(w) for w in listed["words"][:, :, 7].ravel()}) > 3
    n_built = 0
    for q in np.nonzero(rec["n_top"] > 1)[0]:
        ex = explain.build(c, int(q), rec[q], nodes[q], plugins)
        assert {"ImageLocality", "NodePreferAvoidPods", "NameParity"} <= set(ex.Nodes[0].Scores)
        n_built += 1
    assert n_built > 20


@pytest.mark.gpu
def test_simulator_explain_session_pods_and_template():
    """Simulator.Explain on a C3 session: session pods against the checker's records of the session's pod list, a Pod template
    against the checker on the list with the template appended, and the session's placements, slots and scores unchanged."""
    import copy

    from simon_b200 import synth
    from simon_b200.simulator import NewSimulator, PrepareCluster
    cluster, apps = synth.make_c3(n_nodes=300, n_workloads=40, replicas=8, n_apps=2, seed_no=11, gpu_pct=25)
    sim = NewSimulator()
    sim.RunCluster(PrepareCluster(cluster))
    for a in apps:
        sim.ScheduleApp(a)
    c = sim.compiled
    before = (sim.placements.copy(), sim.gpu_slots.copy(), sim.scores.copy())
    P = c.pods_dims["n_pods"]
    reached = np.nonzero(c.pods["pod_fixed_node"] == -1)[0]
    qs = sorted(int(q) for q in np.random.default_rng(3).choice(reached, 12, replace=False))
    names = [f"{c.pod_recs[q].tmpl.namespace}/{c.pod_recs[q].name}" for q in qs]
    tmpl = copy.deepcopy(c.pod_recs[qs[-1]].tmpl.pod)
    tmpl["metadata"] = {"name": "probe-template", "namespace": "default"}
    tmpl.get("spec", {}).pop("nodeName", None)
    res = sim.Explain(names + [tmpl], top=3)
    for a, b in zip(before, (sim.placements, sim.gpu_slots, sim.scores)):
        np.testing.assert_array_equal(a, b)
    want = expected(c, qs, 3, threads=8)
    for ex, w, q in zip(res, want, qs):
        assert ex.Pod == names[qs.index(q)] and ex.Feasible == w["feasible"]
        assert ex.Node == (c.node_names[w["node"]] if w["node"] >= 0 else "")
        assert [(n.Name, n.Total) for n in ex.Nodes] == [(c.node_names[g], wd[8]) for g, wd in w["top"]]
        assert sum(ex.Rejected.values()) >= int(w["rejected"].max())
        assert len(ex.Lines()) == (len(ex.Nodes[0].Scores) + len(ex.Nodes) if ex.Nodes else 0)
    # the template: the session's pods then the template, as one more pending pod
    from simon_b200.compiler import compile_cluster
    from simon_b200.workloads import make_valid_pod_by_pod
    p = sim._plan()
    c2 = compile_cluster(p.nodes, p.pods + [make_valid_pod_by_pod(tmpl)], p.ctx)
    w = expected(c2, [P], 3, threads=8)[0]
    ex = res[-1]
    assert ex.Feasible == w["feasible"] and [(n.Name, n.Total) for n in ex.Nodes] == [(c2.node_names[g], wd[8]) for g, wd in w["top"]]
    with pytest.raises(ValueError, match="nodeName"):
        sim.Explain([dict(tmpl, spec=dict(tmpl["spec"], nodeName=c.node_names[0]))])
    sim.Close()
