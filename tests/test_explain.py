"""Explained placement decisions on the CPU: the record checker (tests/explain_oracle.py) on hand-made cases and against the oracle's
own results, and the table of explained-decision kernels the GPU tests cover (tests/test_zz_explain_gpu.py)."""
import numpy as np
import pytest

from explain_oracle import expected, record
from simon_b200 import abi
from util import compiled_kernels, make_case


def _detail(totals):
    d = np.zeros((len(totals), abi.EXPLAIN_WORDS), np.int64)
    d[:, 8] = totals
    d[:, 0] = np.arange(len(totals))          # a word that tells the nodes apart
    return d


def test_ties_go_to_the_earlier_node():
    reasons = np.zeros(6, np.uint32)
    r = record(4, True, reasons, _detail([5, 9, 7, 9, 9, 7]), top_k=4)
    assert r["feasible"] == 6 and not r["rejected"].any()
    assert [n for n, _ in r["top"]] == [1, 3, 4, 2]
    assert [w[8] for _, w in r["top"]] == [9, 9, 9, 7]


def test_ties_follow_the_scenario_order():
    reasons = np.zeros(4, np.uint32)
    r = record(2, True, reasons, _detail([3, 3, 3, 1]), top_k=2, order=[2, 0, 1, 3])
    assert [n for n, _ in r["top"]] == [2, 0]


def test_single_feasible_node_is_listed_with_zero_words():
    reasons = np.array([1 << abi.SFC_CPU, 0, (1 << abi.SFC_CPU) | (1 << abi.SFC_MEM), 1 << abi.SFC_STATIC], np.uint32)
    r = record(1, True, reasons, _detail([0, 77, 0, 0]), top_k=3)
    assert r["feasible"] == 1 and r["top"] == [(1, [0] * abi.EXPLAIN_WORDS)]
    assert (r["rejected"][abi.SFC_CPU], r["rejected"][abi.SFC_MEM], r["rejected"][abi.SFC_STATIC]) == (2, 1, 1)
    assert r["rejected"].sum() == 4


def test_unschedulable_pod_has_no_nodes_and_every_reason_counted():
    reasons = np.array([1 << abi.SFC_PORTS, (1 << abi.SFC_CPU) | (1 << abi.SFC_TOO_MANY_PODS), 1 << abi.SFC_IPA_ANTI], np.uint32)
    r = record(-1, True, reasons, None, top_k=3)
    assert r["feasible"] == 0 and r["top"] == []
    assert [int(r["rejected"][b]) for b in (abi.SFC_PORTS, abi.SFC_CPU, abi.SFC_TOO_MANY_PODS, abi.SFC_IPA_ANTI)] == [1, 1, 1, 1]


@pytest.mark.parametrize("node", [-2, -3, 5])
def test_pod_that_never_reaches_the_scheduler(node):
    r = record(node, False, None, None, top_k=3)
    assert (r["node"], r["feasible"], r["top"]) == (node, 0, []) and not r["rejected"].any()


@pytest.mark.parametrize("kind,kw", [
    ("mix", dict(seed_no=103, n_nodes=95, n_workloads=40, max_replicas=7)),
    ("c3", dict(n_nodes=120, n_workloads=30, replicas=6, n_apps=2, seed_no=21, gpu_pct=25)),
])
def test_checker_agrees_with_the_oracles_own_results(kind, kw):
    """Every pod explained: the first listed node is the oracle's placement with its recorded score, a failed pod's histogram is its
    FitError row, every listed total is the sum of its weighted terms, and the list is ordered by (total desc, node order)."""
    from oracle.binding import Oracle
    _p, c = make_case(kind, **kw)
    P = c.pods_dims["n_pods"]
    o = Oracle(c)
    out, score, fc, fp = o.schedule()
    o.close()
    recs = expected(c, np.arange(P), top_k=4)
    failed = dict(zip(fp.tolist(), fc))
    n_multi = n_ties = 0
    for q, r in enumerate(recs):
        assert r["node"] == out[q], q
        if out[q] == -1:
            np.testing.assert_array_equal(r["rejected"], failed[q])
            assert r["feasible"] == 0 and r["top"] == []
            continue
        if not r["top"]:
            assert c.pods["pod_fixed_node"][q] != -1 or out[q] == -3
            continue
        assert r["top"][0][0] == out[q] and r["top"][0][1][8] == score[q], q
        assert len(r["top"]) == min(4, r["feasible"])
        assert int(r["rejected"][abi.SFC_STATIC]) <= c.n_nodes - r["feasible"]
        keys = [(-w[8], n) for n, w in r["top"]]
        assert keys == sorted(keys)
        for _n, w in r["top"]:
            assert w[8] == w[0] + w[1] + w[2] + w[3] + 2 * w[4] + w[5] + 2 * w[6] + w[7] + w[9]
        n_multi += len(r["top"]) > 1
        n_ties += any(a[1][8] == b[1][8] for a, b in zip(r["top"], r["top"][1:]))
    assert n_multi > P // 4 and (out == -1).any()
    assert n_ties > 0


def test_explain_kernels_are_the_gpu_tests_table():
    """Fails when simon_kernel.cu gains an explained-decision kernel the GPU tests do not run."""
    from test_zz_explain_gpu import VARIANTS
    names = compiled_kernels("simon_explain_")
    assert len(names) == 8 and set(VARIANTS) == names, sorted(names ^ set(VARIANTS))


def test_static_row_split_sums_to_the_oracle_word_and_matches_pyref():
    """explain.static_parts on a cluster with images, preferAvoidPods annotations and a host plugin: for every pod that reaches the
    scheduler with more than one feasible node, the parts sum to the oracle's word 7 on every feasible node, and ImageLocality /
    NodePreferAvoidPods equal the object-level reference's (oracle/pyref.py) times their weights."""
    from explain_oracle import static_mix
    from oracle.pyref import PyRef
    from simon_b200.explain import static_parts
    p, c, plugins = static_mix()
    ref = PyRef(c.node_objs, services=p.ctx.services, replicasets=p.ctx.replicasets, statefulsets=p.ctx.statefulsets,
                creation_order=c.node_orig_index)
    from oracle.binding import Oracle
    o = Oracle(c)
    o.enable_dump()
    seen = {"ImageLocality": set(), "NodePreferAvoidPods": set(), "NameParity": set()}
    checked = 0
    for q in range(c.pods_dims["n_pods"]):
        out = int(o.schedule(q, 1)[0][0])
        if c.pods["pod_fixed_node"][q] != -1 or out < 0:
            continue
        code, detail = o.last_detail()
        feas = np.nonzero(code == 0)[0]
        if len(feas) < 2:
            continue
        pod = c.pod_recs[q].tmpl.pod
        for g, parts in zip(feas, static_parts(c, int(c.pods["pod_class"][q]), feas, plugins)):
            assert sum(parts.values()) == detail[g][7], (q, g, parts, detail[g][7])
            assert parts["ImageLocality"] == ref.image_locality(pod, int(g))
            assert parts["NodePreferAvoidPods"] == 10000 * ref.prefer_avoid(pod, ref.nodes[int(g)])
            for k in seen:
                seen[k].add(parts[k])
        checked += 1
    o.close()
    assert checked > 20 and all(len(v) > 1 for v in seen.values()), seen


def test_lines_format():
    from simon_b200.explain import ExplainedNode, Explanation
    ex = Explanation("default/web-0", "n1", 3, [ExplainedNode("n1", 250, {"NodeAffinity": 100, "PodTopologySpread": 150}),
                                               ExplainedNode("n0", 180, {"NodeAffinity": 80, "PodTopologySpread": 100})])
    assert ex.Lines() == ["Plugin NodeAffinity scores on default/web-0 => [{n1 100} {n0 80}]",
                          "Plugin PodTopologySpread scores on default/web-0 => [{n1 150} {n0 100}]",
                          "Host n1 => Score 250", "Host n0 => Score 180"]
    assert Explanation("default/x", "", 0).Lines() == []


def test_explain_set_refusals_need_a_device_context():
    """simon_explain_set validates its arguments before any device work, but it needs a context with a pod upload, and a context
    cannot exist without a CUDA device (simon_ctx_create fails with SIMON_ERR_CUDA: the engine has no CPU path).  On the CPU the
    entry point is only reachable with a NULL context, which it refuses; the argument refusals run in test_zz_explain_gpu.py."""
    from simon_b200 import engine
    try:
        L = engine.lib()
    except engine.EngineUnavailable:
        pytest.skip("libsimon_gpu.so not built")
    assert L.simon_explain_set(None, None, 0, 3) == -1
    assert L.simon_explain_download(None, 0, 0, None, None) == -1
