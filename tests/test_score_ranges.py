"""Score arithmetic at the edges of its value ranges.

The synthetic generators draw API-typical values (NodeAffinity weights 1..100, maxSkew 1..5), far from the ranges where the
device's 32-bit storage and shortcuts stop being exact.  Each case below is one small hand-built cluster that puts one score
input at such an edge:
  * NodeAffinity raw sums around 2^32 / 100 (where 100 x raw leaves 32 bits) and up to 2^31 - 1,
  * PodTopologySpread ScheduleAnyway constraints with maxSkew up to 2^31 - 1 (raw scores past int32), and around 2^23 (the
    float-reciprocal fast path of the normalisation),
  * DoNotSchedule constraints with maxSkew 0 and -1 (a well-defined filter),
  * a Simon raw score of MinInt64 on every node,
  * the extra column (ImageLocality, NodePreferAvoidPods, extra plugins) at its largest accepted value.

CPU: the C oracle's placements equal oracle/pyref.py's (pyref has no extra plugins: that case is oracle-only), each case
asserts that it reached its edge, and the inputs the engine refuses are refused by the Python compiler and the native one
(simon_host_compile) with the same message.  tests/test_zz_score_ranges_gpu.py compares the device with the oracle on every
case.
"""
import numpy as np
import pytest

from simon_b200 import native_host, objects as O, simulator, synth
from simon_b200.compiler import (EXTRA_MAX, MIN_INT64, SCW_N_IPA_SCORE, SCW_N_PTS_SOFT, SCW_OFF_IPA_SCORE, SCW_OFF_PTS_SOFT,
                                 SCW_STATIC_ROW, CompileError, ExtraScorePlugin, compile_cluster)
from test_engine_limits import HOST, ZONE, _dep, _na_term, _refused_by_both, _spread, _term, class_words
from util import run_pyref

P = "preferredDuringSchedulingIgnoredDuringExecution"
N_NODES = 160
NA32_MAX = (1 << 32) // 100 - 1          # largest raw NodeAffinity score x 100 that fits 32 bits: 42,949,672
# inter-pod affinity weights of the near-bound case: (sum |w|) x pods just under 2^31 with its 6 + 20 + 7 pods
IPA_W_AFF, IPA_W_ANTI = 40_000_000, 25_000_000


def _nodes(n=N_NODES, eph=None):
    """n nodes over 4 zones, with 8..15 cores (several Simon values); every 3rd carries na0=yes, every 5th na1=yes."""
    out = []
    for i in range(n):
        labels = {}
        if i % 3 == 0:
            labels["na0"] = "yes"
        if i % 5 == 0:
            labels["na1"] = "yes"
        nd = synth._node(f"n{i:03d}", 8 + i % 8, f"z{i % 4}", "", 110, labels, None)
        if eph is not None:
            for sect in ("allocatable", "capacity"):
                nd["status"][sect]["ephemeral-storage"] = str(eph(i))
        out.append(nd)
    return out


def _objs(nodes, deps):
    return O.ResourceTypes(Nodes=nodes), [O.AppResource("ranges", O.ResourceTypes(Deployments=deps))]


def na_case(*weights):
    """One Deployment with preferred NodeAffinity terms of these weights on na0=yes, na1=yes: raw scores 0, w0, w1, w0 + w1."""
    prefs = [{"weight": w, "preference": _na_term((f"na{k}", ["yes"]))} for k, w in enumerate(weights)]
    return _objs(_nodes(), [_dep("a", 8, cpu="3", affinity={"nodeAffinity": {P: prefs}})])


def pts_case(*skews, keys=(HOST,)):
    """One Deployment with one ScheduleAnyway constraint per (maxSkew, topology key) on its own pods; a node in an empty domain
    scores maxSkew - 1, so the first pod's raw scores are exactly sum(maxSkew - 1)."""
    tsc = [_spread(k, s, False, app="a") for s, k in zip(skews, keys)]
    return _objs(_nodes(), [_dep("a", 12, cpu="3", topologySpreadConstraints=tsc)])


def hard_case(skew):
    """Three pods of b first, then pods of a under a DoNotSchedule constraint on the hostname counting b, with this maxSkew."""
    tsc = [_spread(HOST, skew, True, app="b")]
    return _objs(_nodes(), [_dep("b", 3, cpu="2"), _dep("a", 6, cpu="2", topologySpreadConstraints=tsc)])


def simon_case(top, low):
    """Simon raw scores `top` on even nodes and `low` on odd ones (ephemeral storage dominates every other share): the pod
    requests R bytes, with R / 128 exact so that 100 x R / 128 lands in [top, top + 1); even nodes have R + 128 allocatable,
    odd ones R + 200 R (share 1/200, raw 0) or R + 64 R (share 1/64, raw 1)."""
    R = -(-128 * top // 100)
    assert 100 * R // 128 == top and low in (0, 1)
    eph = lambda i: R + 128 if i % 2 == 0 else R + (200 if low == 0 else 64) * R
    return _objs(_nodes(eph=eph), [_dep("a", 6, cpu="10m", requests={"ephemeral-storage": str(R)})])


IPA_COUNTS = (100, 29, 57, 58, 14, 50, 1)     # pods of b on nodes 1, 3, 5, ...: 100 x (k / 100) is one ulp below k for 29, 57, 58


def _pod(name, node, labels):
    return {"kind": "Pod", "metadata": {"name": name, "namespace": "default", "labels": labels},
            "spec": {"nodeName": node, "containers": [{"name": "c", "image": "x",
                                                       "resources": {"requests": {"cpu": "1m", "memory": "1Mi"}}}]}}


def ipa_case(w_aff, w_anti=0, counts=IPA_COUNTS, anti_counts=()):
    """Running pods of b (counts[j] on node 2j + 1) and of c (anti_counts[j] on node 2j + 2); the pods of a prefer b's nodes
    with weight w_aff and avoid c's with weight w_anti: raw InterPodAffinity scores w_aff x count_b - w_anti x count_c."""
    cluster, apps = _objs(_nodes(), [])
    for j, k in enumerate(counts):
        cluster.Pods.extend(_pod(f"b{j}-{q}", f"n{2 * j + 1:03d}", {"app": "b"}) for q in range(k))
    for j, k in enumerate(anti_counts):
        cluster.Pods.extend(_pod(f"c{j}-{q}", f"n{2 * j + 2:03d}", {"app": "c"}) for q in range(k))
    aff = {"podAffinity": {P: [{"weight": w_aff, "podAffinityTerm": _term(HOST, app="b")}]}}
    if w_anti:
        aff["podAntiAffinity"] = {P: [{"weight": w_anti, "podAffinityTerm": _term(HOST, app="c")}]}
    apps[0].Resource.Deployments.append(_dep("a", 6, cpu="3", affinity=aff))
    return cluster, apps


EPH_REQ = 10 ** 17


def simon_min_case(uniform=True):
    """A pod requesting 10^17 bytes of ephemeral storage on nodes with 10^17 + 1: share 10^17, 100 x share past int64, raw Simon
    score MinInt64 (amd64 CVTTSD2SQ).  uniform=False: every other node has 10^18, a raw score of 11 there."""
    eph = (lambda i: EPH_REQ + 1) if uniform else (lambda i: EPH_REQ + 1 if i % 2 else 10 * EPH_REQ)
    return _objs(_nodes(eph=eph), [_dep("a", 6, cpu="1", requests={"ephemeral-storage": str(EPH_REQ)})])


def extra_plugins(top=47):
    """Two extra plugins: 100 x 21,464,831 on even nodes, 1 x `top` on every node; with the base 1,000,000 (ImageLocality 0 +
    10,000 x NodePreferAvoidPods 100) the largest extra score is 2^31 - 1 - 500 at top = 47."""
    even = ExtraScorePlugin("even", 21464831, lambda pod, node: 100 if int(O.name_of(node)[1:]) % 2 == 0 else 0)
    one = ExtraScorePlugin("one", top, lambda pod, node: 1)
    return [even, one]


def extra_case():
    """Extra scores at their bound, NodeAffinity 100 on na0 nodes, TaintToleration 100 and Simon 0..100 on top."""
    prefs = [{"weight": 1, "preference": _na_term(("na0", ["yes"]))}]
    return _objs(_nodes(), [_dep("a", 8, cpu="3", affinity={"nodeAffinity": {P: prefs}})])


# name -> (builder, extra plugins or None)
CASES = {
    "na_42949672": (lambda: na_case(NA32_MAX), None),
    "na_42949673": (lambda: na_case(NA32_MAX + 1), None),
    "na_50000000": (lambda: na_case(50_000_000), None),
    "na_2147483647": (lambda: na_case((1 << 31) - 1), None),
    "na_two_terms_32": (lambda: na_case(30_000_001, NA32_MAX - 30_000_001), None),
    "na_two_terms_64": (lambda: na_case(1_500_000_007, 600_000_011), None),
    # maxSkew 2^31 - 1 alone: raw scores from 2^31 - 2 up, past int32 once a node holds a pod
    "pts_host_2147483647": (lambda: pts_case((1 << 31) - 1), None),
    "pts_zone_2147483647": (lambda: pts_case((1 << 31) - 1, keys=(ZONE,)), None),
    "pts_two_2147483647": (lambda: pts_case((1 << 31) - 1, (1 << 31) - 1, keys=(HOST, ZONE)), None),
    "pts_8388606": (lambda: pts_case((1 << 23) - 2), None),
    "pts_8388608": (lambda: pts_case(1 << 23), None),
    "pts_8388609": (lambda: pts_case((1 << 23) + 1), None),
    "pts_zone_8388608": (lambda: pts_case(3, (1 << 23) - 3, keys=(HOST, ZONE)), None),
    # pts_max stays below 2^23 with distinct scores on later pods: the float-reciprocal estimate and its fix-up step
    "pts_8388596": (lambda: pts_case((1 << 23) - 12), None),
    "pts_min_0": (lambda: pts_case(1), None),
    "simon_16777215": (lambda: simon_case((1 << 24) - 1, 0), None),
    "simon_16777216": (lambda: simon_case(1 << 24, 0), None),
    "simon_range_16777215_min_1": (lambda: simon_case(1 << 24, 1), None),
    "simon_16777215_min_1": (lambda: simon_case((1 << 24) - 1, 1), None),
    "ipa_ulp": (lambda: ipa_case(1), None),
    "ipa_ulp_x3": (lambda: ipa_case(3), None),
    "ipa_near_bound": (lambda: ipa_case(IPA_W_AFF, IPA_W_ANTI, counts=(10, 3, 7), anti_counts=(5, 2)), None),
    "hard_skew_0": (lambda: hard_case(0), None),
    "hard_skew_-1": (lambda: hard_case(-1), None),
    "simon_min_uniform": (simon_min_case, None),
    "extra_max": (extra_case, extra_plugins),
}
NA_WEIGHTS = {"na_42949672": (NA32_MAX,), "na_42949673": (NA32_MAX + 1,), "na_50000000": (50_000_000,),
              "na_2147483647": ((1 << 31) - 1,), "na_two_terms_32": (30_000_001, NA32_MAX - 30_000_001),
              "na_two_terms_64": (1_500_000_007, 600_000_011)}
# spread cases: (the pod of a whose scores are checked, 0-based, the side of the bounds its pts_min / pts_max lie on):
#   int32: pts_max past int32; pts64: pts_max >= 2^23 (64-bit division); pts32: 0 < pts_max < 2^23 and pts_min < pts_max
#   (float-reciprocal estimate); eq32: pts_min = pts_max < 2^23
PTS_PROBE = {"pts_host_2147483647": (1, "int32"), "pts_zone_2147483647": (5, "int32"), "pts_two_2147483647": (0, "int32"),
             "pts_8388606": (1, "pts64"), "pts_8388608": (0, "eq32"), "pts_8388609": (0, "pts64"),
             "pts_zone_8388608": (0, "eq32"), "pts_8388596": (3, "pts32"), "pts_min_0": (3, "pts32")}
# Simon cases: (largest, smallest raw score of the row)
SIMON_ROWS = {"simon_16777215": ((1 << 24) - 1, 0), "simon_16777216": (1 << 24, 0),
              "simon_range_16777215_min_1": (1 << 24, 1), "simon_16777215_min_1": ((1 << 24) - 1, 1)}
NA_CASES = sorted(NA_WEIGHTS)
PTS_CASES = sorted(PTS_PROBE)


def build(name):
    """-> (plan, compiled) of case `name`."""
    mk, plugins = CASES[name]
    cluster, apps = mk()
    p = simulator.plan(cluster, apps)
    return p, compile_cluster(p.nodes, p.pods, p.ctx, extra_plugins=plugins() if plugins else None)


def oracle_detail(c, pod):
    """The oracle's placements up to `pod` and its per-node detail of that pod: (out, filter codes, detail rows
    [ba, la, ip, na, pts, tt, sm, ex, total, 0])."""
    from oracle.binding import Oracle
    o = Oracle(c)
    o.enable_dump()
    out = o.schedule(0, pod + 1)[0]
    code, sc = o.last_detail()
    o.close()
    return out, np.array(code, np.int32), np.array(sc, np.int64).reshape(len(code), -1)


def pods_of(c, workload):
    return [i for i, r in enumerate(c.pod_recs) if r.tmpl.workload_name == workload]


def assert_edge(name, c):
    """The case reaches the edge it is named for (on the first scored pod of its class)."""
    if name == "simon_min_uniform":
        assert (c.pods["simon_raw"][:, : c.snap_dims["n_node_classes"]] == MIN_INT64).any()
    if name == "extra_max":
        assert int(c.pods["extra_score"].max()) == EXTRA_MAX
    pod = pods_of(c, "a")[0]
    _out, code, det = oracle_detail(c, pod)
    feas = code == 0
    if name == "hard_skew_-1":
        assert not feas.any()
        return
    assert feas.sum() >= 2, name
    idx = np.array([int(nm[1:]) for nm in c.node_names])     # original node number of each compiled node
    if name in NA_WEIGHTS:
        ws = NA_WEIGHTS[name]
        raw = ws[0] * (idx % 3 == 0) + (ws[1] * (idx % 5 == 0) if len(ws) > 1 else 0)
        na_max = int(raw[feas].max())
        assert (na_max > NA32_MAX) == (name not in ("na_42949672", "na_two_terms_32")), (name, na_max)
        np.testing.assert_array_equal(det[feas, 3], (100 * raw[feas]) // na_max)
        assert (det[feas, 3] == 100).any() and (det[feas, 3] == 0).any()
    if name in SIMON_ROWS:
        row = c.pods["simon_raw"][int(class_words(c, "a")[SCW_STATIC_ROW]), : c.snap_dims["n_node_classes"]]
        assert (int(row.max()), int(row.min())) == SIMON_ROWS[name], (name, row.max(), row.min())
        assert (det[feas, 6] == 100).any() and (det[feas, 6] == 0).any()
    if name.startswith("ipa_"):
        raw = ipa_raw(c, idx)
        assert (det[feas, 2] == [f2i(100.0 * (float(r - min(0, raw.min())) / float(raw.max() - min(0, raw.min()))))
                                 for r in raw[feas]]).all()
        if name.startswith("ipa_ulp"):
            # 100 x (29 / 100) is 28.999999999999996 in float64: truncated, 28
            assert raw.max() == 100 * raw[idx == 1][0] // 100 and 28 in det[feas, 2] and 29 not in det[feas, 2]
        else:
            w = class_words(c, "a")
            sc = w[int(w[SCW_OFF_IPA_SCORE]):int(w[SCW_OFF_IPA_SCORE]) + 3 * int(w[SCW_N_IPA_SCORE])]
            bound = sum(abs(int(x)) for x in sc[2::3]) * len(c.pod_recs)
            assert (1 << 31) * 0.99 < bound < (1 << 31) and raw.min() < 0 < raw.max(), (bound, raw.min(), raw.max())
    if name in PTS_PROBE:
        probe, side = PTS_PROBE[name]
        pod = pods_of(c, "a")[probe]
        out, code, det = oracle_detail(c, pod)
        feas = code == 0
        raw = pts_raw(c, idx, out[pods_of(c, "a")[:probe]])
        lo, hi = int(raw[feas].min()), int(raw[feas].max())
        np.testing.assert_array_equal(det[feas, 4], (100 * (hi + lo - raw[feas])) // hi)
        assert {"int32": hi > (1 << 31) - 1, "pts64": hi >= (1 << 23), "pts32": 0 < hi < (1 << 23) and lo < hi,
                "eq32": 0 < lo == hi < (1 << 23)}[side], (name, lo, hi)
        if name == "pts_min_0":
            assert lo == 0
    if name == "hard_skew_0":
        b_nodes = {int(x) for x in _out[pods_of(c, "b")]}
        assert not feas[sorted(b_nodes)].any() and feas.sum() == c.n_nodes - len(b_nodes)


def pts_raw(c, idx, placed):
    """Raw PodTopologySpread scores of the next pod of a, after the pods of a at `placed`, on every node (all feasible, none
    ignored): sum over its constraints of count x ln(size + 2) + maxSkew - 1, in float64 and truncated (scoring.go)."""
    w = class_words(c, "a")
    soft = w[int(w[SCW_OFF_PTS_SOFT]):int(w[SCW_OFF_PTS_SOFT]) + 5 * int(w[SCW_N_PTS_SOFT])].reshape(-1, 5)
    log = c.snap["log_table"]
    zone = idx % 4
    on = np.bincount(np.asarray(placed, np.int64), minlength=c.n_nodes)
    score = np.zeros(c.n_nodes)
    for (_k, t, skew, host, _d) in soft.tolist():
        if host:
            cnt, size = on, c.n_nodes
        else:
            assert c.topo_keys[t] == ZONE
            per_zone = np.bincount(zone, weights=on, minlength=4)
            cnt, size = per_zone[zone], 4
        score = score + (cnt * log[size + 2] + float(skew - 1))
    return np.trunc(score).astype(np.int64)


def ipa_raw(c, idx):
    """Raw InterPodAffinity scores of the first pod of a: weight x matching running pods on the node, per term."""
    aff = c.pod_recs[pods_of(c, "a")[0]].tmpl.pod["spec"]["affinity"]
    node_of = {}
    for r in c.pod_recs:
        if r.node_name:
            lab = (r.tmpl.pod["metadata"].get("labels") or {}).get("app")
            node_of.setdefault(lab, []).append(c.node_index(r.node_name))
    raw = np.zeros(c.n_nodes, np.int64)
    for kind, sign in (("podAffinity", 1), ("podAntiAffinity", -1)):
        for t in (aff.get(kind) or {}).get(P, []):
            app = t["podAffinityTerm"]["labelSelector"]["matchLabels"]["app"]
            raw += sign * t["weight"] * np.bincount(node_of.get(app, []), minlength=c.n_nodes)
    return raw


def f2i(x):
    return int(x)


@pytest.mark.parametrize("name", sorted(CASES))
def test_case_reaches_its_edge_and_oracles_agree(name):
    from oracle.binding import Oracle
    p, c = build(name)
    assert_edge(name, c)
    o = Oracle(c)
    out = o.schedule()[0]
    o.close()
    assert (out >= 0).sum() >= 3 or name == "hard_skew_-1", name
    if CASES[name][1] is None:
        np.testing.assert_array_equal(out, run_pyref(p, c), err_msg=name)


@pytest.mark.parametrize("name", sorted(k for k in CASES if CASES[k][1] is None))
def test_native_compiler_accepts_the_edge(name):
    native_host.compile_native(*CASES[name][0]())


REFUSED = {
    "na_weight_negative": (lambda: na_case(-5), "preferred node affinity weight -5 is negative"),
    "na_weight_negative_mixed": (lambda: na_case(100, -1), "preferred node affinity weight -1 is negative"),
    "na_sum_2147483648": (lambda: na_case((1 << 31) - 1, 1), "preferred node affinity weights sum to 2"),
    "soft_skew_0": (lambda: pts_case(0), "ScheduleAnyway topology spread constraint with maxSkew 0 < 1"),
    "soft_skew_-3": (lambda: pts_case(-3), "ScheduleAnyway topology spread constraint with maxSkew -3 < 1"),
    "simon_min_mixed": (lambda: simon_min_case(uniform=False), "Simon score of MinInt64 on some nodes but not on all"),
    # maxSkew is an int32 (API type and device entry table): past it, hard and soft constraints alike
    "soft_skew_2147483648": (lambda: pts_case(1 << 31), "topology spread constraint maxSkew 2147483648 is outside int32"),
    "hard_skew_2147483648": (lambda: hard_case(1 << 31), "topology spread constraint maxSkew 2147483648 is outside int32"),
    "hard_skew_-2147483649": (lambda: hard_case(-(1 << 31) - 1), "maxSkew -2147483649 is outside int32"),
}


@pytest.mark.parametrize("case", sorted(REFUSED))
def test_out_of_range_scores_are_refused_by_both_compilers(case):
    mk, text = REFUSED[case]
    _refused_by_both(*mk(), text)


def test_soft_skew_missing_is_refused():
    """A ScheduleAnyway constraint without maxSkew compiles as maxSkew 0: refused like an explicit 0."""
    cluster, apps = pts_case(1)
    del apps[0].Resource.Deployments[0]["spec"]["template"]["spec"]["topologySpreadConstraints"][0]["maxSkew"]
    _refused_by_both(cluster, apps, "maxSkew 0 < 1")


def test_extra_column_bound_both_sides():
    """The extra column accepts 2^31 - 1 - 500 (the device adds NodeAffinity, TaintToleration, 2 x Simon and Open-Local, up to
    500 in all, in int32) and refuses one more.  Extra plugins exist in the Python compiler only."""
    cluster, apps = extra_case()
    p = simulator.plan(cluster, apps)
    c = compile_cluster(p.nodes, p.pods, p.ctx, extra_plugins=extra_plugins(47))
    assert int(c.pods["extra_score"].max()) == EXTRA_MAX == (1 << 31) - 1 - 500
    with pytest.raises(CompileError, match="extra plugin scores overflow the 32-bit extra column"):
        compile_cluster(p.nodes, p.pods, p.ctx, extra_plugins=extra_plugins(48))
