"""The engine's fixed limits (DESIGN.md section 2), each reached exactly by a small cluster built from plain objects, and each
exceeded by one.

Every builder below sits AT one limit and asserts from the compiled dims and class records that it got there: 8 scalar resources,
1,024 label atoms (16 words; selectors on bit 63 of every word, the int64 sign bit), 256 distinct taints (4 words), a node with
all 256 taints PreferNoSchedule (a TaintToleration count that does not fit the static-verdict record), 8 topologies (the 7th key
at topology index 7), 32 constraint/term entries per class (32 host-port entries; 8 hard + 8 soft spread constraints + 16
inter-pod terms; a mix), a commit list of more than 64 counters, a class record of several thousand words, and 8 GPU-share
devices per node with pods that put more than 15 slots on one device.

CPU: the builders reach their limits; one past each limit is refused by the Python compiler and by the native one
(simon_host_compile) alike; the native compiler's columns equal the Python compiler's; simon_host_plan_fit_error equals
simulator.format_fit_error; the C oracle's placements equal oracle/pyref.py's.  tests/test_zz_engine_limits_gpu.py compares
the device with the C oracle on the same builders.
"""
import ctypes as C

import numpy as np
import pytest

from simon_b200 import native_host, objects as O, simulator, synth
from simon_b200.abi import SFC_SCALAR0
from simon_b200.compiler import (CompileError, SCW_N_ENT, SCW_N_INC, SCW_N_IPA_AFF, SCW_N_IPA_ANTI, SCW_N_IPA_EXIST,
                                 SCW_N_IPA_SCORE, SCW_N_PORTS, SCW_N_PTS_HARD, SCW_N_PTS_SOFT, compile_cluster)
from util import run_oracle, run_pyref

R = "requiredDuringSchedulingIgnoredDuringExecution"
P = "preferredDuringSchedulingIgnoredDuringExecution"


# ---- objects ----------------------------------------------------------------------------------------------------------------

def _node(name, cores=16, labels=None, taints=None, extra=None, zone="z0", gpus=None):
    """A node of `cores` cores and 4 GiB per core; extra: more allocatable resources; gpus: (devices, memory per device)."""
    n = synth._node(name, cores, zone, "", 100, labels, taints)
    if zone is None:
        del n["metadata"]["labels"]["topology.kubernetes.io/zone"]
    for sect in ("allocatable", "capacity"):
        n["status"][sect].update(extra or {})
        if gpus:
            n["status"][sect]["alibabacloud.com/gpu-count"] = str(gpus[0])
            n["status"][sect]["alibabacloud.com/gpu-mem"] = str(gpus[0] * gpus[1])
    return n


def _dep(name, replicas, cpu="500m", requests=None, labels=None, ports=(), gpu=None, **spec):
    """A Deployment; labels default to app=<name>; ports: host ports; gpu: (gpu-count, gpu-mem per device)."""
    labels = dict(labels or {"app": name})
    req = {"cpu": cpu, "memory": "256Mi"}
    req.update(requests or {})
    c = {"name": "c", "image": f"registry.local/{name}:v1", "resources": {"requests": req}}
    if ports:
        c["ports"] = [{"containerPort": p, "hostPort": p} for p in ports]
    meta = {"labels": labels}
    if gpu:
        meta["annotations"] = {"alibabacloud.com/gpu-count": str(gpu[0]), "alibabacloud.com/gpu-mem": str(gpu[1])}
    return {"apiVersion": "apps/v1", "kind": "Deployment", "metadata": {"name": name, "namespace": "default"},
            "spec": {"replicas": replicas, "selector": {"matchLabels": labels},
                     "template": {"metadata": meta, "spec": dict(containers=[c], **spec)}}}


def _objs(nodes, deps):
    return O.ResourceTypes(Nodes=nodes), [O.AppResource("limits", O.ResourceTypes(Deployments=deps))]


def _sel(**kv):
    return {"matchLabels": dict(kv)}


def _spread(key, skew, hard, **sel):
    return {"topologyKey": key, "maxSkew": skew, "whenUnsatisfiable": "DoNotSchedule" if hard else "ScheduleAnyway",
            "labelSelector": _sel(**sel)}


def _term(key, **sel):
    return {"labelSelector": _sel(**sel), "topologyKey": key}


def _na_term(*exprs):
    return {"matchExpressions": [{"key": k, "operator": "In", "values": list(v)} for k, v in exprs]}


HOST, ZONE = "kubernetes.io/hostname", "topology.kubernetes.io/zone"


# ---- builders: each AT one limit -----------------------------------------------------------------------------------------------

SCALARS = [f"limits.test/r{k}" for k in range(8)]


def scalars8(n_scalars=8):
    """8 extended resources, each requested by some pod and missing or short on some nodes: every Insufficient <r_k> occurs."""
    nodes = []
    for i in range(24):
        extra = {SCALARS[k] if k < 8 else f"limits.test/r{k}": str((3 * i + k) % 5) for k in range(n_scalars) if (3 * i + k) % 5}
        nodes.append(_node(f"n{i:02d}", 16, extra=extra, zone=f"z{i % 3}"))
    names = SCALARS + [f"limits.test/r{k}" for k in range(8, n_scalars)]
    deps = [_dep(f"s{k}", 40, requests={names[k]: "1"}) for k in range(n_scalars)]
    deps += [_dep(f"mix{j}", 8, requests={names[j]: "2", names[(j + 3) % n_scalars]: "1"}) for j in range(8)]
    return _objs(nodes, deps)


def atoms1024(extra_atom=False):
    """1,024 label atoms: node-label pairs (w<w>, b<j>) for 16 words x 64 values, interned first by one class's preferred terms
    (atom 64 w + j).  Node selectors, required and preferred terms then sit on atoms 63/64, 127/128, ..., 1023."""
    nodes = [_node(f"n{i:03d}", 16, labels={f"w{w}": f"b{(i + 5 * w) % 64}" for w in range(16)}) for i in range(128)]
    fill = {"nodeAffinity": {P: [{"weight": w + 1, "preference": _na_term((f"w{w}", [f"b{j}" for j in range(64)]))} for w in range(16)]}}
    deps = [_dep("fill", 4, affinity=fill)]
    deps += [_dep(f"sel{w}", 12, cpu="2", nodeSelector={f"w{w}": "b63"}) for w in range(16)]
    deps += [_dep(f"req{w}", 12, cpu="2", affinity={"nodeAffinity": {R: {"nodeSelectorTerms": [_na_term((f"w{w + 1}", ["b0"]))]}}})
             for w in range(15)]
    deps += [_dep(f"pref{w}", 6, cpu="3", affinity={"nodeAffinity": {P: [
        {"weight": 50, "preference": _na_term((f"w{w}", ["b63"]))},
        {"weight": 30, "preference": _na_term((f"w{(w + 1) % 16}", ["b0"]))}]}}) for w in range(16)]
    if extra_atom:
        deps.append(_dep("extra", 1, nodeSelector={"w0": "b64"}))
    return _objs(nodes, deps)


TAINT_EDGES = [0, 63, 64, 127, 128, 191, 192, 255]


def taints256(extra_taint=False):
    """256 distinct NoSchedule taints t000..t255, all on the first node (so that their ids are 0..255), and the word-boundary ones
    on other nodes; each tol<id> class tolerates exactly one of them."""
    nodes = [_node("sink", 64, taints=[{"key": f"t{i:03d}", "effect": "NoSchedule"} for i in range(256)])]
    for j in range(40):
        ts = []
        if j < 32:
            ts.append(TAINT_EDGES[j % 8])
        elif j < 36:
            ts += [TAINT_EDGES[2 * (j - 32) + 1], TAINT_EDGES[(2 * (j - 32) + 2) % 8]]
        nodes.append(_node(f"n{j:02d}", 16, taints=[{"key": f"t{t:03d}", "effect": "NoSchedule"} for t in ts]))
    if extra_taint:
        nodes.append(_node("one-more", 16, taints=[{"key": "t256", "effect": "NoSchedule"}]))
    deps = [_dep(f"tol{t}", 14, cpu="2", tolerations=[{"key": f"t{t:03d}", "operator": "Exists", "effect": "NoSchedule"}])
            for t in TAINT_EDGES]
    deps += [_dep("none", 40, cpu="2"), _dep("all", 10, cpu="4", tolerations=[{"operator": "Exists"}])]
    return _objs(nodes, deps)


def soft_taints256():
    """All 256 taints PreferNoSchedule on three nodes (TaintToleration counts 256 there for a class that tolerates none); fewer on
    others.  A class with a DoNotSchedule zone spread and a node selector runs on them too."""
    nodes = []
    for i in range(48):
        k = 256 if i % 16 == 0 else (i * 11) % 97
        taints = [{"key": f"s{t:03d}", "effect": "PreferNoSchedule"} for t in range(k)]
        nodes.append(_node(f"n{i:02d}", 16, taints=taints, zone=f"z{i % 3}", labels={"pool": "a" if i % 4 else "b"}))
    tol_half = [{"key": f"s{t:03d}", "operator": "Exists", "effect": "PreferNoSchedule"} for t in range(128)]
    deps = [_dep("none", 200, cpu="4"), _dep("half", 24, cpu="1", tolerations=tol_half),
            _dep("all", 16, cpu="1", tolerations=[{"operator": "Exists"}]),
            _dep("spread", 30, cpu="1", nodeSelector={"pool": "a"}, topologySpreadConstraints=[_spread(ZONE, 1, True, app="spread")])]
    return _objs(nodes, deps)


TOPO_KEYS = [f"topo.test/k{i}" for i in range(1, 9)]


def topo8(n_keys=7):
    """Topology keys k1..k7 besides the node itself: k1..k6 interned by the first class's soft constraints, so that k7 is
    topology index 7; spread, affinity and anti-affinity on k7; some nodes lack k7 or k3."""
    nodes = []
    for i in range(60):
        lab = {TOPO_KEYS[q]: f"d{q}-{i % (q + 2)}" for q in range(n_keys)}
        if i % 6 == 5:
            del lab[TOPO_KEYS[6]]
        if i % 10 == 3:
            del lab[TOPO_KEYS[2]]
        nodes.append(_node(f"n{i:02d}", 16, labels=lab, zone=None))
    k7 = TOPO_KEYS[6]
    deps = [_dep("soft6", 30, topologySpreadConstraints=[_spread(TOPO_KEYS[q], 1 + q, False, app="soft6") for q in range(6)])]
    deps += [_dep(f"extra{q}", 2, topologySpreadConstraints=[_spread(TOPO_KEYS[q], 1, False, app="soft6")]) for q in range(7, n_keys)]
    deps += [_dep("hard7", 40, cpu="1", topologySpreadConstraints=[_spread(k7, 1, True, app="hard7")]),
             _dep("aff7", 16, affinity={"podAffinity": {R: [_term(k7, app="hard7")]}}),
             _dep("anti7", 10, affinity={"podAntiAffinity": {R: [_term(k7, app="anti7")]},
                                        "nodeAffinity": {R: {"nodeSelectorTerms": [{"matchExpressions": [{"key": k7, "operator": "Exists"}]}]}}}),
             _dep("pref7", 20, cpu="1", topologySpreadConstraints=[_spread(k7, 2, False, app="pref7")],
                  affinity={"podAffinity": {P: [{"weight": 80, "podAffinityTerm": _term(k7, app="hard7")}]},
                            "podAntiAffinity": {P: [{"weight": 40, "podAffinityTerm": _term(k7, app="soft6")}]}})]
    return _objs(nodes, deps)


def entries32(n_ports=32, n_hard=8, n_soft=8, n_mixed=32):
    """Three classes at 32 entries.  A: host ports 1..32, each shared with one partner workload b<i> (one port entry per distinct
    set of users).  E: n_hard DoNotSchedule + n_soft ScheduleAnyway constraints + preferred pod (anti-)affinity terms up to 32.
    M: 8 host ports, 4 hard, 4 soft, 4 required anti-affinity terms, preferred terms up to n_mixed.  The constraints of one kind
    of one class each use their own topology key (DESIGN.md section 7)."""
    nodes = [_node(f"n{i:02d}", 32, zone=f"z{i % 4}", labels={TOPO_KEYS[q]: f"d{q}-{i % (q + 2)}" for q in range(6)}) for i in range(20)]
    keys = [HOST, ZONE] + TOPO_KEYS[:6]
    deps = [_dep("a", 8, cpu="1", ports=range(1, n_ports + 1))]
    deps += [_dep(f"b{i}", 1, cpu="1", ports=[i]) for i in range(1, n_ports + 1)]
    deps += [_dep(f"x{j}", 3, cpu="1") for j in range(8)] + [_dep(f"y{j}", 3, cpu="1") for j in range(8)]
    n_terms = 32 - n_hard - n_soft
    tsc = [_spread(keys[j % 8], 1 + j % 3, True, app=f"x{j % 8}") for j in range(n_hard)]
    tsc += [_spread(keys[(j + 3) % 8], 2, False, app=f"y{j % 8}") for j in range(n_soft)]
    aff = [{"weight": 10 + j, "podAffinityTerm": _term(HOST if j < 8 else ZONE, app=f"x{j % 8}")} for j in range((n_terms + 1) // 2)]
    anti = [{"weight": 5 + j, "podAffinityTerm": _term(ZONE if j < 8 else HOST, app=f"y{j % 8}")} for j in range(n_terms // 2)]
    deps.append(_dep("e", 24, cpu="1", topologySpreadConstraints=tsc, affinity={"podAffinity": {P: aff}, "podAntiAffinity": {P: anti}}))
    deps += [_dep(f"c{j}", 2, cpu="1", ports=[100 + j]) for j in range(8)]
    m_pref = n_mixed - 8 - 4 - 4 - 4
    deps.append(_dep("m", 10, cpu="1", ports=range(100, 108),
                     topologySpreadConstraints=[_spread(keys[j], 3, True, app=f"x{j}") for j in range(4)] +
                                               [_spread(keys[4 + j], 2, False, app=f"y{j}") for j in range(4)],
                     affinity={"podAntiAffinity": {R: [_term(HOST, app=f"y{4 + j}") for j in range(4)],
                                                   P: [{"weight": 20, "podAffinityTerm": _term(ZONE, app=f"x{j}")} for j in range(m_pref // 2)]},
                               "podAffinity": {P: [{"weight": 30, "podAffinityTerm": _term(HOST, app=f"x{4 + j % 4}") if j < 4 else
                                                    _term(ZONE, app=f"y{j % 8}")} for j in range(m_pref - m_pref // 2)]}}))
    return _objs(nodes, deps)


def commit_list_long(n_counted=70):
    """Class t is counted by n_counted hard spread constraints of other workloads, each with its own selector (tier=shared and
    l<j>=x): t's commit list holds more than 64 counters."""
    nodes = [_node(f"n{i:02d}", 32, zone=f"z{i % 3}") for i in range(30)]
    tl = {"app": "t", "tier": "shared"}
    tl.update({f"l{j}": "x" for j in range(n_counted)})
    deps = [_dep("t", 80, cpu="12", labels=tl, topologySpreadConstraints=[_spread(ZONE, 2, True, app="t")])]
    deps += [_dep(f"w{j}", 2, cpu="1", labels={"app": f"w{j}", "tier": "shared", f"l{j}": "x"},
                  topologySpreadConstraints=[_spread(HOST if j % 2 else ZONE, 8, True, tier="shared", **{f"l{j}": "x"})])
             for j in range(n_counted)]
    return _objs(nodes, deps)


def big_record():
    """One class with 20 required node-affinity terms of 8 expressions over 120 of 128 values each and 6 such preferred terms:
    thousands of selector-program words, since a first class interns the atoms so that every key's values spread over all 16
    label words.  The class is also counted by 40 spread constraints of other workloads."""
    rng = np.random.default_rng(5)
    nodes = [_node(f"n{i:02d}", 32, zone=f"z{i % 3}", labels={f"k{e}": f"v{int(rng.integers(128))}" for e in range(8)})
             for i in range(80)]
    # atom (k<e>, v<q>) = 8 q + e
    fill = {"nodeAffinity": {P: [{"weight": 1, "preference": _na_term(*[(f"k{e}", [f"v{q}"]) for e in range(8)])} for q in range(128)]}}

    def term():
        return _na_term(*[(f"k{e}", [f"v{j}" for j in sorted(rng.choice(128, 120, replace=False))]) for e in range(8)])
    labels = {"app": "big", "tier": "shared"}
    labels.update({f"l{j}": "x" for j in range(40)})
    na = {R: {"nodeSelectorTerms": [term() for _ in range(20)]}, P: [{"weight": 10 * (q + 1), "preference": term()} for q in range(6)]}
    deps = [_dep("fill", 2, affinity=fill), _dep("big", 120, cpu="20", labels=labels, affinity={"nodeAffinity": na})]
    deps += [_dep(f"w{j}", 2, cpu="1", labels={"app": f"w{j}", "tier": "shared", f"l{j}": "x"},
                  topologySpreadConstraints=[_spread(ZONE, 10, True, tier="shared", **{f"l{j}": "x"})]) for j in range(40)]
    return _objs(nodes, deps)


GI = 1 << 30


def gpu8(n_dev=8):
    """Nodes with 8 GPU-share devices of 16 GiB (some with 4, some none); pods of 1..20 slots, some with more than 15 slots of 1 GiB
    on one device (the slot word saturates at 15, the device memory must not), a pod of 64 slots."""
    nodes = []
    for i in range(16):
        g = None if i % 5 == 4 else ((n_dev, 16 * GI) if i % 3 else (4, 16 * GI))
        nodes.append(_node(f"n{i:02d}", 64, zone=f"z{i % 2}", gpus=g))
    deps = [_dep("g20", 6, cpu="1", gpu=(20, GI)), _dep("g64", 2, cpu="1", gpu=(64, GI)), _dep("g1", 30, cpu="1", gpu=(1, 10 * GI)),
            _dep("g3", 12, cpu="1", gpu=(3, 6 * GI)), _dep("g8", 6, cpu="1", gpu=(8, 9 * GI)), _dep("cpu", 40, cpu="4")]
    return _objs(nodes, deps)


BUILDERS = {"scalars8": scalars8, "atoms1024": atoms1024, "taints256": taints256, "soft_taints256": soft_taints256, "topo8": topo8,
            "entries32": entries32, "commit_list_long": commit_list_long, "big_record": big_record, "gpu8": gpu8}


def compiled(cluster, apps):
    p = simulator.plan(cluster, apps)
    return p, compile_cluster(p.nodes, p.pods, p.ctx)


def class_words(c, name):
    """The class record of the Deployment `name`."""
    cls = {int(c.pods["pod_class"][i]) for i, r in enumerate(c.pod_recs) if r.tmpl.workload_name == name}
    assert len(cls) == 1, (name, cls)
    k = cls.pop()
    off = c.pods["class_off"]
    return c.pods["class_blob"][int(off[k]):int(off[k + 1])]


def n_entries(w):
    return int(sum(int(w[x]) for x in (SCW_N_PORTS, SCW_N_PTS_HARD, SCW_N_PTS_SOFT, SCW_N_IPA_AFF, SCW_N_IPA_ANTI, SCW_N_IPA_EXIST,
                                       SCW_N_IPA_SCORE)))


def soft_counts(c):
    """[class][node] PreferNoSchedule taints the class does not tolerate (TaintToleration's count)."""
    from simon_b200.compiler import SCW_OFF_TOL
    WT, blob, off = int(c.snap_dims["n_taint_words"]), c.pods["class_blob"], c.pods["class_off"]
    soft = c.snap["taint_soft"]
    out = np.zeros((len(off) - 1, c.n_nodes), np.int64)
    for k in range(len(off) - 1):
        w = blob[int(off[k]):]
        tol = w[int(w[SCW_OFF_TOL]) + WT:int(w[SCW_OFF_TOL]) + 2 * WT].astype(np.uint64)
        for q in range(WT):
            out[k] += np.array([bin(int(x)).count("1") for x in (soft[q] & ~tol[q])])
    return out


def check_at_limit(name, c, out, fc):
    """The builder `name` reaches its limit (compiled dims / class records); the oracle's placements `out` and failure histograms
    `fc` show pods both placed and failed."""
    d = c.snap_dims
    sched = out >= 0
    assert sched.any() and (~sched).any(), name
    if name == "scalars8":
        assert d["n_scalars"] == 8 and set(c.scalar_names) == set(SCALARS)
        for k in range(8):
            assert fc[:, SFC_SCALAR0 + k].sum() > 0, f"Insufficient {c.scalar_names[k]} never decided a placement"
    elif name == "atoms1024":
        assert d["n_label_words"] == 16
        lb = c.snap["label_bits"]
        for w in range(16):
            assert ((lb[w] >> np.uint64(63)) & np.uint64(1)).any(), w      # atom 64 w + 63 (the sign bit) is set on some node
            assert (lb[w] & np.uint64(1)).any(), w
    elif name == "taints256":
        assert d["n_taint_words"] == 4
        assert c.taint_atoms == [(f"t{i:03d}", "", "NoSchedule") for i in range(256)]
        g = c.node_index("sink")
        assert (c.snap["taint_hard"][:, g] == np.uint64(2 ** 64 - 1)).all()
    elif name == "soft_taints256":
        assert d["n_taint_words"] == 4
        tt = soft_counts(c)
        assert (tt == 256).any(axis=1).sum() >= 2 and (tt == 256).sum(axis=0).max() >= 2
    elif name == "topo8":
        assert d["n_topos"] == 8 and c.topo_keys[7] == TOPO_KEYS[6]
        assert (c.snap["topo_dom"][7] < 0).any() and (c.snap["topo_dom"][7] >= 0).any()
    elif name == "entries32":
        a, e, m = class_words(c, "a"), class_words(c, "e"), class_words(c, "m")
        assert int(a[SCW_N_PORTS]) == 32 and n_entries(a) == 32 and int(a[SCW_N_ENT]) == 32
        assert (int(e[SCW_N_PTS_HARD]), int(e[SCW_N_PTS_SOFT]), n_entries(e)) == (8, 8, 32)
        assert int(m[SCW_N_PORTS]) == 8 and n_entries(m) == 32 and int(m[SCW_N_IPA_ANTI]) == 4
    elif name == "commit_list_long":
        assert int(class_words(c, "t")[SCW_N_INC]) > 64
    elif name == "big_record":
        w = class_words(c, "big")
        assert 4096 < len(w) <= 16384 and int(w[SCW_N_INC]) > 32
    elif name == "gpu8":
        assert int(c.snap["gpu_count"].max()) == 8
    return True


# ---- CPU tests ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", sorted(BUILDERS))
def test_builder_reaches_its_limit_and_oracles_agree(name):
    """At the limit: the C oracle's placements equal pyref's, the limit decides some placements."""
    p, c = compiled(*BUILDERS[name]())
    out, _score, fc, _fp = run_oracle(c)[0]
    check_at_limit(name, c, out, fc)
    np.testing.assert_array_equal(out, run_pyref(p, c), err_msg=name)


@pytest.mark.parametrize("name", sorted(BUILDERS))
def test_native_columns_equal_python_at_the_limit(name):
    from test_native_host import _diff
    assert _diff(*BUILDERS[name]()) == []


def _refused_by_both(cluster, apps, text):
    with pytest.raises(CompileError, match=text):
        compiled(cluster, apps)
    with pytest.raises(native_host.NativeHostError, match=text):
        native_host.compile_native(cluster, apps)


ONE_PAST = {
    "scalars9": (lambda: scalars8(9), "more than 8 scalar resources"),
    "atoms1025": (lambda: atoms1024(extra_atom=True), "more than 1024 label atoms"),
    "taints257": (lambda: taints256(extra_taint=True), "more than 256 distinct taints"),
    "keys8": (lambda: topo8(8), "more than 7 distinct topology keys"),
    "gpu_devices9": (lambda: gpu8(9), "has more than 8 GPUs"),
}


@pytest.mark.parametrize("case", sorted(ONE_PAST))
def test_one_past_the_limit_is_refused_by_both_compilers(case):
    build, text = ONE_PAST[case]
    _refused_by_both(*build(), text)


def _gpu_count_cluster(count):
    """One node with one 100-unit GPU-share device; a pod of `count` slots of 1 unit, then one of 36 units, then one of 1."""
    nodes = [_node("g", 64, gpus=(1, 100))]
    return _objs(nodes, [_dep("many", 1, gpu=(count, 1)), _dep("rest", 1, gpu=(1, 36)), _dep("one", 1, gpu=(1, 1))])


def test_gpu_count_64_charges_every_slot():
    """64 slots of 1 unit leave 36 of 100 free: the 36-unit pod lands, the next 1-unit pod does not (both oracles)."""
    p, c = compiled(*_gpu_count_cluster(64))
    out = run_oracle(c)[0][0]
    names = [r.tmpl.workload_name for r in c.pod_recs]
    want = {"many": 0, "rest": 0, "one": -1}
    assert [int(x) for x in out] == [want[n] for n in names]
    np.testing.assert_array_equal(out, run_pyref(p, c))


@pytest.mark.parametrize("count", [65, 70])
def test_gpu_count_above_64_is_refused_not_narrowed(count):
    """Reserve records at most 64 slots per pod: a larger gpu-count would be charged as 64 (36 + 6 units free instead of 30 at
    70 slots, so the 36-unit pod would land where the reference fails it).  Both compilers refuse it."""
    _refused_by_both(*_gpu_count_cluster(count), "at most 64 are supported")
    cluster, apps = _gpu_count_cluster(count)
    apps[0].Resource.Deployments[0]["spec"]["template"]["metadata"]["annotations"]["alibabacloud.com/gpu-mem"] = "0"
    compiled(cluster, apps)                 # not a GPU-share pod: gpu-count alone is not read
    native_host.compile_native(cluster, apps)


@pytest.mark.parametrize("name", ["scalars8", "taints256"])
def test_native_fit_error_equals_python_at_the_limit(name):
    """simon_host_plan_fit_error == simulator.format_fit_error for every class, with an empty and a synthetic histogram that names
    all 8 scalar resources."""
    cluster, apps = BUILDERS[name]()
    p, c = compiled(cluster, apps)
    L = native_host.lib()
    req = native_host.request_json(cluster, apps)
    h = C.c_void_p()
    assert L.simon_host_compile(req, len(req), C.byref(h)) == 0
    try:
        counts = np.zeros(24, np.uint32)
        counts[[1, 2, 3, 4, 5, 14, 15, 16, 17, 18, 19]] = [1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 12]
        counts[SFC_SCALAR0:SFC_SCALAR0 + 8] = np.arange(8) + 20
        seen = set()
        for i, rec in enumerate(p.pods):
            if id(rec.tmpl) in seen:
                continue
            seen.add(id(rec.tmpl))
            for cnt in (np.zeros(24, np.uint32), counts):
                out = C.c_void_p()
                assert L.simon_host_plan_fit_error(h, i, cnt.ctypes.data, C.byref(out)) == 0
                got = C.string_at(out).decode()
                L.simon_host_free(out)
                assert got == simulator.format_fit_error(c, rec, cnt)
        assert len(seen) >= 10
    finally:
        L.simon_host_plan_free(h)

