"""PodTopologySpread constraints of one kind that share a topology key, on the CPU: the C oracle against the object-level
restatement (oracle/pyref.py), on seeded clusters (synth.make_same_key) and on hand-built known answers.

The reference counts matching pods per topology PAIR (key, value): every DoNotSchedule constraint adds its own selector's matches
into the pair it shares with the others on its key, and the global minimum is taken per key over those sums
(podtopologyspread/filtering.go:215-265).  ScheduleAnyway does the same for non-hostname keys (scoring.go:57-105), but only the
constraint that first creates a pair grows its topology size, so a later constraint on the key weighs log(0 + 2); hostname
constraints count their own selector on the node and are not summed (scoring.go:183-210).  A pod that k of the key's selectors
match therefore adds k to the key's count.
"""
import numpy as np
import pytest

from simon_b200 import abi, simulator, synth
from simon_b200.compiler import SCW_N_ENT, SCW_OFF_ENT, compile_cluster
from simon_b200.objects import AppResource, ResourceTypes
from util import assert_matches_walk, make_case, pyref_walk

ZONE, HOST = "topology.kubernetes.io/zone", "kubernetes.io/hostname"
SEEDS = [1, 2, 3, 4, 5, 6, 7, 8]


def entry_rows(c):
    """Every class's entry table rows (include/simon_gpu.h SCW_OFF_ENT), [n][8]."""
    blob, off = c.pods["class_blob"], c.pods["class_off"]
    rows = [np.asarray(blob[int(off[k]) + int(blob[int(off[k]) + SCW_OFF_ENT]):][:8 * int(blob[int(off[k]) + SCW_N_ENT])]).reshape(-1, 8)
            for k in range(len(off) - 1)]
    return np.concatenate(rows) if rows else np.zeros((0, 8), np.int64)


def oracle_run(c, dump_pod=None):
    """(out, score, fail_counts, fail_pod, state[, per-node pts and totals of pod dump_pod])"""
    from oracle.binding import Oracle
    o = Oracle(c)
    if dump_pod is None:
        res = o.schedule() + (o.state(),)
    else:
        o.enable_dump()
        res = o.schedule(0, dump_pod + 1) + (o.state(), o.last_detail()[1])
    o.close()
    return res


# ---- seeded clusters -------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("seed", SEEDS)
def test_c_oracle_matches_pyref_same_key(seed):
    """Node, winning total and failure histogram of every pod against a per-pod PyRef.schedule_one walk."""
    p, c = make_case("same_key", seed_no=seed)
    out, score, fc, fp, _st = oracle_run(c)
    assert_matches_walk(pyref_walk(p, c), out, score, fc, fp, f"seed {seed}")
    assert (out >= 0).sum() > len(out) // 2


def test_same_key_generator_covers_its_cases():
    """Over the seeds: summed counters (a class whose commit increments one counter several times), size-0 ScheduleAnyway
    entries, both kinds on one key in one class, each of hostname / zone / rack, failures of both spread reasons."""
    mult = size0 = both = 0
    keys, reasons = set(), set()
    for seed in SEEDS:
        p, c = make_case("same_key", seed_no=seed)
        e = entry_rows(c)
        mult += int((e[:, 5] > 1).sum())
        size0 += int(((e[:, 0] == 2) & (e[:, 6] == abi.SOFT_SIZE0_WOFF)).sum())
        for r in p.pods:
            tsc = r.tmpl.pod["spec"].get("topologySpreadConstraints") or []
            kinds = {}
            for t in tsc:
                kinds.setdefault(t["topologyKey"], set()).add(t["whenUnsatisfiable"])
                keys.add(t["topologyKey"])
            both += any(len(v) == 2 for v in kinds.values())
        _o, _s, fc, _fp, _st = oracle_run(c)
        reasons |= {b for b in (abi.SFC_PTS_MISSING, abi.SFC_PTS_SKEW) if fc[:, b].any()}
    assert mult > 0 and size0 > 0 and both > 0
    assert keys == {HOST, ZONE, "example.com/rack"} and reasons == {abi.SFC_PTS_MISSING, abi.SFC_PTS_SKEW}


# ---- known answers ---------------------------------------------------------------------------------------------------------

def _node(name, zone, cores):
    return synth._node(name, cores, zone, "", 100)


def _running(name, node, labels):
    return {"apiVersion": "v1", "kind": "Pod", "metadata": {"name": name, "namespace": "default", "labels": labels},
            "spec": {"nodeName": node, "containers": [{"name": "c", "image": "x", "resources": {"requests": {"cpu": "100m", "memory": "400Mi"}}}]}}


def _pod(name, labels, cons, cpu_m=100):
    return {"apiVersion": "v1", "kind": "Pod", "metadata": {"name": name, "namespace": "default", "labels": labels},
            "spec": {"topologySpreadConstraints": cons,
                     "containers": [{"name": "c", "image": "x", "resources": {"requests": {"cpu": f"{cpu_m}m", "memory": f"{4 * cpu_m}Mi"}}}]}}


def _spread(key, when, skew, sel):
    return {"maxSkew": skew, "topologyKey": key, "whenUnsatisfiable": when, "labelSelector": {"matchLabels": sel}}


def kat_case(name):
    """-> (plan, compiled) of one known-answer cluster (see the tests below for what each is and what it must give)."""
    cluster, pods = ResourceTypes(), []
    ax, by, xy = {"a": "x"}, {"b": "y"}, {"a": "x", "b": "y"}
    if name == "sum_blocks":
        for z, cores in (("A", 4), ("B", 4), ("C", 40)):
            cluster.Nodes.extend([_node(f"{z.lower()}1", z, cores), _node(f"{z.lower()}2", z, cores)])
        cons = [_spread(ZONE, "DoNotSchedule", 2, ax), _spread(ZONE, "DoNotSchedule", 2, by)]
        pods = [_pod(f"p{i:02d}", xy, cons, 100 + 10 * i) for i in range(24)]
    elif name == "critical_path":
        cluster.Nodes.extend([_node("a1", "A", 4), _node("b1", "B", 4), _node("c1", "C", 4)])
        cluster.Pods.extend([_running("ra", "a1", ax), _running("rb", "b1", by), _running("rc", "c1", xy)])
        cons = [_spread(ZONE, "DoNotSchedule", 1, ax), _spread(ZONE, "DoNotSchedule", 1, by)]
        pods = [_pod(f"p{i}", xy, cons) for i in range(3)]
    elif name == "soft_zone_log2":
        cluster.Nodes.extend([_node("a1", "A", 8), _node("b1", "B", 8), _node("c1", "C", 8)])
        cluster.Pods.extend([_running("rb", "b1", ax), _running("rc1", "c1", ax), _running("rc2", "c1", by), _running("rc3", "c1", by)])
        pods = [_pod("p", {"app": "t"}, [_spread(ZONE, "ScheduleAnyway", 5, ax), _spread(ZONE, "ScheduleAnyway", 5, by)])]
    elif name == "soft_hostname":
        cluster.Nodes.extend([_node("h1", "A", 8), _node("h2", "A", 8), _node("h3", "A", 8)])
        cluster.Pods.extend([_running("r2", "h2", ax), _running("r3", "h3", xy)])
        pods = [_pod("p", {"app": "t"}, [_spread(HOST, "ScheduleAnyway", 1, ax), _spread(HOST, "ScheduleAnyway", 1, by)])]
    else:
        raise KeyError(name)
    app = AppResource("kat", ResourceTypes())
    app.Resource.Pods.extend(pods)
    p = simulator.plan(cluster, [app])
    return p, compile_cluster(p.nodes, p.pods, p.ctx)


def _zone_of(c, out):
    return [c.node_objs[int(i)]["metadata"]["labels"][ZONE] for i in out]


def test_summed_count_blocks_a_zone_each_constraint_alone_allows():
    """Six nodes, two per zone; zone C's have ten times the CPU, so the scores are far from equal across zones.  24 pods labelled
    a=x, b=y with rising CPU requests, each with two DoNotSchedule zone constraints (maxSkew 2) selecting a=x and b=y: every placed
    pod adds 2 to its zone's summed count, and a zone passes only if count + 1 - min <= 2, i.e. count <= min + 1, so (counts being
    even) only the zones at the minimum pass.  After pod 3k + 1 went to some zone, that zone is at min + 2: the sum blocks it although
    either constraint alone (count min + 1, skew 2) would allow it.  So every three consecutive pods 3k, 3k+1, 3k+2 go to three
    different zones, and all 24 are placed, 8 per zone."""
    p, c = kat_case("sum_blocks")
    out, score, fc, fp, _st = oracle_run(c)
    assert_matches_walk(pyref_walk(p, c), out, score, fc, fp, "sum_blocks")
    z = _zone_of(c, out)
    assert (out >= 0).all()
    for k in range(8):
        assert sorted(z[3 * k:3 * k + 3]) == ["A", "B", "C"], (k, z)


def test_minimum_is_taken_over_the_summed_counts():
    """Zones A (a1), B (b1) and C (c1), equal nodes.  Running: a=x on a1, b=y on b1, a=x,b=y on c1 (equal requests): summed zone
    counts 1, 1, 2, min 1.  Three pods a=x,b=y with DoNotSchedule zone constraints a=x and b=y (maxSkew 1):
      p0: A 1+1-1 = 1, B 1, C 2+1-1 = 2 > 1: A or B, whose nodes score the same; the tie goes to a1, first in node order
          -> A (counts 3, 1, 2);
      p1: min 1: A 3 > 1, B 1, C 2 > 1 -> B (counts 3, 3, 2);
      p2: min 2: A 2 > 1, B 2 > 1, C 1 -> C.
    Per-constraint counts would give minimum 0 for both selectors and leave p0 with no zone at all."""
    p, c = kat_case("critical_path")
    out, score, fc, fp, _st = oracle_run(c)
    assert_matches_walk(pyref_walk(p, c), out, score, fc, fp, "critical_path")
    assert [c.node_names[int(i)] for i in out[-3:]] == ["a1", "b1", "c1"]


def test_second_schedule_anyway_constraint_on_a_key_weighs_log_2():
    """Zones A, B, C, one equal node each.  Running: a=x on b1; a=x, b=y, b=y on c1: summed zone counts 0, 1, 3.  The pod has
    ScheduleAnyway zone constraints a=x and b=y, maxSkew 5 each.  The first creates all three pairs: size 3, weight ln 5; the
    second creates none: size 0, weight ln 2.  Raw scores f2i(n ln 5 + 4 + n ln 2 + 4) = 8, 10 (10.30), 14 (14.91), normalised
    100 (14 + 8 - raw) // 14 = 100, 85, 57; a1 wins.  (Both weights ln 5 would give 8, 11, 17 and 100, 82, 47.)"""
    p, c = kat_case("soft_zone_log2")
    P = len(p.pods)
    out, score, fc, fp, _st, sc = oracle_run(c, dump_pod=P - 1)
    assert_matches_walk(pyref_walk(p, c), out, score, fc, fp, "soft_zone_log2")
    idx = [c.node_names.index(n) for n in ("a1", "b1", "c1")]
    assert [int(sc[i][4]) for i in idx] == [100, 85, 57]
    assert c.node_names[int(out[-1])] == "a1"


def test_two_hostname_schedule_anyway_constraints_stay_unsummed():
    """Nodes h1, h2, h3.  Running: a=x on h2; a=x,b=y on h3.  The pod has ScheduleAnyway hostname constraints a=x and b=y (maxSkew 1):
    each counts its own selector on the node and has size 3 (weight ln 5): raw f2i(0) = 0, f2i(ln 5) = 1, f2i(2 ln 5) = 3,
    normalised 100, 66, 0; h1 wins.  (Summed like a zone key, with the second at size 0, they would give 0, 2, 4 and 100, 50, 0.)"""
    p, c = kat_case("soft_hostname")
    P = len(p.pods)
    out, score, fc, fp, _st, sc = oracle_run(c, dump_pod=P - 1)
    assert_matches_walk(pyref_walk(p, c), out, score, fc, fp, "soft_hostname")
    idx = [c.node_names.index(n) for n in ("h1", "h2", "h3")]
    assert [int(sc[i][4]) for i in idx] == [100, 66, 0]
    assert c.node_names[int(out[-1])] == "h1"


def test_pyref_detail_agrees_with_the_known_answers():
    """The restatement's own per-node spread scores give the same numbers as the two ScheduleAnyway known answers."""
    from oracle.pyref import PyRef
    for name, nodes, want in (("soft_zone_log2", ("a1", "b1", "c1"), [100, 85, 57]), ("soft_hostname", ("h1", "h2", "h3"), [100, 66, 0])):
        p, c = kat_case(name)
        ref = PyRef(c.node_objs, creation_order=c.node_orig_index)
        for rec in p.pods[:-1]:
            ref.commit(rec.tmpl.pod, ref.by_name[rec.node_name], reserve_gpu=False)
        detail: dict = {}
        ref.schedule_one(p.pods[-1].tmpl.pod, detail)
        assert [detail[ref.nodes.index(ref.by_name[n])]["pts"] for n in nodes] == want, name


def test_spread_bound_counts_multiplicity(monkeypatch):
    """The compile-time bound on ScheduleAnyway counts (pods x constraints x ln(nodes + 2) < 2^31 - 2) counts a constraint once per
    selector of its key that a class matches: four zone constraints that all match their own pods count sixteen times.  With the
    bound lowered to 10 pods x 8 x ln 6, ten such pods on four nodes pass it once per constraint (4) and not with the
    multiplicity (16)."""
    import math
    from simon_b200 import compiler
    cluster = ResourceTypes()
    cluster.Nodes.extend([_node(f"n{i}", f"z{i % 2}", 4) for i in range(4)])
    xy = {"a": "x", "b": "y"}
    cons = [_spread(ZONE, "ScheduleAnyway", 1, sel) for sel in ({"a": "x"}, {"b": "y"}, xy, {"a": "x"})]
    app = AppResource("a", ResourceTypes())
    app.Resource.Pods.extend(_pod(f"p{i}", xy, cons) for i in range(10))
    p = simulator.plan(cluster, [app])
    compile_cluster(p.nodes, p.pods, p.ctx)
    monkeypatch.setattr(compiler, "PTS_COUNTS_MAX", 10 * 8 * math.log(6))
    with pytest.raises(compiler.CompileError, match="2\\^31"):
        compile_cluster(p.nodes, p.pods, p.ctx)
