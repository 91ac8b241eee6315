"""Trace replay on the device (simon_trace_run, Engine.trace_run, Simulator.ReplayTrace).

Every run of a trace - creates placed by the batch placement variants, deletes by simon_trace_remove, samples by simon_trace_sample -
against the trace checker (tests/checkers.c), which applies one event at a time: nodes, GPU slot words, scores, failure histograms
and the samples after every event.  The own-score cache and feasible-set summary hazards a removal creates are built on purpose; random
mixes run under forced geometries, with the static-verdict cache off and on the large-cluster variant; a trace without deletes equals a
grow batch; each scenario of a batch equals the same trace alone; the C-entry refusals; ReplayTrace end to end with a sweep over k."""
import copy
import os

import numpy as np
import pytest

from simon_b200 import abi, capacity, grow, simulator, synth, trace
from simon_b200.compiler import compile_cluster
from simon_b200.engine import Engine
from simon_b200.objects import ResourceTypes
from test_grow import session
from test_trace import _node, _pod, ev

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C_, D_ = abi.TRACE_CREATE, abi.TRACE_DELETE


def _superset(kind="mix", n_nodes=120, seed=31):
    """(grow set with no candidate nodes: the session's pods, then the app's pods as the tail, and the session's node scenario)."""
    cluster, apps = synth.make_mix(seed_no=seed, n_nodes=n_nodes, n_workloads=30, max_replicas=6)
    if kind == "gpu":
        sim = session(cluster, apps)
        app = copy.deepcopy(apps[0])
        for w in app.Resource.Deployments + app.Resource.StatefulSets + app.Resource.Jobs:
            w["metadata"]["name"] += "-t"
        app.Name = "trace"
        app.Resource.DaemonSets = []
    else:
        sim = session(cluster)
        app = apps[0]
    gs = grow.build(sim, [app], [], 0)
    nodes = list(sim._plan().nodes)
    gs.scenarios = capacity.scenario_nodes(gs.compiled, nodes, len(nodes), 0, 1, [0])
    return gs


def _random_trace(gs, rng, p_delete=0.4, max_run=4):
    """Creates of every tail pod in order, interleaved with runs of deletes of random live pods (prefix pods that are not DaemonSet
    pods, and earlier creates)."""
    c = gs.compiled
    from simon_b200.scaledown import pod_guard
    guard = pod_guard(c)
    alive = [q for q in range(gs.n_prefix) if guard[q] < 0]
    events = []
    for q in range(gs.n_prefix, c.pods_dims["n_pods"]):
        if rng.random() < p_delete and alive:
            for _ in range(int(rng.integers(1, max_run + 1))):
                if not alive:
                    break
                events.append((D_, alive.pop(int(rng.integers(len(alive))))))
        events.append((C_, q))
        if guard[q] < 0:
            alive.append(q)
    return np.array(events, np.uint32)


def _check(eng, gs, events, scenarios, what=""):
    import checkers
    from oracle.binding import Oracle
    E = len(events)
    # every 7th event and the last: most runs hold several events, as without samples
    at = sorted(set(range(0, E, 7)) | {E - 1}) if E else []
    got = eng.trace_run(gs.placed, gs.n_prefix, events, scenarios, samples=at, detail=True)
    o = Oracle(gs.compiled)
    for i, nodes in enumerate(scenarios):
        want = checkers.trace(o, gs.placed, gs.n_prefix, nodes, events)
        g = got[i]
        w = f"{what} scenario {i}"
        np.testing.assert_array_equal(g["node"], want["node"], err_msg=w)
        np.testing.assert_array_equal(g["gpu_slots"], want["gpu_slots"], err_msg=w)
        if eng.record_scores:
            np.testing.assert_array_equal(g["score"], want["score"], err_msg=w)
        np.testing.assert_array_equal(g["fail_pod"], want["fail_pod"], err_msg=w)
        np.testing.assert_array_equal(g["fail_counts"], want["fail_counts"], err_msg=w)
        for k in ("n_scheduled", "n_unscheduled", "n_removed", "n_running"):
            assert g[k] == want[k], (w, k)
        np.testing.assert_array_equal(g["samples"]["event"], at, err_msg=w)
        for f, v in want["samples"].items():
            np.testing.assert_array_equal(g["samples"][f], v[at], err_msg=f"{w} sample {f}")
    o.close()
    return got


def test_random_mix_matches_checker():
    gs = _superset("mix")
    rng = np.random.default_rng(5)
    events = _random_trace(gs, rng)
    with Engine(gs.compiled, record_scores=True) as eng:
        _check(eng, gs, events, [gs.scenarios[0].nodes], "mix")
        assert eng.last_trace["run_launches"] >= eng.last_trace["runs"] > 1


def test_gpu_share_mix_matches_checker():
    gs = _superset("gpu", seed=33)
    rng = np.random.default_rng(6)
    events = _random_trace(gs, rng, p_delete=0.6)
    with Engine(gs.compiled, record_scores=True) as eng:
        got = _check(eng, gs, events, [gs.scenarios[0].nodes], "gpu")
    assert got[0]["n_removed"] > 0


@pytest.mark.parametrize("opts", [dict(cluster_ctas=2, threads_per_cta=64), dict(cluster_ctas=1, threads_per_cta=64),
                                  dict(static_cache=False), dict(force_large=True, cluster_ctas=2, threads_per_cta=64)],
                         ids=["2x64", "1x64", "no-static-cache", "large"])
def test_variants_match_checker(opts):
    gs = _superset("mix", n_nodes=300, seed=35)
    events = _random_trace(gs, np.random.default_rng(7))
    with Engine(gs.compiled, record_scores=True, **opts) as eng:
        _check(eng, gs, events, [gs.scenarios[0].nodes], str(opts))
        li = eng.last_launch()
        if opts.get("force_large"):
            assert li["large"] and li["kernel"] == "simon_place_kernel_big"
        elif "threads_per_cta" in opts:
            # 300 nodes on 2 x 64 threads: 3 slots per thread, the unrolled variant; on 1 x 64: 5 slots, the run-time one
            npt = -(-300 // (opts["cluster_ctas"] * 64))
            assert li["node_slots"] == npt and li["kernel"] == f"simon_place_kernel_256_{npt if npt <= 4 else 0}"


def _hazard(pods, events):
    """The trace on two 4000m nodes n0, n1 whose session pods `pods` are bound to them, against the checker; -> the engine's result."""
    sim = session(ResourceTypes(Nodes=[_node("n0", "4000m"), _node("n1", "4000m")], Pods=pods))
    ts = trace.build(sim, ev(*events))
    gs = grow.GrowSet(ts.compiled, ts.n_prefix, ts.placed, ts.n_base, 0, 1, ts.scenarios, [])
    with Engine(ts.compiled, record_scores=True) as eng:
        got = _check(eng, gs, ts.events, [ts.scenarios[0].nodes], "hazard")[0]
    names = [ts.compiled.node_names[g] if g >= 0 else None for g in got["node"].tolist()]
    return dict(zip((ts.compiled.pod_recs[ts.n_prefix + t].name for t in range(len(names))), names))


def test_stale_infeasible_own_state_after_delete():
    """Class A is evaluated on n0 while a blocker leaves it 1000m (its own-state entry: Fit false at one pod); the blocker leaves and a
    small pod takes n0 back to one pod with 3900m free.  A's next pod fits only n0: a stale entry would fail it."""
    mk = lambda n, cpu: _pod(n, cpu, labels={"app": n.rstrip("0123456789")})
    placed = _hazard([mk("blocker", "3000m") | {"spec": mk("blocker", "3000m")["spec"] | {"nodeName": "n0"}},
                      mk("full", "4000m") | {"spec": mk("full", "4000m")["spec"] | {"nodeName": "n1"}}],
                     [(1, trace.CREATE, mk("a1", "2000m")), (2, trace.DELETE, "default/blocker"), (3, trace.CREATE, mk("s1", "100m")),
                      (4, trace.CREATE, mk("a2", "2000m"))])
    assert placed == {"a1": None, "s1": "n0", "a2": "n0"}


def test_stale_feasible_own_state_after_delete():
    """Class A is evaluated on n0 holding one 100m pod (Fit true at one pod) and placed there; both pods leave and a 3500m pod takes n0
    back to one pod.  A's next pod fits nowhere: a stale entry would place it on n0, past its allocatable cpu."""
    mk = lambda n, cpu: _pod(n, cpu, labels={"app": n.rstrip("0123456789")})
    placed = _hazard([mk("small", "100m") | {"spec": mk("small", "100m")["spec"] | {"nodeName": "n0"}},
                      mk("full", "4000m") | {"spec": mk("full", "4000m")["spec"] | {"nodeName": "n1"}}],
                     [(1, trace.CREATE, mk("a1", "2000m")), (2, trace.DELETE, "default/small"), (2, trace.DELETE, "default/a1"),
                      (3, trace.CREATE, mk("b1", "3500m")), (4, trace.CREATE, mk("a2", "2000m"))])
    assert placed == {"a1": "n0", "b1": "n0", "a2": None}


def test_delete_run_over_hundreds_of_nodes():
    """A class whose summary is stored while it fits nowhere, revisited right after a delete run that frees all 300 nodes (an
    infeasible -> feasible flip on every node), then class switches on the freed nodes."""
    nodes = [_node(f"n{i}", "4000m") for i in range(300)]
    pods = [_pod(f"old-{i}", "3000m", labels={"app": "old"}) for i in range(300)]
    sim = session(ResourceTypes(Nodes=nodes, Pods=pods))
    mk = lambda n, cpu: _pod(n, cpu, labels={"app": "x"})
    events = [(1, trace.CREATE, mk("a0", "2000m")), (2, trace.CREATE, mk("b0", "500m")), (2, trace.CREATE, mk("a9", "2000m"))]
    events += [(3, trace.DELETE, f"default/old-{i}") for i in range(300)]
    events += [(4, trace.CREATE, mk("a1", "2000m")), (5, trace.CREATE, mk("b1", "500m")), (6, trace.DELETE, "default/b0"),
               (7, trace.CREATE, mk("c0", "3900m")), (8, trace.CREATE, mk("b2", "500m")), (9, trace.CREATE, mk("a2", "2000m"))]
    ts = trace.build(sim, ev(*events))
    with Engine(ts.compiled, record_scores=True) as eng:
        gs = grow.GrowSet(ts.compiled, ts.n_prefix, ts.placed, ts.n_base, 0, 1, ts.scenarios, [])
        got = _check(eng, gs, ts.events, [ts.scenarios[0].nodes], "delete run")
    assert got[0]["n_removed"] == 301 and got[0]["n_unscheduled"] == 2


def test_no_deletes_equals_grow_and_batch_equals_alone():
    gs = _superset("gpu", seed=37)
    events = np.array([(C_, q) for q in range(gs.n_prefix, gs.compiled.pods_dims["n_pods"])], np.uint32)
    nodes = gs.scenarios[0].nodes
    rng = np.random.default_rng(8)
    sub = [nodes, nodes[::-1].copy(), rng.permutation(nodes).astype(np.uint32)]
    with Engine(gs.compiled, record_scores=True) as eng:
        t = eng.trace_run(gs.placed, gs.n_prefix, events, sub)
        g = eng.grow_run(gs.placed, gs.n_prefix, sub)
        for a, b in zip(t, g):
            for k in ("node", "gpu_slots", "score", "fail_pod", "fail_counts", "n_scheduled", "n_unscheduled", "req_mcpu", "req_mem"):
                np.testing.assert_array_equal(a[k], b[k], err_msg=k)
        mixed = _random_trace(gs, rng)
        batch = eng.trace_run(gs.placed, gs.n_prefix, mixed, sub, samples=[0, len(mixed) - 1])
        for i, s in enumerate(sub):
            alone = eng.trace_run(gs.placed, gs.n_prefix, mixed, [s], samples=[0, len(mixed) - 1])[0]
            for k in ("node", "gpu_slots", "score", "fail_pod", "fail_counts", "n_removed", "req_mcpu"):
                np.testing.assert_array_equal(batch[i][k], alone[k], err_msg=f"{i} {k}")
            assert batch[i]["samples"].tobytes() == alone["samples"].tobytes()


def test_refusals():
    gs = _superset("mix", n_nodes=60, seed=39)
    P, n0 = gs.compiled.pods_dims["n_pods"], gs.n_prefix
    creates = [(C_, q) for q in range(n0, P)]
    from simon_b200.scaledown import pod_guard
    td = next(q for q in range(n0, P) if pod_guard(gs.compiled)[q] < 0)         # a tail pod that is not a DaemonSet pod
    with Engine(gs.compiled) as eng:
        run = lambda evs, **kw: eng.trace_run(gs.placed, n0, np.array(evs, np.uint32).reshape(-1, 2), **kw)
        for evs, msg in [([(7, n0)] + creates[1:], "unknown op"),
                         (creates[1:], "not the next tail pod"),
                         (creates + [(C_, n0)], "not the next tail pod"),
                         (creates[:-1], "creates"),
                         ([(D_, td)] + creates, "before its create"),
                         (creates + [(D_, td), (D_, td)], "again"),
                         (creates + [(D_, P)], "out of range")]:
            with pytest.raises(RuntimeError, match=msg):
                run(evs)
        with pytest.raises(RuntimeError, match="ascending"):
            run(creates, samples=[1, 0])
        with pytest.raises(RuntimeError, match="ascending"):
            run(creates, samples=[len(creates)])
        ds = [q for q in range(n0) if pod_guard(gs.compiled)[q] >= 0]
        if ds:
            with pytest.raises(RuntimeError, match="DaemonSet"):
                run([(D_, ds[0])] + creates)
        with pytest.raises(RuntimeError, match="no node"):
            eng.trace_run(gs.placed, n0, np.array(creates, np.uint32), [np.zeros(0, np.uint32)])
        with pytest.raises(RuntimeError, match="leaves out"):
            eng.trace_run(gs.placed, n0, np.array(creates, np.uint32), [np.array([0], np.uint32)])
        # another batch after a trace batch: the trace downloads refuse
        eng.trace_run(gs.placed, n0, np.array(creates, np.uint32))
        eng.grow_run(gs.placed, n0, [gs.scenarios[0].nodes], detail=False)
        from simon_b200.engine import lib
        assert lib().simon_trace_download(eng.h, 0, None, None, None, None, None) != 0


def test_replay_trace_reference_example_sweep():
    """demo_1 running the simple app, then a trace of 24 pods with lifetimes, replayed for k = 0..4 copies of newnode/demo_1; the
    session is left as it was."""
    import yaml
    from simon_b200 import apply as A
    from test_zz_grow_gpu import REF
    cfg = {"apiVersion": "simon/v1alpha1", "kind": "Config", "metadata": {"name": "c"},
           "spec": {"cluster": {"customConfig": "example/cluster/demo_1"},
                    "appList": [{"name": "simple", "path": "example/application/simple"}], "newNode": "example/newnode/demo_1"}}
    path = os.path.join(os.environ.get("TMPDIR", "/tmp"), f"trace-cfg-{os.getpid()}.yaml")
    with open(path, "w") as fh:
        fh.write(yaml.safe_dump(cfg))
    try:
        cluster, apps, new_node = A.load_config(path, base_dir=REF)
    finally:
        os.remove(path)
    sim = simulator.NewSimulator()
    sim.RunCluster(simulator.PrepareCluster(cluster))
    sim.ScheduleApp(apps[0])
    before = (sim.placements.copy(), sim.gpu_slots.copy(), sim.engine, sim.compiled)
    items = [(_pod(f"t-{i}", "4000m"), float(i), float(i + 6) if i % 3 else None) for i in range(24)]
    r = sim.ReplayTrace(trace.from_lifetimes(items), new_node=new_node, kmax=4, samples=10)
    assert sim.engine is before[2] and sim.compiled is before[3] and np.array_equal(sim.placements, before[0])
    assert len(r.PerK) == 5 and all(len(t.Samples["time"]) == 10 for t in r.PerK)
    fails = [len(t.Failures) for t in r.PerK]
    assert fails[0] > 0 and fails[-1] <= fails[0]
    # the copies' DaemonSet pods are created at the start of the scenarios they join
    creates = [t.Creates for t in r.PerK]
    assert creates[0] == 24 and creates == sorted(creates)
    if r.MinNodes >= 0:
        assert fails[r.MinNodes] == 0 and all(p.Node is not None for p in r.Pods)
        assert r.AllFromMinNodes == all(f == 0 for f in fails[r.MinNodes:])
    # each k equals the checker
    ts = trace.build(sim, trace.from_lifetimes(items), new_node, 4)
    gs = grow.GrowSet(ts.compiled, ts.n_prefix, ts.placed, ts.n_base, 4, 1, ts.scenarios, [])
    with Engine(ts.compiled, record_scores=True) as eng:
        _check(eng, gs, ts.events, [s.nodes for s in ts.scenarios], "reference")
    sim.Close()


def test_large_cluster_variant_past_20480_nodes():
    """40,000 nodes, past what the shared-memory variants hold (20,480 nodes, DESIGN.md section 3, and a 16 x 384 x 4 geometry fits a
    few thousand more on small classes): the placement launches of a trace run the large-cluster variant."""
    cluster, apps = synth.make_c2(n_nodes=40000, n_workloads=6, replicas=20, n_apps=2, seed_no=41)
    sim = session(cluster, apps[:1])
    gs = grow.build(sim, [apps[1]], [], 0)
    nodes = list(sim._plan().nodes)
    gs.scenarios = capacity.scenario_nodes(gs.compiled, nodes, len(nodes), 0, 1, [0])
    events = _random_trace(gs, np.random.default_rng(9))
    with Engine(gs.compiled, record_scores=True) as eng:
        got = _check(eng, gs, events, [gs.scenarios[0].nodes], "large")
        li = eng.last_launch()
    assert li["large"] and li["kernel"] == "simon_place_kernel_big" and li["n_nodes"] == 40000, li
    assert got[0]["n_removed"] > 0


def test_state_at_a_sample_equals_survivors_resumed():
    """On a cluster without GPU share, the state a trace leaves after event e equals compiling the pods alive then (in pod order) and
    resuming from their nodes: the creates after e, with no later deletes, land on the same nodes and fail with the same histograms."""
    cluster, apps = synth.make_mix(seed_no=43, n_nodes=120, n_workloads=30, max_replicas=6)
    for n in cluster.Nodes:
        for k in ("allocatable", "capacity"):
            for r in ("alibabacloud.com/gpu-count", "alibabacloud.com/gpu-mem"):
                n["status"][k].pop(r, None)
    sim = session(cluster)
    gs = grow.build(sim, [apps[0]], [], 0)
    p = sim._plan()
    nodes = list(p.nodes)
    gs.scenarios = capacity.scenario_nodes(gs.compiled, nodes, len(nodes), 0, 1, [0])
    c, n0, P = gs.compiled, gs.n_prefix, gs.compiled.pods_dims["n_pods"]
    full = _random_trace(gs, np.random.default_rng(10), p_delete=0.6)
    e = int(np.nonzero(full[:, 0] == C_)[0][(P - n0) // 2])          # the middle create: events [0, e) are kept
    head = full[:e]
    made = head[head[:, 0] == C_][:, 1]
    later = np.arange(int(made.max()) + 1 if len(made) else n0, P)
    events = np.concatenate([head, np.stack([np.full(len(later), C_), later], 1)]).astype(np.uint32)
    with Engine(c, record_scores=True) as eng:
        got = eng.trace_run(gs.placed, n0, events, [gs.scenarios[0].nodes], samples=[e - 1])[0]
    where = {q: int(gs.placed[q]) for q in range(n0)}
    where.update({q: int(got["node"][q - n0]) for q in range(n0, P)})
    for q in head[head[:, 0] == D_][:, 1]:
        where[int(q)] = -1
    alive = [q for q in range(int(later[0]) if len(later) else P) if where[q] >= 0]
    c2 = compile_cluster(nodes, [c.pod_recs[q] for q in alive] + [c.pod_recs[q] for q in later], p.ctx)
    prefix = np.array([c2.node_index(c.node_names[where[q]]) for q in alive], np.int32)
    with Engine(c2, record_scores=True) as eng2:
        out, _, fc, fp = eng2.schedule_resume(prefix)
    mine = [c.node_names[g] if g >= 0 else None for g in got["node"][later - n0].tolist()]
    theirs = [c2.node_names[g] if g >= 0 else None for g in out[len(alive):].tolist()]
    assert mine == theirs
    assert got["samples"]["n_running"][0] == len(alive)
    fails = {int(q): j for j, q in enumerate(got["fail_pod"].tolist())}
    later_fails = [fails[int(q)] for q in later if int(q) in fails]
    np.testing.assert_array_equal(got["fail_counts"][later_fails], fc)
    assert len(fp) == len(later_fails)


def test_refusals_of_pod_kinds():
    """Refused before any device work: a tail pod bound by spec.nodeName, a delete of a GPU-share pod of more than 15 slots, and a create
    or delete of a pod with Open-Local volumes."""
    from simon_b200.workloads import make_valid_pod_by_pod
    sim = session(ResourceTypes(Nodes=[_node("n0"), _node("n1")], Pods=[_pod("old")]))
    p = sim._plan()
    n0 = len(p.pods)
    bound = make_valid_pod_by_pod(_pod("bound", node="n0"))
    wide = make_valid_pod_by_pod(_pod("wide", "100m", ann={"alibabacloud.com/gpu-mem": "1Gi", "alibabacloud.com/gpu-count": "16"}))
    for rec, evs, msg in [(bound, [(C_, n0)], "spec.nodeName"), (wide, [(C_, n0), (D_, n0)], "slot word")]:
        c = compile_cluster(p.nodes, list(p.pods) + [rec], p.ctx)
        with Engine(c) as eng:
            with pytest.raises(RuntimeError, match=msg):
                eng.trace_run(sim.placements, n0, np.array(evs, np.uint32))
    from test_zz_grow_gpu import _case, _mixed_local
    sim, app, _ = _case("local", n_nodes=60)
    gs = grow.build(sim, [app], [], 0)
    c, n0, P = gs.compiled, gs.n_prefix, gs.compiled.pods_dims["n_pods"]
    local = np.asarray(c.storage.class_local, bool)[np.asarray(c.pods["pod_class"])]
    assert local[n0:].any()
    with Engine(c) as eng:
        with pytest.raises(RuntimeError, match="creates pod .*Open-Local"):
            eng.trace_run(gs.placed, n0, np.array([(C_, q) for q in range(n0, P)], np.uint32))
    # the same cluster with its app running: a delete of one of its pods with volumes, on a superset with no tail
    cluster, apps = _mixed_local(11, 60)
    sim = session(cluster, apps, simulator.WithOpenLocal(devices=True))
    gs = grow.build(sim, [], [], 0)
    c, n0 = gs.compiled, gs.n_prefix
    local = np.asarray(c.storage.class_local, bool)[np.asarray(c.pods["pod_class"])]
    from simon_b200.scaledown import pod_guard
    q = int(np.nonzero(local[:n0] & (pod_guard(c)[:n0] < 0))[0][0])
    with Engine(c) as eng:
        with pytest.raises(RuntimeError, match="deletes pod .*Open-Local"):
            eng.trace_run(gs.placed, n0, np.array([(D_, q)], np.uint32))
