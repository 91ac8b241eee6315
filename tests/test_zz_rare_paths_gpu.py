"""Kernel paths that no earlier GPU test reaches, written after the round's GPU minutes were spent (first GPU run = the
driver's; the file sorts last so that a failure here cannot mask the rest of the suite under `pytest -x`):

  * soft spread over a topology with more domains than the per-decision bitmask holds (SCW_ANY_TABLE: per-domain tables
    in global memory instead of the 6 x 64-bit presence words);
  * the kernel variant with a run-time number of nodes per thread at <= 256 threads (NPT_T = 0: more than 4 nodes per thread),
    and next to it the unrolled 3-slot variant at 320 threads; tests/test_zz_kernel_variants_gpu.py covers every variant,
    simon_place_kernel_320_0 (more than 4 nodes per thread at 257-320 threads) included.
"""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
pytestmark = pytest.mark.gpu


def rack_cluster(n_nodes=1200, n_workloads=24, replicas=12, seed_no=31):
    """C2-shaped cluster whose nodes carry a `rack` label with n_nodes/2 values; workloads spread over racks."""
    from simon_b200 import synth
    cluster, apps = synth.make_c2(n_nodes=n_nodes, n_workloads=n_workloads, replicas=replicas, seed_no=seed_no)
    for i, n in enumerate(cluster.Nodes):
        n["metadata"]["labels"]["rack"] = f"rack-{i // 2:04d}"
    for w, d in enumerate(apps[0].Resource.Deployments):
        name = d["metadata"]["name"]
        cons = [{"maxSkew": 1 + w % 3, "topologyKey": "rack", "whenUnsatisfiable": "ScheduleAnyway",
                 "labelSelector": {"matchLabels": {"app": name}}}]
        if w % 4 == 0:
            cons.append({"maxSkew": 2, "topologyKey": "topology.kubernetes.io/zone", "whenUnsatisfiable": "ScheduleAnyway",
                         "labelSelector": {"matchLabels": {"app": name}}})
        if w % 5 == 0:
            cons[0]["whenUnsatisfiable"] = "DoNotSchedule"
        d["spec"]["template"]["spec"]["topologySpreadConstraints"] = cons
    return cluster, apps


def _compile(cluster, apps):
    from simon_b200 import simulator
    from simon_b200.compiler import compile_cluster
    p = simulator.plan(cluster, apps)
    return p, compile_cluster(p.nodes, p.pods, p.ctx)


def _cmp(c, **kw):
    from simon_b200.engine import Engine
    from util import run_oracle
    (ref, rscore, rfc, rfp), rstate = run_oracle(c)
    with Engine(c, device=0, record_scores=True, **kw) as eng:
        out, score, fc, fp = eng.schedule()
        st = eng.state()
    np.testing.assert_array_equal(out, ref)
    sched = ref >= 0
    np.testing.assert_array_equal(score[sched & (rscore > 0)], rscore[sched & (rscore > 0)])
    np.testing.assert_array_equal(fc, rfc)
    for k in rstate:
        np.testing.assert_array_equal(st[k], rstate[k], err_msg=k)


def test_soft_spread_over_a_topology_larger_than_the_bitmask():
    from simon_b200.compiler import SCW_ANY_TABLE
    p, c = _compile(*rack_cluster())
    blob, off = c.pods["class_blob"], c.pods["class_off"]
    assert any(blob[off[i] + SCW_ANY_TABLE] for i in range(len(off) - 1))       # the table method is really selected
    _cmp(c)


@pytest.mark.parametrize("cs,tpb", [(1, 64), (1, 320), (1, 128)])
def test_runtime_nodes_per_thread_variants(cs, tpb):
    """700 nodes on one CTA: 11 and 6 node slots per thread at 64 and 128 threads (run-time slot count), 3 at 320 threads."""
    from util import make_case
    p, c = make_case("c3", n_nodes=700, n_workloads=80, replicas=12, n_apps=2, seed_no=13)
    _cmp(c, cluster_ctas=cs, threads_per_cta=tpb)
    kernel = {64: "simon_place_kernel_256_0", 128: "simon_place_kernel_256_0", 320: "simon_place_kernel_320_3"}[tpb]
    from simon_b200.engine import Engine
    with Engine(c, device=0, cluster_ctas=cs, threads_per_cta=tpb) as eng:
        eng.schedule(download=False)
        assert eng.last_launch()["kernel"] == kernel
