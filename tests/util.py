"""Shared helpers for the tests: build a plan + compiled cluster from a synthetic config."""
import os
import re

import numpy as np

from simon_b200 import simulator, synth
from simon_b200.compiler import compile_cluster


def make_case(kind="c3", **kw):
    cluster, apps = {"c3": synth.make_c3, "c2": synth.make_c2, "mix": synth.make_mix, "same_key": synth.make_same_key}[kind](**kw)
    p = simulator.plan(cluster, apps)
    c = compile_cluster(p.nodes, p.pods, p.ctx)
    return p, c


KERNEL_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "open-simulator_b200", "csrc", "simon_kernel.cu")


def compiled_kernels(prefix):
    """The kernels named prefix* that simon_kernel.cu defines: the entries of its SIMON_PLACE_VARIANTS list, from which the kernels
    and the host's variant table are generated, and any kernel defined outside that list."""
    src = open(KERNEL_SRC).read()
    m = re.search(r"^#define SIMON_PLACE_VARIANTS\(X\)((?:.*\\\n)*.*)", src, re.M)
    assert m, "simon_kernel.cu has no SIMON_PLACE_VARIANTS list"
    names = set(re.findall(r"\bX\((\w+),", m.group(1)))
    names |= set(re.findall(r"\b(\w+)\(const __grid_constant__", src))
    return {n for n in names if n.startswith(prefix)}


def run_oracle(c):
    from oracle.binding import Oracle
    o = Oracle(c)
    out = o.schedule()
    st = o.state()
    o.close()
    return out, st


def run_oracle_ext(c):
    """run_oracle plus the state the parity of extended resources and GPU share needs: (out, state, state_ext, GPU slot words)."""
    from oracle.binding import Oracle
    o = Oracle(c)
    out = o.schedule()
    res = out, o.state(), o.state_ext(), o.gpu_slot_words()
    o.close()
    return res


def assert_ext_equal(eng, rext, rslots, what=""):
    """Engine.state_ext() and the per-pod GPU-share device slots equal the oracle's."""
    ext = eng.state_ext()
    for k in rext:
        np.testing.assert_array_equal(ext[k], rext[k], err_msg=f"{what} {k}")
    np.testing.assert_array_equal(eng.gpu_slot_words(), rslots, err_msg=f"{what} GPU slots")


def run_pyref(p, c):
    from oracle.pyref import PyRef
    ref = PyRef(c.node_objs, services=p.ctx.services, replicasets=p.ctx.replicasets, statefulsets=p.ctx.statefulsets,
                creation_order=c.node_orig_index)
    return np.array(ref.run([x.tmpl.pod for x in p.pods], [x.node_name for x in p.pods]), dtype=np.int32)


def _sfc_of(reason: str, scalar_names) -> int:
    from simon_b200 import abi
    fixed = {"static": abi.SFC_STATIC, "ports": abi.SFC_PORTS, "Too many pods": abi.SFC_TOO_MANY_PODS, "Insufficient cpu": abi.SFC_CPU,
             "Insufficient memory": abi.SFC_MEM, "Insufficient ephemeral-storage": abi.SFC_EPH, "pts-missing": abi.SFC_PTS_MISSING,
             "pts-skew": abi.SFC_PTS_SKEW, "ipa-aff": abi.SFC_IPA_AFF, "ipa-anti": abi.SFC_IPA_ANTI, "ipa-exist": abi.SFC_IPA_EXIST,
             "gpu": abi.SFC_GPU, "local": abi.SFC_LOCAL}
    if reason in fixed:
        return fixed[reason]
    assert reason.startswith("Insufficient "), reason
    return abi.SFC_SCALAR0 + list(scalar_names).index(reason[len("Insufficient "):])


def pyref_walk(p, c, open_local=None, ref_out=None):
    """PyRef.schedule_one pod by pod, as PyRef.run commits: -> (node [P], winning total [P], feasible node count [P], failure
    histogram [P][N_FAIL_CODES] in simon_fail_code columns).  Pods bound by spec.nodeName get their node, total 0 and no failure.
    open_local: PyRef's Open-Local setting, (storage classes, devices).  ref_out: a list that receives the PyRef afterwards."""
    from oracle.pyref import PyRef
    from simon_b200 import abi
    ref = PyRef(c.node_objs, services=p.ctx.services, replicasets=p.ctx.replicasets, statefulsets=p.ctx.statefulsets,
                creation_order=c.node_orig_index, open_local=open_local)
    if ref_out is not None:
        ref_out.append(ref)
    P = len(p.pods)
    node, total, feas = np.full(P, -1, np.int32), np.zeros(P, np.int64), np.zeros(P, np.int64)
    hist = np.zeros((P, abi.N_FAIL_CODES), np.uint32)
    for i, rec in enumerate(p.pods):
        pod = rec.tmpl.pod
        if rec.node_name:
            ns = ref.by_name.get(rec.node_name)
            if ns is None:
                node[i] = -2
            else:
                ref.commit(pod, ns, reserve_gpu=False)
                node[i] = ref.nodes.index(ns)
            continue
        detail: dict = {}
        idx, best, h = ref.schedule_one(pod, detail)
        node[i], feas[i] = idx, len(detail)
        if idx >= 0:
            total[i] = best
            ref.commit(pod, ref.nodes[idx])
        for reason, n in h.items():
            hist[i, _sfc_of(reason, c.scalar_names)] += n
    return node, total, feas, hist


def assert_matches_walk(walk, out, score, fail_counts, fail_pod, what=""):
    """A run's nodes, winning totals (pods with one feasible node are not scored: the engine and the oracle record 0) and per-pod
    failure histograms equal pyref_walk's."""
    node, total, feas, hist = walk
    bad = np.nonzero(out != node)[0]
    assert len(bad) == 0, f"{what}: {len(bad)} placements differ, first pods {bad[:6]}: got {out[bad[:6]]} pyref {node[bad[:6]]}"
    scored = (node >= 0) & (feas > 1)
    bad = np.nonzero(scored & (score != total))[0]
    assert len(bad) == 0, f"{what}: totals differ at pods {bad[:6]}: got {score[bad[:6]]} pyref {total[bad[:6]]}"
    failed = np.nonzero(node == -1)[0]
    np.testing.assert_array_equal(np.asarray(fail_pod), failed, err_msg=f"{what}: failing pods")
    np.testing.assert_array_equal(np.asarray(fail_counts), hist[failed], err_msg=f"{what}: failure histograms")


class CompiledArrays:
    """A compiled cluster restored from stored columns (what Engine / Oracle consume: the arrays of include/simon_gpu.h)."""

    def __init__(self, npz):
        import json
        self.snap = {k[6:]: npz[k] for k in npz.files if k.startswith("snap__")}
        self.pods = {k[6:]: npz[k] for k in npz.files if k.startswith("pods__")}
        self.snap_dims = json.loads(bytes(npz["snap_dims"]).decode())
        self.pods_dims = json.loads(bytes(npz["pods_dims"]).decode())
        self.facts = json.loads(bytes(npz["facts"]).decode()) if "facts" in npz.files else {}
        self.n_nodes = int(self.snap_dims["n_nodes"])
        self.node_names = self.facts.get("node_names", [str(i) for i in range(self.n_nodes)])
