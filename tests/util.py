"""Shared helpers for the tests: build a plan + compiled cluster from a synthetic config."""
import os
import re

import numpy as np

from simon_b200 import simulator, synth
from simon_b200.compiler import compile_cluster


def make_case(kind="c3", **kw):
    cluster, apps = {"c3": synth.make_c3, "c2": synth.make_c2, "mix": synth.make_mix}[kind](**kw)
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
