"""ctypes binding of the grow-batch checker (tests/grow_oracle.c; TEST INFRASTRUCTURE ONLY), used on an oracle.binding.Oracle:
grow(o, placed, n_prefix, nodes) and the oracle's state afterwards through the Oracle's own accessors."""
from __future__ import annotations

import ctypes as C

import numpy as np

from checkers import build_checker
from simon_b200 import abi

_LIB = None


def lib():
    """The checker, built by the recipe of tests/checkers.py (it includes no other checker source)."""
    global _LIB
    if _LIB is None:
        L = C.CDLL(build_checker("grow_oracle", []))
        L.simon_oracle_grow.restype = C.c_int
        L.simon_oracle_grow.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32] + [C.c_void_p] * 6
        _LIB = L
    return _LIB


def grow(o, placed, n_prefix, nodes) -> dict:
    """One grow scenario (active nodes `nodes`, scenario order) on the oracle `o` (oracle.binding.Oracle; Oracle(c, open_local=True)
    runs Open-Local) from the live placement placed[:n_prefix].  -> dict in the shape of one Engine.grow_run(detail=True) entry, with
    n_scheduled / n_unscheduled and without the occupancy sums."""
    pl = np.ascontiguousarray(np.asarray(placed)[:n_prefix], dtype=np.int32)
    nd = np.ascontiguousarray(nodes, dtype=np.uint32)
    T = o.c.pods_dims["n_pods"] - int(n_prefix)
    node = np.zeros(max(T, 1), np.int32)
    score = np.zeros(max(T, 1), np.int64)
    slots = np.zeros(max(T, 1), np.uint32)
    fc = np.zeros((max(T, 1), abi.N_FAIL_CODES), np.uint32)
    fp = np.zeros(max(T, 1), np.uint32)
    nf = C.c_uint32(0)
    rc = lib().simon_oracle_grow(o.h, pl.ctypes.data if len(pl) else None, int(n_prefix), nd.ctypes.data, len(nd), node.ctypes.data,
                                 score.ctypes.data, slots.ctypes.data, fc.ctypes.data, fp.ctypes.data, C.byref(nf))
    if rc != 0:
        raise RuntimeError(f"simon_oracle_grow rc={rc}")
    node = node[:T]
    f = nf.value
    sched = (node >= 0) & (np.asarray(o.c.pods["pod_fixed_node"])[int(n_prefix):] == -1)
    return dict(node=node, score=score[:T], gpu_slots=slots[:T], fail_counts=fc[:f], fail_pod=fp[:f], n_unscheduled=f,
                n_scheduled=int(sched.sum()))
