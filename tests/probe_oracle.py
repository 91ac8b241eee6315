"""ctypes binding of the headroom-probe checker (tests/probe_oracle.c; TEST INFRASTRUCTURE ONLY), used on an oracle.binding.Oracle:
probe(o, placed, pod, max_replicas) and the oracle's state afterwards through the Oracle's own accessors."""
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
        L = C.CDLL(build_checker("probe_oracle", []))
        L.simon_oracle_probe.restype = C.c_int
        L.simon_oracle_probe.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32] + [C.c_void_p] * 5
        _LIB = L
    return _LIB


def probe(o, placed, pod, max_replicas) -> dict:
    """One probe on the oracle `o` (oracle.binding.Oracle; Oracle(c, open_local=True) runs Open-Local) from the live placement
    `placed`.  -> dict in the shape of one Engine.probe_run(detail=True) entry, without the occupancy sums."""
    pl = np.ascontiguousarray(placed, dtype=np.int32)
    R = int(max_replicas)
    n = C.c_uint32(0)
    node = np.zeros(max(R, 1), np.int32)
    score = np.zeros(max(R, 1), np.int64)
    slots = np.zeros(max(R, 1), np.uint32)
    fc = np.zeros(abi.N_FAIL_CODES, np.uint32)
    rc = lib().simon_oracle_probe(o.h, pl.ctypes.data, int(pod), R, C.byref(n), node.ctypes.data, score.ctypes.data,
                                  slots.ctypes.data, fc.ctypes.data)
    if rc != 0:
        raise RuntimeError(f"simon_oracle_probe rc={rc}")
    k = n.value
    return dict(n_placed=k, stop_reason=abi.PROBE_STOP_UNSCHEDULABLE if k < R else abi.PROBE_STOP_MAX_REPLICAS,
                node=node[:k], score=score[:k], gpu_slots=slots[:k], fail_counts=fc)
