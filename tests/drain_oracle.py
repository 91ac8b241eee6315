"""ctypes binding of the drain checker (tests/drain_oracle.c; TEST INFRASTRUCTURE ONLY), used on an oracle.binding.Oracle:
drain(o, placed, remain, class_local) and the oracle's state afterwards through the Oracle's own accessors."""
from __future__ import annotations

import ctypes as C

import numpy as np

from checkers import load_checker


def lib():
    return load_checker("drain_oracle", {
        "simon_oracle_drain": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32] + [C.c_void_p] * 9)})


def drain(o, placed, remain, class_local=None) -> dict:
    """One drain on the oracle `o` (oracle.binding.Oracle): the live placement `placed`, the remaining nodes in their order.
    -> dict in the shape of one Engine.drain_run(detail=True) entry, without the occupancy sums."""
    pl = np.ascontiguousarray(placed, dtype=np.int32)
    rm = np.ascontiguousarray(remain, dtype=np.uint32)
    P = len(pl)
    counts = np.zeros(5, np.uint32)
    ev = np.zeros(max(P, 1), np.uint32)
    node = np.zeros(max(P, 1), np.int32)
    score = np.zeros(max(P, 1), np.int64)
    slots = np.zeros(max(P, 1), np.uint32)
    blk = np.zeros(max(P, 1), np.uint32)
    fc = np.zeros((max(P, 1), 24), np.uint32)
    fp = np.zeros(max(P, 1), np.uint32)
    loc = None if class_local is None else np.ascontiguousarray(class_local, dtype=np.uint8)
    rc = lib().simon_oracle_drain(o.h, pl.ctypes.data, rm.ctypes.data, len(rm), None if loc is None else loc.ctypes.data,
                                  counts.ctypes.data, ev.ctypes.data, node.ctypes.data, score.ctypes.data, slots.ctypes.data,
                                  blk.ctypes.data, fc.ctypes.data, fp.ctypes.data)
    if rc != 0:
        raise RuntimeError(f"simon_oracle_drain rc={rc}")
    ne, npl, nf, nb, nv = (int(x) for x in counts)
    return dict(n_evicted=ne, n_placed=npl, n_unscheduled=nf, n_blocked=nb, n_vanished=nv, evicted=ev[:ne], node=node[:ne],
                score=score[:ne], gpu_slots=slots[:ne], blocked=blk[:nb], fail_counts=fc[:nf], fail_pod=fp[:nf])
