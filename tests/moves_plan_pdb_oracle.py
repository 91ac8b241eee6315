"""ctypes binding of the migration-plan checker with a PodDisruptionBudget table (tests/moves_plan_pdb_oracle.c; TEST INFRASTRUCTURE
ONLY), used on an oracle.binding.Oracle: plan_pdb(o, moves, placement, slots, max_moves, min_gain, scope, pod_off, pod_pdb, allowed)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from checkers import load_checker


def lib():
    return load_checker("moves_plan_pdb_oracle", {
        "simon_oracle_moves_plan_pdb": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32] + [C.c_void_p] * 4 +
                                        [C.c_uint32, C.c_int32, C.c_uint32] + [C.c_void_p] * 8)})


def plan_pdb(o, moves, placement, slots, max_moves: int, min_gain: int, scope: int, pod_off, pod_pdb, allowed, class_local=None):
    """A migration plan on the oracle's current state, which it leaves in the plan's end state, honouring the PDB table: the pod -> PDB
    CSR (pod_off, pod_pdb) and each PDB's allowed disruptions on the live placement.  placement / slots: the live placement and GPU
    slot words.  -> dict(steps [n, 6] int64 (move, pod, from, to, gain, gpu slots), stop_reason, excluded, pdb_blocked, placement,
    slots, state, state_ext)."""
    L = lib()
    a = np.ascontiguousarray(moves, dtype=np.uint32).reshape(-1, 2)
    pl = np.array(placement, dtype=np.int32)
    sl = np.array(slots, dtype=np.uint32)
    loc = None if class_local is None else np.ascontiguousarray(class_local, dtype=np.uint8)
    off = np.ascontiguousarray(pod_off, dtype=np.uint32)
    ids = np.ascontiguousarray(pod_pdb, dtype=np.uint32)
    ids = ids if ids.size else np.zeros(1, np.uint32)
    al = np.ascontiguousarray(allowed, dtype=np.int32)
    n_pdbs = len(al)
    al = al if al.size else np.zeros(1, np.int32)
    steps = np.zeros((max(max_moves, 1), 6), np.int32)
    n, stop, exc, blk = C.c_uint32(0), C.c_uint32(0), C.c_uint32(0), C.c_uint32(0)
    rc = L.simon_oracle_moves_plan_pdb(o.h, scope, len(a), a.ctypes.data, pl.ctypes.data, sl.ctypes.data,
                                       None if loc is None else loc.ctypes.data, max_moves, min_gain, n_pdbs, off.ctypes.data,
                                       ids.ctypes.data, al.ctypes.data, steps.ctypes.data, C.byref(n), C.byref(stop), C.byref(exc),
                                       C.byref(blk))
    if rc != 0:
        raise RuntimeError(f"simon_oracle_moves_plan_pdb rc={rc}")
    st = steps[:n.value].astype(np.int64)
    st[:, 5] &= 0xffffffff
    return dict(steps=st, stop_reason=int(stop.value), excluded=int(exc.value), pdb_blocked=int(blk.value), placement=pl, slots=sl,
                state=o.state(), state_ext=o.state_ext())
