"""ctypes binding of the migration-plan checker (tests/moves_plan_oracle.c; TEST INFRASTRUCTURE ONLY), used on an
oracle.binding.Oracle: plan(o, moves, placement, slots, max_moves, min_gain, scope)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from checkers import load_checker


def lib():
    return load_checker("moves_plan_oracle", {
        "simon_oracle_moves_plan": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32] + [C.c_void_p] * 4 + [C.c_uint32, C.c_int32] +
                                    [C.c_void_p] * 4)})


STEP_FIELDS = ("move", "pod", "from", "to", "gain", "gpu_slots")


def plan(o, moves, placement, slots, max_moves: int, min_gain: int = 1, scope: int = 0, class_local=None):
    """A migration plan on the oracle's current state, which it leaves in the plan's end state.  placement / slots: the live
    placement and GPU slot words.  -> dict(steps [n, 6] int64 (move, pod, from, to, gain, gpu slots), stop_reason, excluded,
    placement, slots, state, state_ext)."""
    a = np.ascontiguousarray(moves, dtype=np.uint32).reshape(-1, 2)
    pl = np.array(placement, dtype=np.int32)
    sl = np.array(slots, dtype=np.uint32)
    loc = None if class_local is None else np.ascontiguousarray(class_local, dtype=np.uint8)
    steps = np.zeros((max(max_moves, 1), 6), np.int32)
    n, stop, exc = C.c_uint32(0), C.c_uint32(0), C.c_uint32(0)
    rc = lib().simon_oracle_moves_plan(o.h, scope, len(a), a.ctypes.data, pl.ctypes.data, sl.ctypes.data,
                                       None if loc is None else loc.ctypes.data, max_moves, min_gain, steps.ctypes.data,
                                       C.byref(n), C.byref(stop), C.byref(exc))
    if rc != 0:
        raise RuntimeError(f"simon_oracle_moves_plan rc={rc}")
    st = steps[:n.value].astype(np.int64)
    st[:, 5] &= 0xffffffff
    return dict(steps=st, stop_reason=int(stop.value), excluded=int(exc.value), placement=pl, slots=sl,
                state=o.state(), state_ext=o.state_ext())
