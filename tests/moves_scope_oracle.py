"""ctypes binding of the move-scope checker (tests/moves_scope_oracle.c; TEST INFRASTRUCTURE ONLY), used on an
oracle.binding.Oracle: moves_score(o, moves, placement, scope) and gpu_used(o)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from checkers import load_checker


def lib():
    return load_checker("moves_scope_oracle", {
        "simon_oracle_moves_score_scoped": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32] + [C.c_void_p] * 6),
        "simon_oracle_gpu_used": (None, [C.c_void_p, C.c_void_p])})


def moves_score(o, moves, placement, scope: int = 0, class_local=None):
    """Candidate moves [(pod, target)] on the oracle's current state under a move scope (abi.MOVES_SCOPE_* bits).
    -> (gain, code, gpu_slots); gpu_slots is None unless GPU share is in scope.  class_local: per class 1 = Open-Local volumes."""
    a = np.ascontiguousarray(moves, dtype=np.uint32).reshape(-1, 2)
    pl = np.ascontiguousarray(placement, dtype=np.int32)
    n = len(a)
    gain = np.zeros(max(n, 1), np.int32)
    code = np.zeros(max(n, 1), np.uint32)
    slots = np.zeros(max(n, 1), np.uint32)
    loc = None if class_local is None else np.ascontiguousarray(class_local, dtype=np.uint8)
    rc = lib().simon_oracle_moves_score_scoped(o.h, scope, n, a.ctypes.data, pl.ctypes.data, None if loc is None else loc.ctypes.data,
                                               gain.ctypes.data, code.ctypes.data, slots.ctypes.data)
    if rc != 0:
        raise RuntimeError(f"simon_oracle_moves_score_scoped rc={rc}")
    return gain[:n], code[:n], (slots[:n] if scope & 1 else None)


def gpu_used(o) -> np.ndarray:
    """The oracle's GPU-share device memory in use, [8][N]."""
    N = o.c.n_nodes
    out = np.zeros((8, max(N, 1)), np.int64)
    lib().simon_oracle_gpu_used(o.h, out.ctypes.data)
    return out[:, :N]
