"""ctypes binding of the move-scope checker (tests/moves_scope_oracle.c; TEST INFRASTRUCTURE ONLY), used on an
oracle.binding.Oracle: moves_score(o, moves, placement, scope) and gpu_used(o)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(_HERE)
_LIB = None
CFLAGS = ["-O2", "-fPIC", "-shared", "-std=c11", "-D_GNU_SOURCE", "-pthread", "-Wall", "-Wextra", "-ffp-contract=off", "-fno-fast-math"]


def build() -> str:
    so = os.path.join(ROOT, "build", "libmoves_scope_oracle.so")
    srcs = [os.path.join(_HERE, "moves_scope_oracle.c"), os.path.join(ROOT, "oracle", "simon_oracle.c"),
            os.path.join(ROOT, "include", "simon_gpu.h")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in srcs):
        os.makedirs(os.path.dirname(so), exist_ok=True)
        subprocess.check_call([os.environ.get("CC", "gcc")] + CFLAGS + ["-o", so, srcs[0], "-lm"])
    return so


def lib():
    global _LIB
    if _LIB is None:
        L = C.CDLL(build())
        L.simon_oracle_moves_score_scoped.restype = C.c_int
        L.simon_oracle_moves_score_scoped.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32] + [C.c_void_p] * 6
        L.simon_oracle_gpu_used.argtypes = [C.c_void_p, C.c_void_p]
        _LIB = L
    return _LIB


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
