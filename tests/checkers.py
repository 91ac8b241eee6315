"""The build recipe of the C checkers under tests/ (TEST INFRASTRUCTURE ONLY): tests/<name>.c includes oracle/simon_oracle.c and
becomes build/lib<name>.so; each checker's module (moves_scope_oracle.py, ...) wraps its entry points."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(_HERE)
# no FMA contraction, no fast math: the checkers round as the oracle does
CFLAGS = ["-O2", "-fPIC", "-shared", "-std=c11", "-D_GNU_SOURCE", "-pthread", "-Wall", "-Wextra", "-ffp-contract=off", "-fno-fast-math"]
# checker -> the other checker sources under tests/ it includes
CHECKERS = {
    "moves_scope_oracle": [],
    "moves_plan_oracle": ["moves_scope_oracle.c"],
    "moves_plan_pdb_oracle": ["moves_scope_oracle.c"],
    "drain_oracle": [],
}
_LOADED = {}


def build_checker(name: str, sources) -> str:
    """Compile tests/<name>.c into build/lib<name>.so unless that is newer than it, the tests/ files `sources`, the oracle and the
    header."""
    so = os.path.join(ROOT, "build", f"lib{name}.so")
    srcs = [os.path.join(_HERE, f) for f in [f"{name}.c"] + list(sources)] + \
        [os.path.join(ROOT, "oracle", "simon_oracle.c"), os.path.join(ROOT, "include", "simon_gpu.h")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in srcs):
        os.makedirs(os.path.dirname(so), exist_ok=True)
        subprocess.check_call([os.environ.get("CC", "gcc")] + CFLAGS + ["-o", so, srcs[0], "-lm"])
    return so


def load_checker(name: str, signatures: dict) -> C.CDLL:
    """The checker `name`, built if needed, with the restype and argtypes of `signatures` ({entry point: (restype, argtypes)})."""
    if name not in _LOADED:
        L = C.CDLL(build_checker(name, CHECKERS[name]))
        for fn, (restype, argtypes) in signatures.items():
            f = getattr(L, fn)
            f.restype, f.argtypes = restype, argtypes
        _LOADED[name] = L
    return _LOADED[name]
