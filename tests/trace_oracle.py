"""ctypes binding of the trace-replay checker (tests/trace_oracle.c; TEST INFRASTRUCTURE ONLY), used on an oracle.binding.Oracle:
trace(o, placed, n_prefix, nodes, events) replays one scenario one event at a time."""
from __future__ import annotations

import ctypes as C

import numpy as np

from checkers import build_checker
from simon_b200 import abi

_LIB = None
SAMPLE_FIELDS = ("n_running", "n_failed", "idle_devices", "partial_devices", "req_mcpu", "alloc_mcpu", "req_mem", "alloc_mem",
                 "gpu_used", "gpu_total")


def lib():
    """The checker, built by the recipe of tests/checkers.py; it includes the move-scope checker for the oracle's uncommit()."""
    global _LIB
    if _LIB is None:
        L = C.CDLL(build_checker("trace_oracle", ["moves_scope_oracle.c"]))
        L.simon_oracle_trace.restype = C.c_int
        L.simon_oracle_trace.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32] + [C.c_void_p] * 7
        _LIB = L
    return _LIB


def trace(o, placed, n_prefix, nodes, events) -> dict:
    """One scenario (active nodes `nodes`, scenario order) of a trace replay on the oracle `o` from the live placement
    placed[:n_prefix]; events are (op, pod) pairs.  -> dict in the shape of one Engine.trace_run(detail=True) entry without the
    occupancy sums at the end, with samples [n_events] of every event (a dict of SAMPLE_FIELDS arrays)."""
    pl = np.ascontiguousarray(np.asarray(placed)[:n_prefix], dtype=np.int32)
    nd = np.ascontiguousarray(nodes, dtype=np.uint32)
    ev = np.ascontiguousarray(np.asarray(events, dtype=np.uint32).reshape(-1, 2))
    T = o.c.pods_dims["n_pods"] - int(n_prefix)
    E = len(ev)
    node = np.full(max(T, 1), -9, np.int32)
    score = np.zeros(max(T, 1), np.int64)
    slots = np.zeros(max(T, 1), np.uint32)
    fc = np.zeros((max(T, 1), abi.N_FAIL_CODES), np.uint32)
    fp = np.zeros(max(T, 1), np.uint32)
    counts = np.zeros(4, np.uint32)
    sm = np.zeros((max(E, 1), len(SAMPLE_FIELDS)), np.int64)
    rc = lib().simon_oracle_trace(o.h, pl.ctypes.data if len(pl) else None, int(n_prefix), nd.ctypes.data, len(nd),
                                  ev.ctypes.data if E else None, E, node.ctypes.data, score.ctypes.data, slots.ctypes.data,
                                  fc.ctypes.data, fp.ctypes.data, counts.ctypes.data, sm.ctypes.data)
    if rc != 0:
        raise RuntimeError(f"simon_oracle_trace rc={rc}")
    f = int(counts[1])
    return dict(node=node[:T], score=score[:T], gpu_slots=slots[:T], fail_counts=fc[:f], fail_pod=fp[:f], n_scheduled=int(counts[0]),
                n_unscheduled=f, n_removed=int(counts[2]), n_running=int(counts[3]),
                samples={k: sm[:E, i] for i, k in enumerate(SAMPLE_FIELDS)})
