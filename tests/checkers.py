"""The CPU checkers (TEST INFRASTRUCTURE ONLY): tests/checkers.c includes oracle/simon_oracle.c and becomes
build/libsimon_checkers.so.  This module builds it, declares every entry point once and wraps them for tests that run on an
oracle.binding.Oracle; OracleRunner is rolling.run_waves's runner on the wave checker."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from simon_b200 import abi, rolling

_HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(_HERE)
# no FMA contraction, no fast math: the checkers round as the oracle does
CFLAGS = ["-O2", "-fPIC", "-shared", "-std=c11", "-D_GNU_SOURCE", "-pthread", "-Wall", "-Wextra", "-ffp-contract=off", "-fno-fast-math"]
SOURCES = [os.path.join(_HERE, "checkers.c"), os.path.join(ROOT, "oracle", "simon_oracle.c"), os.path.join(ROOT, "include", "simon_gpu.h")]
LIB = os.path.join(ROOT, "build", "libsimon_checkers.so")

_P, _U32 = C.c_void_p, C.c_uint32
# entry point -> (restype, argtypes)
_SIGNATURES = {
    "simon_oracle_last_reasons": (None, [_P, _P]),
    "simon_oracle_drain": (C.c_int, [_P, _P, _P, _U32] + [_P] * 9),
    "simon_oracle_grow": (C.c_int, [_P, _P, _U32, _P, _U32] + [_P] * 6),
    "simon_oracle_probe": (C.c_int, [_P, _P, _U32, _U32] + [_P] * 5),
    "simon_oracle_trace": (C.c_int, [_P, _P, _U32, _P, _U32, _P, _U32] + [_P] * 7),
    "simon_oracle_moves_score_scoped": (C.c_int, [_P, _U32, _U32] + [_P] * 6),
    "simon_oracle_gpu_used": (None, [_P, _P]),
    "simon_oracle_moves_plan": (C.c_int, [_P, _U32, _U32] + [_P] * 4 + [_U32, C.c_int32, _U32] + [_P] * 8),
    "simon_oracle_wave": (C.c_int, [_P] * 5 + [_U32, _P, _U32, C.c_int, C.c_int] + [_P] * 13),
}
_LIB = None


def build() -> str:
    """Compile tests/checkers.c into build/libsimon_checkers.so unless that is newer than it, the oracle and the header."""
    if not os.path.exists(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(s) for s in SOURCES):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        subprocess.check_call([os.environ.get("CC", "gcc")] + CFLAGS + ["-o", LIB, SOURCES[0], "-lm"])
    return LIB


def lib() -> C.CDLL:
    """The checker library, built if needed, with every entry point's restype and argtypes."""
    global _LIB
    if _LIB is None:
        L = C.CDLL(build())
        for fn, (restype, argtypes) in _SIGNATURES.items():
            f = getattr(L, fn)
            f.restype, f.argtypes = restype, argtypes
        _LIB = L
    return _LIB


def _check(name: str, rc: int):
    if rc != 0:
        raise RuntimeError(f"{name} rc={rc}")


def last_reasons(o) -> np.ndarray:
    """The filter verdict of every node for the last pod that reached the oracle's scheduler: 0 feasible, else a bitmask of
    simon_fail_code."""
    N = o.c.n_nodes
    out = np.zeros(max(N, 1), np.uint32)
    lib().simon_oracle_last_reasons(o.h, out.ctypes.data)
    return out[:N]


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
    fc = np.zeros((max(P, 1), abi.N_FAIL_CODES), np.uint32)
    fp = np.zeros(max(P, 1), np.uint32)
    loc = None if class_local is None else np.ascontiguousarray(class_local, dtype=np.uint8)
    _check("simon_oracle_drain", lib().simon_oracle_drain(
        o.h, pl.ctypes.data, rm.ctypes.data, len(rm), None if loc is None else loc.ctypes.data, counts.ctypes.data, ev.ctypes.data,
        node.ctypes.data, score.ctypes.data, slots.ctypes.data, blk.ctypes.data, fc.ctypes.data, fp.ctypes.data))
    ne, npl, nf, nb, nv = (int(x) for x in counts)
    return dict(n_evicted=ne, n_placed=npl, n_unscheduled=nf, n_blocked=nb, n_vanished=nv, evicted=ev[:ne], node=node[:ne],
                score=score[:ne], gpu_slots=slots[:ne], blocked=blk[:nb], fail_counts=fc[:nf], fail_pod=fp[:nf])


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
    _check("simon_oracle_grow", lib().simon_oracle_grow(
        o.h, pl.ctypes.data if len(pl) else None, int(n_prefix), nd.ctypes.data, len(nd), node.ctypes.data, score.ctypes.data,
        slots.ctypes.data, fc.ctypes.data, fp.ctypes.data, C.byref(nf)))
    node = node[:T]
    f = nf.value
    sched = (node >= 0) & (np.asarray(o.c.pods["pod_fixed_node"])[int(n_prefix):] == -1)
    return dict(node=node, score=score[:T], gpu_slots=slots[:T], fail_counts=fc[:f], fail_pod=fp[:f], n_unscheduled=f,
                n_scheduled=int(sched.sum()))


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
    _check("simon_oracle_probe", lib().simon_oracle_probe(o.h, pl.ctypes.data, int(pod), R, C.byref(n), node.ctypes.data,
                                                          score.ctypes.data, slots.ctypes.data, fc.ctypes.data))
    k = n.value
    return dict(n_placed=k, stop_reason=abi.PROBE_STOP_UNSCHEDULABLE if k < R else abi.PROBE_STOP_MAX_REPLICAS,
                node=node[:k], score=score[:k], gpu_slots=slots[:k], fail_counts=fc)


TRACE_SAMPLE_FIELDS = ("n_running", "n_failed", "idle_devices", "partial_devices", "req_mcpu", "alloc_mcpu", "req_mem", "alloc_mem",
                       "gpu_used", "gpu_total")


def trace(o, placed, n_prefix, nodes, events) -> dict:
    """One scenario (active nodes `nodes`, scenario order) of a trace replay on the oracle `o` from the live placement
    placed[:n_prefix]; events are (op, pod) pairs.  -> dict in the shape of one Engine.trace_run(detail=True) entry without the
    occupancy sums at the end, with samples [n_events] of every event (a dict of TRACE_SAMPLE_FIELDS arrays)."""
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
    sm = np.zeros((max(E, 1), len(TRACE_SAMPLE_FIELDS)), np.int64)
    _check("simon_oracle_trace", lib().simon_oracle_trace(
        o.h, pl.ctypes.data if len(pl) else None, int(n_prefix), nd.ctypes.data, len(nd), ev.ctypes.data if E else None, E,
        node.ctypes.data, score.ctypes.data, slots.ctypes.data, fc.ctypes.data, fp.ctypes.data, counts.ctypes.data, sm.ctypes.data))
    f = int(counts[1])
    return dict(node=node[:T], score=score[:T], gpu_slots=slots[:T], fail_counts=fc[:f], fail_pod=fp[:f], n_scheduled=int(counts[0]),
                n_unscheduled=f, n_removed=int(counts[2]), n_running=int(counts[3]),
                samples={k: sm[:E, i] for i, k in enumerate(TRACE_SAMPLE_FIELDS)})


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
    _check("simon_oracle_moves_score_scoped", lib().simon_oracle_moves_score_scoped(
        o.h, scope, n, a.ctypes.data, pl.ctypes.data, None if loc is None else loc.ctypes.data, gain.ctypes.data, code.ctypes.data,
        slots.ctypes.data))
    return gain[:n], code[:n], (slots[:n] if scope & 1 else None)


def gpu_used(o) -> np.ndarray:
    """The oracle's GPU-share device memory in use, [8][N]."""
    N = o.c.n_nodes
    out = np.zeros((8, max(N, 1)), np.int64)
    lib().simon_oracle_gpu_used(o.h, out.ctypes.data)
    return out[:, :N]


def plan_pdb(o, moves, placement, slots, max_moves: int, min_gain: int, scope: int, pod_off, pod_pdb, allowed, class_local=None):
    """A migration plan on the oracle's current state, which it leaves in the plan's end state, honouring the PDB table: the pod -> PDB
    CSR (pod_off, pod_pdb) and each PDB's allowed disruptions on the live placement.  placement / slots: the live placement and GPU
    slot words.  -> dict(steps [n, 6] int64 (move, pod, from, to, gain, gpu slots), stop_reason, excluded, pdb_blocked, placement,
    slots, state, state_ext)."""
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
    _check("simon_oracle_moves_plan", lib().simon_oracle_moves_plan(
        o.h, scope, len(a), a.ctypes.data, pl.ctypes.data, sl.ctypes.data, None if loc is None else loc.ctypes.data, max_moves,
        min_gain, n_pdbs, off.ctypes.data, ids.ctypes.data, al.ctypes.data, steps.ctypes.data, C.byref(n), C.byref(stop),
        C.byref(exc), C.byref(blk)))
    st = steps[:n.value].astype(np.int64)
    st[:, 5] &= 0xffffffff
    return dict(steps=st, stop_reason=int(stop.value), excluded=int(exc.value), pdb_blocked=int(blk.value), placement=pl, slots=sl,
                state=o.state(), state_ext=o.state_ext())


def plan(o, moves, placement, slots, max_moves: int, min_gain: int = 1, scope: int = 0, class_local=None):
    """plan_pdb without a PDB table.  -> the same dict without pdb_blocked."""
    r = plan_pdb(o, moves, placement, slots, max_moves, min_gain, scope, [0], [], [], class_local)
    del r["pdb_blocked"]
    return r


def wave(o, placement, slots, remain, apply: bool = False, state=None, join=None, retire: bool = False) -> dict:
    """One wave on the oracle `o` from the base it holds (placement / slots / state: its placement, slot words and node states, updated
    in place with apply; state None: every node present), joining the nodes `join` first.  apply with retire: the joined nodes
    become present and the drained ones retire; apply without it: the drained nodes come back.  -> dict in the shape of one
    Engine.wave_run(joins=...) entry, with req_mcpu / req_mem but without the allocatable sums."""
    rm = np.ascontiguousarray(remain, dtype=np.uint32)
    jn = np.ascontiguousarray(() if join is None else join, dtype=np.uint32)
    P = len(placement)
    counts = np.zeros(7, np.uint32)
    z = lambda dt: np.zeros(max(P, 1), dt)                     # noqa: E731
    ev, node, score, sl, blk = z(np.uint32), z(np.int32), z(np.int64), z(np.uint32), z(np.uint32)
    jp, jnode, jscore, jsl = z(np.uint32), z(np.int32), z(np.int64), z(np.uint32)
    fc = np.zeros((max(P, 1), abi.N_FAIL_CODES), np.uint32)
    fp = z(np.uint32)
    sums = np.zeros(2, np.int64)
    _check("simon_oracle_wave", lib().simon_oracle_wave(
        o.h, placement.ctypes.data, slots.ctypes.data, None if state is None else state.ctypes.data, rm.ctypes.data, len(rm),
        jn.ctypes.data if len(jn) else None, len(jn), int(apply), int(retire), counts.ctypes.data, ev.ctypes.data, node.ctypes.data,
        score.ctypes.data, sl.ctypes.data, blk.ctypes.data, jp.ctypes.data, jnode.ctypes.data, jscore.ctypes.data, jsl.ctypes.data,
        fc.ctypes.data, fp.ctypes.data, sums.ctypes.data))
    ne, npl, nf, nb, nv, nj, njf = (int(x) for x in counts)
    return dict(n_evicted=ne, n_placed=npl, n_unscheduled=nf, n_blocked=nb, n_vanished=nv, evicted=ev[:ne], node=node[:ne],
                score=score[:ne], gpu_slots=sl[:ne], blocked=blk[:nb], fail_counts=fc[njf:njf + nf], fail_pod=fp[njf:njf + nf],
                n_join=nj, n_join_placed=nj - njf, n_join_unscheduled=njf, join_pods=jp[:nj], join_node=jnode[:nj],
                join_score=jscore[:nj], join_gpu_slots=jsl[:nj], join_fail_counts=fc[:njf], join_fail_pod=fp[:njf],
                req_mcpu=int(sums[0]), req_mem=int(sums[1]))


class OracleRunner(rolling.WaveRunner):
    """rolling.run_waves's runner on the wave checker, for plain waves as well as waves that join and retire nodes.  `o` must hold the
    state `placed` leaves when begin(placed, present) is called (an Oracle right after its schedule(); for a superset, grow with the
    present nodes).  PDB violations are counted on the host against rolling.pdb_allowed on the base."""

    def __init__(self, o, pdbs=None):
        self.o, self.pdbs = o, pdbs
        c = o.c
        self.ac, self.am = np.asarray(c.snap["alloc_mcpu"]), np.asarray(c.snap["alloc_mem"])
        self.runs = []

    def begin(self, placed, present=None):
        self.placed = np.array(placed, dtype=np.int32)
        self.slots = np.array(self.o.gpu_slot_words(), dtype=np.uint32)
        self.slots[self.placed < 0] = 0
        n = self.o.c.n_nodes
        self.state = np.ones(n, np.uint8) if present is None else np.asarray(present, dtype=bool).astype(np.uint8)

    def run(self, remain_lists, joins=None):
        self.last = [np.asarray(r, dtype=np.uint32) for r in remain_lists]
        self.last_joins = [np.zeros(0, np.uint32)] * len(self.last) if joins is None else [np.asarray(j, np.uint32) for j in joins]
        self.runs.append(len(remain_lists))
        allowed = rolling.pdb_allowed(self.pdbs, self.placed) if self.pdbs is not None else None
        out = []
        for rl, jl in zip(self.last, self.last_joins):
            r = wave(self.o, self.placed, self.slots, rl, state=self.state, join=jl)
            idx = rl.astype(np.int64)
            r.update(alloc_mcpu=int(self.ac[idx].sum()), alloc_mem=int(self.am[idx].sum()))
            vp, vc = [], []
            if allowed is not None:
                cnt = {}
                for q in r["evicted"].tolist():
                    for j in self.pdbs.pod_pdb[self.pdbs.pod_off[q]:self.pdbs.pod_off[q + 1]].tolist():
                        cnt[j] = cnt.get(j, 0) + 1
                for j in sorted(cnt):
                    if cnt[j] > allowed[j]:
                        vp.append(j)
                        vc.append(cnt[j])
            r.update(n_pdb_violated=len(vp), pdb_violated=np.array(vp, np.uint32), pdb_evicted=np.array(vc, np.uint32))
            out.append(r)
        return out

    def commit(self, i: int, retire: bool = False):
        wave(self.o, self.placed, self.slots, self.last[i], True, self.state, self.last_joins[i], retire)

    def placement(self):
        return self.placed.copy(), self.slots.copy()
