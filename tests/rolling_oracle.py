"""ctypes binding of the rolling-wave checker (tests/rolling_oracle.c; TEST INFRASTRUCTURE ONLY), used on an oracle.binding.Oracle
that holds the wave base, and OracleRunner: rolling.plan_rolling's runner on the CPU."""
from __future__ import annotations

import ctypes as C

import numpy as np

from checkers import build_checker
from simon_b200 import abi, rolling

_LIB = None


def lib():
    """The checker, built by the recipe of tests/checkers.py (it includes the move-scope checker for uncommit)."""
    global _LIB
    if _LIB is None:
        L = C.CDLL(build_checker("rolling_oracle", ["moves_scope_oracle.c"]))
        L.simon_oracle_wave.restype = C.c_int
        L.simon_oracle_wave.argtypes = [C.c_void_p] * 4 + [C.c_uint32, C.c_int] + [C.c_void_p] * 9
        _LIB = L
    return _LIB


def wave(o, placement, slots, remain, apply: bool) -> dict:
    """One wave on the oracle `o` from the base it holds (placement / slots: its placement, updated in place with apply).  -> dict in the
    shape of one Engine.wave_run entry, with req_mcpu / req_mem but without the allocatable sums."""
    rm = np.ascontiguousarray(remain, dtype=np.uint32)
    P = len(placement)
    counts = np.zeros(5, np.uint32)
    ev = np.zeros(max(P, 1), np.uint32)
    node = np.zeros(max(P, 1), np.int32)
    score = np.zeros(max(P, 1), np.int64)
    sl = np.zeros(max(P, 1), np.uint32)
    blk = np.zeros(max(P, 1), np.uint32)
    fc = np.zeros((max(P, 1), abi.N_FAIL_CODES), np.uint32)
    fp = np.zeros(max(P, 1), np.uint32)
    sums = np.zeros(2, np.int64)
    rc = lib().simon_oracle_wave(o.h, placement.ctypes.data, slots.ctypes.data, rm.ctypes.data, len(rm), int(apply), counts.ctypes.data,
                                 ev.ctypes.data, node.ctypes.data, score.ctypes.data, sl.ctypes.data, blk.ctypes.data, fc.ctypes.data,
                                 fp.ctypes.data, sums.ctypes.data)
    if rc != 0:
        raise RuntimeError(f"simon_oracle_wave rc={rc}")
    ne, npl, nf, nb, nv = (int(x) for x in counts)
    return dict(n_evicted=ne, n_placed=npl, n_unscheduled=nf, n_blocked=nb, n_vanished=nv, evicted=ev[:ne], node=node[:ne],
                score=score[:ne], gpu_slots=sl[:ne], blocked=blk[:nb], fail_counts=fc[:nf], fail_pod=fp[:nf],
                req_mcpu=int(sums[0]), req_mem=int(sums[1]))


class OracleRunner(rolling.WaveRunner):
    """rolling.plan_rolling's runner on the checker.  `o` must hold the state `placed` leaves when begin(placed) is called (an
    Oracle right after its schedule()).  PDB violations are counted on the host against rolling.pdb_allowed on the base."""

    def __init__(self, o, pdbs=None):
        self.o, self.pdbs = o, pdbs
        c = o.c
        self.ac, self.am = np.asarray(c.snap["alloc_mcpu"]), np.asarray(c.snap["alloc_mem"])
        self.runs = []

    def begin(self, placed):
        self.placed = np.array(placed, dtype=np.int32)
        self.slots = np.array(self.o.gpu_slot_words(), dtype=np.uint32)

    def run(self, remain_lists):
        self.last = [np.asarray(r, dtype=np.uint32) for r in remain_lists]
        self.runs.append(len(remain_lists))
        allowed = rolling.pdb_allowed(self.pdbs, self.placed) if self.pdbs is not None else None
        out = []
        for rl in self.last:
            r = wave(self.o, self.placed, self.slots, rl, False)
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

    def commit(self, i: int):
        wave(self.o, self.placed, self.slots, self.last[i], True)

    def placement(self):
        return self.placed.copy(), self.slots.copy()
