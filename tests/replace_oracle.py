"""ctypes binding of the node-pool replacement checker (tests/replace_oracle.c; TEST INFRASTRUCTURE ONLY), used on an
oracle.binding.Oracle that holds the wave base, and OracleRunner: rolling.run_waves's runner on the CPU, for plain waves as well as
waves that join and retire nodes."""
from __future__ import annotations

import ctypes as C

import numpy as np

from checkers import build_checker
from simon_b200 import abi, rolling

_LIB = None


def lib():
    """The checker, built by the recipe of tests/checkers.py (it includes the rolling-wave and move-scope checkers)."""
    global _LIB
    if _LIB is None:
        L = C.CDLL(build_checker("replace_oracle", ["rolling_oracle.c", "moves_scope_oracle.c"]))
        L.simon_oracle_replace.restype = C.c_int
        L.simon_oracle_replace.argtypes = [C.c_void_p] * 5 + [C.c_uint32, C.c_void_p, C.c_uint32, C.c_int] + [C.c_void_p] * 13
        _LIB = L
    return _LIB


def wave(o, placement, slots, state, remain, join, apply: bool) -> dict:
    """One wave on the oracle `o` from the base it holds (placement / slots / state: updated in place with apply).  -> dict in the
    shape of one Engine.wave_run(joins=...) entry, with req_mcpu / req_mem but without the allocatable sums."""
    rm = np.ascontiguousarray(remain, dtype=np.uint32)
    jn = np.ascontiguousarray(join, dtype=np.uint32)
    P = len(placement)
    counts = np.zeros(7, np.uint32)
    z = lambda dt: np.zeros(max(P, 1), dt)                     # noqa: E731
    ev, node, score, sl, blk = z(np.uint32), z(np.int32), z(np.int64), z(np.uint32), z(np.uint32)
    jp, jnode, jscore, jsl = z(np.uint32), z(np.int32), z(np.int64), z(np.uint32)
    fc = np.zeros((max(P, 1), abi.N_FAIL_CODES), np.uint32)
    fp = z(np.uint32)
    sums = np.zeros(2, np.int64)
    rc = lib().simon_oracle_replace(o.h, placement.ctypes.data, slots.ctypes.data, state.ctypes.data, rm.ctypes.data, len(rm),
                                    jn.ctypes.data if len(jn) else None, len(jn), int(apply), counts.ctypes.data, ev.ctypes.data,
                                    node.ctypes.data, score.ctypes.data, sl.ctypes.data, blk.ctypes.data, jp.ctypes.data,
                                    jnode.ctypes.data, jscore.ctypes.data, jsl.ctypes.data, fc.ctypes.data, fp.ctypes.data,
                                    sums.ctypes.data)
    if rc != 0:
        raise RuntimeError(f"simon_oracle_replace rc={rc}")
    ne, npl, nf, nb, nv, nj, njf = (int(x) for x in counts)
    return dict(n_evicted=ne, n_placed=npl, n_unscheduled=nf, n_blocked=nb, n_vanished=nv, evicted=ev[:ne], node=node[:ne],
                score=score[:ne], gpu_slots=sl[:ne], blocked=blk[:nb], fail_counts=fc[njf:njf + nf], fail_pod=fp[njf:njf + nf],
                n_join=nj, n_join_placed=nj - njf, n_join_unscheduled=njf, join_pods=jp[:nj], join_node=jnode[:nj],
                join_score=jscore[:nj], join_gpu_slots=jsl[:nj], join_fail_counts=fc[:njf], join_fail_pod=fp[:njf],
                req_mcpu=int(sums[0]), req_mem=int(sums[1]))


class OracleRunner(rolling.WaveRunner):
    """rolling.run_waves's runner on the checker.  `o` must hold the state `placed` leaves when begin(placed, present) is called (for
    a superset: grow_oracle.grow with the present nodes).  PDB violations are counted on the host against rolling.pdb_allowed on the
    base."""

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
            r = wave(self.o, self.placed, self.slots, self.state, rl, jl, False)
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
        assert retire, "the replacement checker retires the drained nodes"
        wave(self.o, self.placed, self.slots, self.state, self.last[i], self.last_joins[i], True)

    def placement(self):
        return self.placed.copy(), self.slots.copy()
