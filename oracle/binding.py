"""ctypes binding of oracle/libsimon_oracle.so (TEST INFRASTRUCTURE ONLY — see oracle/simon_oracle.c)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from simon_b200 import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def build(force: bool = False) -> str:
    so = os.path.join(_HERE, "libsimon_oracle.so")
    src = os.path.join(_HERE, "simon_oracle.c")
    hdr = os.path.join(_HERE, "..", "include", "simon_gpu.h")
    if force or not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.check_call(["make", "-C", _HERE, "-B", "libsimon_oracle.so"], stdout=subprocess.DEVNULL)
    return so


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        _LIB.simon_oracle_create.restype = C.c_void_p
        _LIB.simon_oracle_create.argtypes = [C.c_void_p, C.c_void_p]
        _LIB.simon_oracle_destroy.argtypes = [C.c_void_p]
        _LIB.simon_oracle_reset.argtypes = [C.c_void_p]
        _LIB.simon_oracle_set_active.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
        _LIB.simon_oracle_enable_dump.argtypes = [C.c_void_p]
        _LIB.simon_oracle_last_detail.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        _LIB.simon_oracle_schedule.restype = C.c_int
        _LIB.simon_oracle_schedule.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p,
                                               C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
        _LIB.simon_oracle_state.argtypes = [C.c_void_p] + [C.c_void_p] * 6
        _LIB.simon_oracle_state_ext.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        _LIB.simon_oracle_gpu_slots.restype = C.c_int
        _LIB.simon_oracle_gpu_slots.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]
        _LIB.simon_oracle_moves_score.restype = C.c_int
        _LIB.simon_oracle_moves_score.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        _LIB.simon_oracle_set_threads.restype = C.c_int
        _LIB.simon_oracle_set_threads.argtypes = [C.c_void_p, C.c_int]
        _LIB.simon_oracle_set_storage.restype = C.c_int
        _LIB.simon_oracle_set_storage.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        _LIB.simon_oracle_storage_state.restype = C.c_int
        _LIB.simon_oracle_storage_state.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    return _LIB


class Oracle:
    def __init__(self, compiled, threads: int = 1, open_local: bool = False):
        """open_local: run Open-Local (Filter, Score, Bind) on the storage tables of a cluster compiled with open_local=True,
        and with its devices when it was compiled with local_devices=True; without it the oracle has no Open-Local."""
        self.c = compiled
        self.snap, self.pods, self._keep = abi.marshal(compiled)
        self.h = lib().simon_oracle_create(C.byref(self.snap), C.byref(self.pods))
        if not self.h:
            raise MemoryError("simon_oracle_create failed")
        self.open_local = open_local
        if open_local:
            st = compiled.storage
            if st is None:
                raise ValueError("Oracle(open_local=True) needs a cluster compiled with open_local=True")
            # the oracle reads these arrays for its whole life: they are kept with it
            self.storage, self._storage_keep = abi.marshal_storage(st)
            self.devices, self._devices_keep = abi.marshal_devices(st) if st.devices else (None, [])
            rc = lib().simon_oracle_set_storage(self.h, C.byref(self.storage),
                                                C.byref(self.devices) if self.devices is not None else None)
            if rc != 0:
                self.close()
                raise RuntimeError(f"simon_oracle_set_storage rc={rc}")
        self.threads = 1
        if threads > 1:
            self.set_threads(threads)

    def set_threads(self, n: int) -> int:
        """Share the per-node loops between n host threads (spin-waiting pool); placements do not depend on n."""
        self.threads = int(lib().simon_oracle_set_threads(self.h, int(n)))
        return self.threads

    def close(self):
        if self.h:
            lib().simon_oracle_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset(self):
        lib().simon_oracle_reset(self.h)

    def set_active(self, nodes=None):
        if nodes is None:
            lib().simon_oracle_set_active(self.h, None, 0)
        else:
            a = np.ascontiguousarray(nodes, dtype=np.uint32)
            lib().simon_oracle_set_active(self.h, a.ctypes.data, len(a))

    def schedule(self, first=0, count=None, max_fail=None):
        P = self.c.pods_dims["n_pods"]
        count = P - first if count is None else count
        max_fail = count if max_fail is None else max_fail
        out_node = np.full(count, -9, np.int32)
        out_score = np.zeros(count, np.int64)
        fail_counts = np.zeros((max(max_fail, 1), abi.N_FAIL_CODES), np.uint32)
        fail_pod = np.zeros(max(max_fail, 1), np.uint32)
        n_fail = C.c_uint32(0)
        rc = lib().simon_oracle_schedule(self.h, first, count, out_node.ctypes.data, out_score.ctypes.data,
                                         fail_counts.ctypes.data, fail_pod.ctypes.data, max_fail, C.byref(n_fail))
        if rc != 0:
            raise RuntimeError(f"simon_oracle_schedule rc={rc}")
        nf = min(n_fail.value, max_fail)
        return out_node, out_score, fail_counts[:nf], fail_pod[:nf]

    def enable_dump(self):
        lib().simon_oracle_enable_dump(self.h)

    def last_detail(self):
        N = self.c.n_nodes
        code = np.zeros(N, np.int32)
        sc = np.zeros((N, 10), np.int64)
        lib().simon_oracle_last_detail(self.h, code.ctypes.data, sc.ctypes.data)
        return code, sc

    def moves_score(self, moves, placement):
        """Candidate moves [(pod, target)] on the oracle's CURRENT state; placement[pod] = node the pod runs on (or < 0)."""
        a = np.ascontiguousarray(moves, dtype=np.uint32).reshape(-1, 2)
        pl = np.ascontiguousarray(placement, dtype=np.int32)
        gain = np.zeros(max(len(a), 1), np.int32)
        code = np.zeros(max(len(a), 1), np.uint32)
        rc = lib().simon_oracle_moves_score(self.h, len(a), a.ctypes.data, pl.ctypes.data, gain.ctypes.data, code.ctypes.data)
        if rc != 0:
            raise RuntimeError(f"simon_oracle_moves_score rc={rc}")
        return gain[:len(a)], code[:len(a)]

    def state(self):
        N = self.c.n_nodes
        arrs = [np.zeros(N, np.int64) for _ in range(5)] + [np.zeros(N, np.int32)]
        lib().simon_oracle_state(self.h, *[a.ctypes.data for a in arrs])
        return dict(zip(["req_mcpu", "req_mem", "req_eph", "nz_mcpu", "nz_mem", "num_pods"], arrs))

    def state_ext(self):
        """Engine.state_ext's columns: req_scalar [K][N] and GPU-share device memory in use gpu_used [8][N]."""
        N, K = self.c.n_nodes, int(self.c.snap_dims["n_scalars"])
        rs = np.zeros((max(K, 1), max(N, 1)), np.int64)
        gu = np.zeros((8, max(N, 1)), np.int64)
        lib().simon_oracle_state_ext(self.h, rs.ctypes.data, gu.ctypes.data)
        return dict(req_scalar=rs[:K, :N], gpu_used=gu[:, :N])

    def gpu_slot_words(self, first=0, count=None):
        """Engine.gpu_slot_words: per pod 4 bits per device = the GPU-share slots Reserve gave it there."""
        P = self.c.pods_dims["n_pods"]
        count = P - first if count is None else count
        a = np.zeros(max(count, 1), np.uint32)
        rc = lib().simon_oracle_gpu_slots(self.h, first, count, a.ctypes.data)
        if rc != 0:
            raise RuntimeError(f"simon_oracle_gpu_slots rc={rc}")
        return a[:count]

    def storage_state(self):
        """Open-Local state (Oracle(open_local=True)): (VG requested [V][N], allocated device slot masks [N] or None without
        devices), as Engine.storage_state / Engine.device_state report them."""
        st = self.c.storage
        V, N = st.n_vgs, self.c.n_nodes
        vg = np.zeros(max(V * N, 1), np.int64)
        dev = np.zeros(max(N, 1), np.uint32)
        rc = lib().simon_oracle_storage_state(self.h, vg.ctypes.data, dev.ctypes.data)
        if rc != 0:
            raise RuntimeError(f"simon_oracle_storage_state rc={rc}")
        return vg[:V * N].reshape(V, N), (dev[:N] if st.devices else None)
