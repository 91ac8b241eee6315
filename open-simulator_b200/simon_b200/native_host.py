"""ctypes binding of the NATIVE host side (csrc/simon_host.cpp, inside libsimon_gpu.so): the snapshot compiler and
simulator.Simulate() as C-ABI calls taking the objects as JSON — what the Go shim calls (go/gpu_cgo.go).

    compile_native(cluster, apps)  -> NativeCompiled   (same column names / dims as compiler.Compiled: the Python compiler is the
                                                        test-side mirror; tests/test_native_host.py compares the two)
    simulate_native(cluster, apps) -> dict             (simon_host_simulate's result JSON, parsed)

Reference seams: simulator.Simulate pkg/simulator/core.go:67-119; see include/simon_gpu.h.
"""
from __future__ import annotations

import ctypes as C
import json
import os
from dataclasses import asdict
from typing import Dict, List

import numpy as np

from . import abi
from .objects import AppResource, ResourceTypes

_LIB = None


def lib():
    """libsimon_gpu.so (or the library named by SIMON_HOST_LIB: a development build of csrc/simon_host.cpp alone)."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = os.environ.get("SIMON_HOST_LIB")
    if path:
        _LIB = abi.bind(C.CDLL(path), partial=True)
    else:
        from .engine import lib as _engine_lib
        _LIB = _engine_lib()
    return _LIB


class NativeHostError(RuntimeError):
    def __init__(self, rc: int, msg: str):
        super().__init__(f"native host error {rc}: {msg}")
        self.rc = rc
        self.msg = msg


def request_json(cluster: ResourceTypes, apps: List[AppResource]) -> bytes:
    """The request the Go side builds with encoding/json: Go field names of ResourceTypes / AppResource (pkg/simulator/core.go:38-57)."""
    req = {"cluster": asdict(cluster) if not isinstance(cluster, dict) else cluster,
           "apps": [{"Name": a.Name, "Resource": asdict(a.Resource)} for a in apps]}
    return json.dumps(req, separators=(",", ":")).encode("utf-8")


def _arr(ptr, dtype, n):
    if n == 0 or not ptr:
        return np.zeros(0, dtype)
    return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(np.ctypeslib.as_ctypes_type(dtype))), shape=(n,)).copy()


class NativeCompiled:
    """Columns produced by simon_host_compile, copied into numpy arrays with the shapes compiler.Compiled uses."""

    def __init__(self, req: bytes):
        L = lib()
        h = C.c_void_p()
        rc = L.simon_host_compile(req, len(req), C.byref(h))
        if rc != 0:
            raise NativeHostError(rc, (L.simon_host_last_error() or b"").decode())
        try:
            snap, pods = abi.SimonSnapshot(), abi.SimonPodset()
            L.simon_host_plan_columns(h, C.byref(snap), C.byref(pods))
            self.info = json.loads(L.simon_host_plan_describe(h).decode())
            N, K, WL, WT, T = snap.n_nodes, snap.n_scalars, snap.n_label_words, snap.n_taint_words, snap.n_topos
            NC = snap.n_node_classes
            self.n_nodes = N
            self.snap_dims = {"n_nodes": N, "n_scalars": K, "n_label_words": WL, "n_taint_words": WT, "n_topos": T,
                              "n_node_classes": NC, "n_log": snap.n_log}
            K1 = max(K, 1)
            self.snap = {
                "topo_ndom": _arr(snap.topo_ndom, np.uint32, T), "alloc_mcpu": _arr(snap.alloc_mcpu, np.int64, N),
                "alloc_mem": _arr(snap.alloc_mem, np.int64, N), "alloc_eph": _arr(snap.alloc_eph, np.int64, N),
                "alloc_scalar": _arr(snap.alloc_scalar, np.int64, K1 * N).reshape(K1, N),
                "alloc_pods": _arr(snap.alloc_pods, np.int32, N), "node_flags": _arr(snap.node_flags, np.uint32, N),
                "label_bits": _arr(snap.label_bits, np.uint64, WL * N).reshape(WL, N),
                "taint_hard": _arr(snap.taint_hard, np.uint64, WT * N).reshape(WT, N),
                "taint_soft": _arr(snap.taint_soft, np.uint64, WT * N).reshape(WT, N),
                "topo_dom": _arr(snap.topo_dom, np.int32, T * N).reshape(T, N), "node_class": _arr(snap.node_class, np.int32, N),
                "gpu_count": _arr(snap.gpu_count, np.int32, N), "gpu_dev_mem": _arr(snap.gpu_dev_mem, np.int64, N),
                "gpu_total_mem": _arr(snap.gpu_total_mem, np.int64, N), "log_table": _arr(snap.log_table, np.float64, snap.n_log),
            }
            Cn, P = pods.n_classes, pods.n_pods
            self.pods_dims = {"n_classes": Cn, "n_pods": P, "n_counters": pods.n_counters, "n_static_sigs": pods.n_static_sigs,
                              "n_static_rows": pods.n_static_rows, "n_extra_rows": pods.n_extra_rows}
            class_off = _arr(pods.class_off, np.uint64, Cn + 1)
            n_blob = max(int(class_off[-1]) if Cn else 0, 1)
            n_extra = max(pods.n_extra_rows, 1)
            self.pods = {
                "class_off": class_off, "class_blob": _arr(pods.class_blob, np.int64, n_blob),
                "pod_class": _arr(pods.pod_class, np.int32, P), "pod_fixed_node": _arr(pods.pod_fixed_node, np.int32, P),
                "pod_pin_node": _arr(pods.pod_pin_node, np.int32, P),
                "counter_topo": _arr(pods.counter_topo, np.uint32, max(pods.n_counters, 1)),
                "simon_raw": _arr(pods.simon_raw, np.int64, pods.n_static_rows * NC).reshape(pods.n_static_rows, NC),
                "extra_score": _arr(pods.extra_score, np.int32, n_extra * max(N, 1)).reshape(n_extra, max(N, 1)),
            }
            self.node_names = self.info["nodeNames"]
            self.node_orig_index = self.info["nodeOrigIndex"]
            self.scalar_names = self.info["scalarNames"]
        finally:
            L.simon_host_plan_free(h)

    def pod_keys(self):
        """(workload kind, namespace, workload name, ordinal) per pod, in scheduling order (PodRec.key())."""
        t = self.info["templates"]
        out = []
        for ti, name, o in zip(self.info["podTemplate"], self.info["podName"], self.info["podOrdinal"]):
            tt = t[ti]
            out.append((tt["kind"], tt["namespace"], name if tt["kind"] == "Pod" else tt["workload"], o))
        return out


def compile_native(cluster: ResourceTypes, apps: List[AppResource]) -> NativeCompiled:
    return NativeCompiled(request_json(cluster, apps))


def simulate_native(cluster: ResourceTypes, apps: List[AppResource], device: int = 0, req: bytes = None) -> Dict:
    """simulator.Simulate through the native host side: objects (JSON) in -> placements and failure messages out."""
    L = lib()
    req = req if req is not None else request_json(cluster, apps)
    opts = abi.SimonCtxOpts(device, 0, 0, 0)
    out = C.c_void_p()
    n = C.c_uint64(0)
    import time
    t0 = time.perf_counter()
    rc = L.simon_host_simulate(req, len(req), C.byref(opts), C.byref(out), C.byref(n))
    simulate_native.last_call_s = time.perf_counter() - t0        # wall clock of the C-ABI call itself
    if rc != 0:
        raise NativeHostError(rc, (L.simon_host_last_error() or b"").decode())
    try:
        t0 = time.perf_counter()
        res = json.loads(C.string_at(out, n.value).decode())
        simulate_native.last_decode_s = time.perf_counter() - t0
        return res
    finally:
        L.simon_host_free(out)


def capacity_search_native(cluster: ResourceTypes, apps: List[AppResource], specs: List[dict], ks: List[int], device: int = 0, rank: int = 0,
                           world: int = 1, max_cpu: int = 100, max_mem: int = 100, dry_run: bool = False) -> Dict:
    """The add-node search of `simon apply` (pkg/apply/apply.go:203-259) through simon_host_capacity_search: this rank's shard of the
    (spec, k) scenarios; combine "bestKey" across ranks with one all-reduce(MIN) (capacity.torch_all_reduce_min)."""
    L = lib()
    req = json.loads(request_json(cluster, apps))
    req.update({"newNodes": list(specs), "ks": [int(k) for k in ks], "maxCPU": int(max_cpu), "maxMemory": int(max_mem),
                "rank": int(rank), "world": int(world), "dryRun": bool(dry_run)})
    raw = json.dumps(req, separators=(",", ":")).encode("utf-8")
    opts = abi.SimonCtxOpts(device, 0, 0, 0)
    out = C.c_void_p()
    n = C.c_uint64(0)
    rc = L.simon_host_capacity_search(raw, len(raw), C.byref(opts), C.byref(out), C.byref(n))
    if rc != 0:
        raise NativeHostError(rc, (L.simon_host_last_error() or b"").decode())
    try:
        return json.loads(C.string_at(out, n.value).decode())
    finally:
        L.simon_host_free(out)
