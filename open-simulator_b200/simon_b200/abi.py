"""The one Python copy of include/simon_gpu.h: its constants (header names without the SIMON_ prefix), ctypes mirrors of its structs,
the signature of every entry point, and the marshalling of a Compiled cluster.  tests/test_abi.py checks all of it against the
header."""
from __future__ import annotations

import ctypes as C

import numpy as np

ABI_VERSION = 3

# ---- limits ----
MAX_SCALARS = 8
MAX_GPU_DEV = 8
MAX_GPU_SLOTS = 64      # alibabacloud.com/gpu-count of a GPU-share pod
MAX_LABEL_WORDS = 16
MAX_TAINT_WORDS = 4
MAX_TOPOS = 8
MAX_VGS = 8             # Open-Local VGs per node
MAX_VOLS = 8            # Open-Local LVM PVCs per class
MAX_DEVS = 16           # Open-Local SSD + HDD devices per node
MAX_DEV_VOLS = 8        # Open-Local SSD + HDD PVCs per class
N_FAIL_CODES = 24
SOFT_SIZE0_WOFF = 6     # entry-table word offset of a later same-key ScheduleAnyway constraint: topology size 0

NODE_UNSCHEDULABLE = 1
NODE_HAS_LABELS = 2

# ---- pod class records: word indices (enum simon_class_word), flags, node-selection requirement ops ----
(SCW_REQ_MCPU, SCW_REQ_MEM, SCW_REQ_EPH, SCW_NZ_MCPU, SCW_NZ_MEM, SCW_SCORE_MCPU, SCW_SCORE_MEM, SCW_GPU_MEM,
 SCW_GPU_COUNT, SCW_FLAGS, SCW_NODE_NAME, SCW_STATIC_ROW, SCW_EXTRA_ROW, SCW_GUARD_NODE, SCW_STATIC_SIG, SCW_OFF_SCALARS, SCW_OFF_TOL, SCW_OFF_SEL,
 SCW_OFF_PREF, SCW_N_PREF, SCW_OFF_PORTS, SCW_N_PORTS, SCW_OFF_PTS_HARD, SCW_N_PTS_HARD, SCW_OFF_PTS_SOFT,
 SCW_N_PTS_SOFT, SCW_OFF_IPA_AFF, SCW_N_IPA_AFF, SCW_OFF_IPA_ANTI, SCW_N_IPA_ANTI, SCW_OFF_IPA_EXIST,
 SCW_N_IPA_EXIST, SCW_OFF_IPA_SCORE, SCW_N_IPA_SCORE, SCW_OFF_INC, SCW_N_INC, SCW_OFF_ENT, SCW_N_ENT, SCW_ANY_TABLE,
 SCW_ELIG_SIG, SCW_HDR_WORDS) = range(41)
CLS_HAS_REQUEST = 1
CLS_TOL_UNSCHED = 2
CLS_IPA_SELF_MATCH = 4
CLS_SIMON_NOREQ = 8
CLS_PINNED = 16            # node-selection programs refer to the pod's own pin node (REQ_NODE_IS payload -3): DaemonSet pods
REQ_ANY, REQ_NONE, REQ_NODE_IS, REQ_NODE_ISNOT = 1, 2, 3, 4

# ---- failure histogram columns (enum simon_fail_code); a filter verdict is a bitmask of (1 << code) ----
SFC_STATIC, SFC_PORTS, SFC_TOO_MANY_PODS, SFC_CPU, SFC_MEM, SFC_EPH, SFC_SCALAR0 = range(7)     # SFC_SCALAR0 + k: scalar resource k
SFC_PTS_MISSING, SFC_PTS_SKEW, SFC_IPA_AFF, SFC_IPA_ANTI, SFC_IPA_EXIST, SFC_GPU, SFC_LOCAL = range(14, 21)

# simon_ctx_opts.flags
OPT_RECORD_SCORES = 1
OPT_NO_PIN_FAST = 2
OPT_FORCE_LARGE = 4
OPT_NO_STATIC_CACHE = 8

# move codes other than filter verdicts, and the bias of the per-pod best-move key
MOVE_NOOP, MOVE_NOT_PLACED, MOVE_NOT_MOVABLE, MOVE_BAD_INDEX = 1 << 24, 1 << 25, 1 << 26, 1 << 27
MOVE_GAIN_BIAS = 1000
# simon_moves_set_scope: admit GPU-share classes / classes with DoNotSchedule spread constraints as move candidates
MOVES_SCOPE_GPU_SHARE, MOVES_SCOPE_HARD_SPREAD = 1, 2
# simon_moves_plan stop reasons
PLAN_STOP_NO_MOVE, PLAN_STOP_MAX_MOVES = 1, 2
# simon_probe_run stop reasons
PROBE_STOP_UNSCHEDULABLE, PROBE_STOP_MAX_REPLICAS = 1, 2
# explained decisions (simon_explain_set): largest top_k, words per listed node, the record node of a pod no call has covered
EXPLAIN_MAX_TOP = 16
EXPLAIN_WORDS = 10
EXPLAIN_NOT_RUN = -4
# simon_trace_event ops
TRACE_CREATE, TRACE_DELETE = 1, 2


class SimonSnapshot(C.Structure):
    _fields_ = [
        ("n_nodes", C.c_uint32), ("n_scalars", C.c_uint32), ("n_label_words", C.c_uint32),
        ("n_taint_words", C.c_uint32), ("n_topos", C.c_uint32), ("n_node_classes", C.c_uint32),
        ("n_log", C.c_uint32), ("reserved", C.c_uint32),
        ("topo_ndom", C.c_void_p), ("alloc_mcpu", C.c_void_p), ("alloc_mem", C.c_void_p), ("alloc_eph", C.c_void_p),
        ("alloc_scalar", C.c_void_p), ("alloc_pods", C.c_void_p), ("node_flags", C.c_void_p),
        ("label_bits", C.c_void_p), ("taint_hard", C.c_void_p), ("taint_soft", C.c_void_p),
        ("topo_dom", C.c_void_p), ("node_class", C.c_void_p), ("gpu_count", C.c_void_p),
        ("gpu_dev_mem", C.c_void_p), ("gpu_total_mem", C.c_void_p), ("log_table", C.c_void_p),
    ]


class SimonPodset(C.Structure):
    _fields_ = [
        ("n_classes", C.c_uint32), ("n_pods", C.c_uint32), ("n_counters", C.c_uint32),
        ("n_static_rows", C.c_uint32), ("n_extra_rows", C.c_uint32), ("n_static_sigs", C.c_uint32),
        ("class_off", C.c_void_p), ("class_blob", C.c_void_p), ("pod_class", C.c_void_p),
        ("pod_fixed_node", C.c_void_p), ("pod_pin_node", C.c_void_p), ("counter_topo", C.c_void_p), ("simon_raw", C.c_void_p),
        ("extra_score", C.c_void_p),
    ]


class SimonCtxOpts(C.Structure):
    _fields_ = [("device", C.c_int32), ("cluster_ctas", C.c_uint32), ("threads_per_cta", C.c_uint32),
                ("flags", C.c_uint32)]


class SimonLaunchInfo(C.Structure):
    _fields_ = [("kernel", C.c_char * 48), ("n_nodes", C.c_uint32), ("cluster_ctas", C.c_uint32), ("threads_per_cta", C.c_uint32),
                ("node_slots", C.c_uint32), ("n_scenarios", C.c_uint32), ("large", C.c_uint32), ("local", C.c_uint32),
                ("reserved", C.c_uint32), ("smem_bytes", C.c_uint64)]


class SimonScenario(C.Structure):
    _fields_ = [("n_nodes", C.c_uint32), ("reserved", C.c_uint32), ("nodes", C.c_void_p)]


class SimonScenarioResult(C.Structure):
    _fields_ = [("n_unscheduled", C.c_uint32), ("n_scheduled", C.c_uint32),
                ("req_mcpu", C.c_int64), ("alloc_mcpu", C.c_int64), ("req_mem", C.c_int64), ("alloc_mem", C.c_int64),
                ("elapsed_ms", C.c_float), ("reserved", C.c_uint32)]


class SimonDrainResult(C.Structure):
    _fields_ = [("n_evicted", C.c_uint32), ("n_placed", C.c_uint32), ("n_unscheduled", C.c_uint32), ("n_blocked", C.c_uint32),
                ("n_vanished", C.c_uint32), ("n_pdb_violated", C.c_uint32),
                ("req_mcpu", C.c_int64), ("alloc_mcpu", C.c_int64), ("req_mem", C.c_int64), ("alloc_mem", C.c_int64)]


class SimonJoinResult(C.Structure):
    _fields_ = [("n_join", C.c_uint32), ("n_placed", C.c_uint32), ("n_unscheduled", C.c_uint32), ("reserved", C.c_uint32)]


class SimonScenarioLocalResult(C.Structure):
    _fields_ = [("vg_requested", C.c_int64), ("vg_capacity", C.c_int64), ("reserved", C.c_uint64)]


class SimonProbe(C.Structure):
    _fields_ = [("pod", C.c_uint32), ("max_replicas", C.c_uint32)]


class SimonProbeResult(C.Structure):
    _fields_ = [("n_placed", C.c_uint32), ("stop_reason", C.c_uint32),
                ("req_mcpu", C.c_int64), ("alloc_mcpu", C.c_int64), ("req_mem", C.c_int64), ("alloc_mem", C.c_int64)]


class SimonTraceEvent(C.Structure):
    _fields_ = [("op", C.c_uint32), ("pod", C.c_uint32)]


class SimonTraceResult(C.Structure):
    _fields_ = [("n_scheduled", C.c_uint32), ("n_unscheduled", C.c_uint32), ("n_removed", C.c_uint32), ("n_running", C.c_uint32),
                ("req_mcpu", C.c_int64), ("alloc_mcpu", C.c_int64), ("req_mem", C.c_int64), ("alloc_mem", C.c_int64)]


class SimonTracePoint(C.Structure):
    _fields_ = [("event", C.c_uint32), ("n_running", C.c_uint32), ("n_failed", C.c_uint32), ("idle_devices", C.c_uint32),
                ("partial_devices", C.c_uint32), ("reserved", C.c_uint32),
                ("req_mcpu", C.c_int64), ("alloc_mcpu", C.c_int64), ("req_mem", C.c_int64), ("alloc_mem", C.c_int64),
                ("gpu_used", C.c_int64), ("gpu_total", C.c_int64)]


# simon_trace_point, as the structured array Engine.trace_run returns
TRACE_POINT_DTYPE = np.dtype(SimonTracePoint)


class SimonMovesResult(C.Structure):
    _fields_ = [("best_key", C.c_uint64), ("n_feasible", C.c_uint32), ("n_topk", C.c_uint32),
                ("kernel_ms", C.c_float), ("reserved", C.c_uint32)]


class SimonStorage(C.Structure):
    _fields_ = [("n_vgs", C.c_uint32), ("n_classes", C.c_uint32),
                ("node_n_vg", C.c_void_p), ("vg_capacity", C.c_void_p), ("vg_requested", C.c_void_p), ("vg_name", C.c_void_p),
                ("class_local", C.c_void_p), ("vol_off", C.c_void_p), ("vol_size", C.c_void_p), ("vol_vg", C.c_void_p)]


def marshal_storage(st):
    """storage.StorageTables -> (SimonStorage, arrays that must outlive the upload call)."""
    keep = [np.ascontiguousarray(a, dtype=t) for a, t in (
        (st.node_n_vg, np.int32), (st.vg_capacity, np.int64), (st.vg_requested, np.int64), (st.vg_name, np.int32),
        (st.class_local, np.uint8), (st.vol_off, np.uint32), (st.vol_size, np.int64), (st.vol_vg, np.int32))]
    keep = [a if a.size else np.zeros(1, a.dtype) for a in keep]
    s = SimonStorage(st.n_vgs, len(st.class_local), *[a.ctypes.data for a in keep])
    return s, keep


class SimonDevices(C.Structure):
    _fields_ = [("n_slots", C.c_uint32), ("n_classes", C.c_uint32),
                ("node_n_ssd", C.c_void_p), ("node_n_hdd", C.c_void_p), ("dev_capacity", C.c_void_p), ("dev_alloc", C.c_void_p),
                ("ssd_off", C.c_void_p), ("ssd_size", C.c_void_p), ("hdd_off", C.c_void_p), ("hdd_size", C.c_void_p)]


def marshal_devices(st):
    """storage.StorageTables compiled with devices=True -> (SimonDevices, arrays that must outlive the upload call)."""
    keep = [np.ascontiguousarray(a, dtype=t) for a, t in (
        (st.node_n_ssd, np.uint8), (st.node_n_hdd, np.uint8), (st.dev_capacity, np.int64), (st.dev_alloc, np.uint32),
        (st.ssd_off, np.uint32), (st.ssd_size, np.int64), (st.hdd_off, np.uint32), (st.hdd_size, np.int64))]
    keep = [a if a.size else np.zeros(1, a.dtype) for a in keep]
    s = SimonDevices(st.n_dev_slots, len(st.class_local), *[a.ctypes.data for a in keep])
    return s, keep


class SimonExplainRecord(C.Structure):
    _fields_ = [("node", C.c_int32), ("feasible", C.c_uint32), ("n_top", C.c_uint32), ("reserved", C.c_uint32),
                ("rejected", C.c_uint32 * N_FAIL_CODES)]


class SimonExplainNode(C.Structure):
    _fields_ = [("node", C.c_int32), ("reserved", C.c_uint32), ("words", C.c_int64 * EXPLAIN_WORDS)]


# the same two as the structured arrays Engine.explanations returns
EXPLAIN_RECORD_DTYPE = np.dtype(SimonExplainRecord)
EXPLAIN_NODE_DTYPE = np.dtype(SimonExplainNode)


# simon_plan_step, as the structured array Engine.moves_plan passes
PLAN_STEP_DTYPE = np.dtype([("move", np.uint32), ("pod", np.uint32), ("from", np.int32), ("to", np.int32), ("gain", np.int32),
                            ("gpu_slots", np.uint32)])


class SimonMovesPlanResult(C.Structure):
    _fields_ = [("n_steps", C.c_uint32), ("stop_reason", C.c_uint32), ("n_excluded", C.c_uint32), ("n_pdb_blocked", C.c_uint32),
                ("kernel_ms", C.c_float), ("reserved2", C.c_uint32)]


class SimonPdbs(C.Structure):
    _fields_ = [("n_pdbs", C.c_uint32), ("n_pods", C.c_uint32), ("pod_off", C.c_void_p), ("pod_pdb", C.c_void_p), ("desired", C.c_void_p)]


def marshal_pdbs(t):
    """disruption.PdbTables -> (SimonPdbs, arrays that must outlive the upload call)."""
    keep = [np.ascontiguousarray(a, dtype=d) for a, d in ((t.pod_off, np.uint32), (t.pod_pdb, np.uint32), (t.desired, np.int32))]
    keep = [a if a.size else np.zeros(1, a.dtype) for a in keep]
    s = SimonPdbs(len(t.desired), len(t.pod_off) - 1, *[a.ctypes.data for a in keep])
    return s, keep


_SNAP_DTYPES = {
    "topo_ndom": np.uint32, "alloc_mcpu": np.int64, "alloc_mem": np.int64, "alloc_eph": np.int64,
    "alloc_scalar": np.int64, "alloc_pods": np.int32, "node_flags": np.uint32, "label_bits": np.uint64,
    "taint_hard": np.uint64, "taint_soft": np.uint64, "topo_dom": np.int32, "node_class": np.int32,
    "gpu_count": np.int32, "gpu_dev_mem": np.int64, "gpu_total_mem": np.int64, "log_table": np.float64,
}
_PODS_DTYPES = {
    "class_off": np.uint64, "class_blob": np.int64, "pod_class": np.int32, "pod_fixed_node": np.int32,
    "counter_topo": np.uint32, "simon_raw": np.int64, "extra_score": np.int32, "pod_pin_node": np.int32,
}
_PODS_OPTIONAL = ("pod_pin_node",)       # NULL when the pod list has no pinned class (columns stored before ABI 3)


def ptr(a: np.ndarray) -> int:
    return a.ctypes.data


def marshal(compiled):
    """-> (SimonSnapshot, SimonPodset, keepalive list). Arrays are made contiguous with the ABI dtypes."""
    keep = []
    snap = SimonSnapshot()
    for k, v in compiled.snap_dims.items():
        setattr(snap, k, int(v))
    for k, dt in _SNAP_DTYPES.items():
        a = np.ascontiguousarray(compiled.snap[k], dtype=dt)
        keep.append(a)
        setattr(snap, k, ptr(a))
    pods = SimonPodset()
    for k, v in compiled.pods_dims.items():
        setattr(pods, k, int(v))
    for k, dt in _PODS_DTYPES.items():
        if k in _PODS_OPTIONAL and compiled.pods.get(k) is None:
            setattr(pods, k, None)
            continue
        a = np.ascontiguousarray(compiled.pods[k], dtype=dt)
        keep.append(a)
        setattr(pods, k, ptr(a))
    return snap, pods, keep


# ---- entry points: name -> (restype, argtypes), in the header's order; structs and arrays are passed as c_void_p ----
_P, _I, _U32, _I32, _PP = C.c_void_p, C.c_int, C.c_uint32, C.c_int32, C.POINTER(C.c_void_p)
_PF, _PU64 = C.POINTER(C.c_float), C.POINTER(C.c_uint64)
SIGNATURES = {
    "simon_gpu_version": (_I, []),
    "simon_ctx_create": (_I, [_P, _PP]),
    "simon_ctx_destroy": (None, [_P]),
    "simon_last_error": (C.c_char_p, [_P]),
    "simon_snapshot_upload": (_I, [_P, _P]),
    "simon_pods_upload": (_I, [_P, _P]),
    "simon_state_reset": (_I, [_P]),
    "simon_schedule": (_I, [_P, _U32, _U32, _P, _P, _P, _P, _U32, _P]),
    "simon_schedule_resume": (_I, [_P, _P, _U32, _P, _P, _P, _P, _U32, _P]),
    "simon_results_download": (_I, [_P, _U32, _U32, _P, _P]),
    "simon_replay": (_I, [_P, _U32, _PF]),
    "simon_stats": (_I, [_P, _P]),
    "simon_last_kernel_ms": (C.c_float, [_P]),
    "simon_launch_count": (C.c_uint64, [_P]),
    "simon_last_launch": (_I, [_P, _P]),
    "simon_state_download": (_I, [_P] * 7),
    "simon_scenarios_run": (_I, [_P, _P, _U32, _P, _P]),
    "simon_gpu_slots_download": (_I, [_P, _U32, _U32, _P]),
    "simon_state_download_ext": (_I, [_P, _P, _P]),
    "simon_debug_set_dump_pod": (_I, [_P, _U32]),
    "simon_debug_dump_read": (_I, [_P, _P, _P]),
    "simon_explain_set": (_I, [_P, _P, _U32, _U32]),
    "simon_explain_download": (_I, [_P, _U32, _U32, _P, _P]),
    "simon_moves_upload": (_I, [_P, _P, _U32, _U32]),
    "simon_moves_run": (_I, [_P, _U32, _P, _P, _P, _P, _P]),
    "simon_moves_replay": (_I, [_P, _U32, _PF]),
    "simon_moves_set_scope": (_I, [_P, _U32]),
    "simon_moves_gpu_slots_download": (_I, [_P, _U32, _U32, _P]),
    "simon_moves_plan": (_I, [_P, _U32, _I32, _P, _P]),
    "simon_moves_plan_download": (_I, [_P, _P, _P]),
    "simon_moves_plan_state_download": (_I, [_P] * 9),
    "simon_storage_upload": (_I, [_P, _P]),
    "simon_storage_state_download": (_I, [_P, _P]),
    "simon_devices_upload": (_I, [_P, _P]),
    "simon_devices_state_download": (_I, [_P, _P]),
    "simon_scenarios_run_local": (_I, [_P, _P, _U32, _P, _P, _P]),
    "simon_scenarios_storage_download": (_I, [_P, _U32, _P, _P]),
    "simon_drain_run": (_I, [_P, _P, _P, _U32, _P]),
    "simon_drain_run_local": (_I, [_P, _P, _P, _U32, _P, _P]),
    "simon_drain_download": (_I, [_P, _U32] + [_P] * 7),
    "simon_drain_pdb_download": (_I, [_P, _U32, _P, _P]),
    "simon_drain_times": (_I, [_P, _PF, _PF]),
    "simon_drain_budget": (_I, [_P, _PU64, _PU64]),
    "simon_wave_begin": (_I, [_P, _P]),
    "simon_wave_run": (_I, [_P, _P, _U32, _P]),
    "simon_wave_commit": (_I, [_P, _U32]),
    "simon_wave_download": (_I, [_P, _P, _P]),
    "simon_wave_times": (_I, [_P, _PF, _PF, _PF]),
    "simon_wave_begin_pool": (_I, [_P, _P, _P]),
    "simon_wave_run_join": (_I, [_P, _P, _P, _U32, _P, _P]),
    "simon_wave_join_download": (_I, [_P, _U32] + [_P] * 6),
    "simon_wave_commit_retire": (_I, [_P, _U32]),
    "simon_wave_presence": (_I, [_P, _P]),
    "simon_probe_run": (_I, [_P, _P, _P, _U32, _P, _P]),
    "simon_probe_download": (_I, [_P, _U32, _P, _P, _P, _P]),
    "simon_probe_times": (_I, [_P, _PF, _PF]),
    "simon_grow_run": (_I, [_P, _P, _U32, _P, _U32, _P, _P]),
    "simon_grow_download": (_I, [_P, _U32] + [_P] * 5),
    "simon_grow_times": (_I, [_P, _PF, _PF]),
    "simon_trace_run": (_I, [_P, _P, _U32, _P, _U32, _P, _U32, _P, _U32, _P]),
    "simon_trace_download": (_I, [_P, _U32] + [_P] * 5),
    "simon_trace_samples_download": (_I, [_P, _U32, _P]),
    "simon_trace_times": (_I, [_P, _PF, _PF, C.POINTER(C.c_uint32), _PU64]),
    "simon_pdbs_upload": (_I, [_P, _P]),
    "simon_pdbs_allowed": (_I, [_P, _P]),
    "simon_host_go118_sort": (_I, [_P, _U32, _P]),
    "simon_host_last_error": (C.c_char_p, []),
    "simon_host_compile": (_I, [C.c_char_p, C.c_uint64, _PP]),
    "simon_host_plan_free": (None, [_P]),
    "simon_host_plan_columns": (_I, [_P, _P, _P]),
    "simon_host_plan_describe": (C.c_char_p, [_P]),
    "simon_host_simulate": (_I, [C.c_char_p, C.c_uint64, _P, _PP, _PU64]),
    "simon_host_free": (None, [_P]),
    "simon_host_capacity_search": (_I, [C.c_char_p, C.c_uint64, _P, _PP, _PU64]),
    "simon_host_plan_fit_error": (_I, [_P, _U32, _P, _PP]),
    "simon_host_quantity_probe": (_I, [C.c_char_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_double)]),
}


def bind(L: C.CDLL, partial: bool = False) -> C.CDLL:
    """Give each entry point of SIGNATURES its restype and argtypes on the loaded library L.  partial: skip the ones L does not export
    (an experiment library, or a build of the host side alone); the shipped library exports every one."""
    for name, (restype, argtypes) in SIGNATURES.items():
        f = getattr(L, name, None) if partial else getattr(L, name)
        if f is not None:
            f.restype, f.argtypes = restype, argtypes
    return L
