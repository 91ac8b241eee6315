"""ctypes binding of libsimon_gpu.so — the C-ABI engine (include/simon_gpu.h).

There is NO CPU fallback: if the shared library is missing or no CUDA device can be opened, constructing an
Engine raises EngineUnavailable.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import List, Optional

import numpy as np

from . import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("SIMON_GPU_LIB") or os.path.join(_HERE, "libsimon_gpu.so")    # the override is for kernel experiments
_LIB = None

EXPORTS = list(abi.SIGNATURES)       # every entry point of include/simon_gpu.h


class EngineUnavailable(RuntimeError):
    pass


def lib():
    global _LIB
    if _LIB is not None:
        return _LIB
    if not os.path.exists(LIB_PATH):
        raise EngineUnavailable(f"{LIB_PATH} not built: run __graft_entry__.build() (nvcc, sm_90a)")
    # an experiment library may lack the newer entry points; the shipped one may not
    _LIB = abi.bind(C.CDLL(LIB_PATH), partial=bool(os.environ.get("SIMON_GPU_LIB")))
    return _LIB


class Engine:
    """One device context holding one compiled cluster (snapshot + ordered pod list)."""

    def __init__(self, compiled, device: int = 0, record_scores: bool = False, cluster_ctas: int = 0,
                 threads_per_cta: int = 0, pin_fast: bool = True, force_large: bool = False, static_cache: bool = True):
        L = lib()
        self.c = compiled
        self.h = C.c_void_p()
        # pin_fast=False: DaemonSet pods take the general one-decision-at-a-time path (SIMON_OPT_NO_PIN_FAST; same results)
        # force_large=True: the large-cluster kernel variant at any size (SIMON_OPT_FORCE_LARGE; same results)
        # static_cache=False: no static verdict cache, every verdict evaluated where it is needed, as past the cache's 2 GiB cap
        # (SIMON_OPT_NO_STATIC_CACHE; same results)
        opts = abi.SimonCtxOpts(device, cluster_ctas, threads_per_cta,
                                (abi.OPT_RECORD_SCORES if record_scores else 0) | (0 if pin_fast else abi.OPT_NO_PIN_FAST) |
                                (abi.OPT_FORCE_LARGE if force_large else 0) | (0 if static_cache else abi.OPT_NO_STATIC_CACHE))
        rc = L.simon_ctx_create(C.byref(opts), C.byref(self.h))
        if rc != 0 or not self.h:
            raise EngineUnavailable(f"simon_ctx_create failed (rc={rc}): no usable CUDA device {device}; "
                                    "the engine has no CPU path")
        self.record_scores = record_scores
        self.snap, self.pods, self._keep = abi.marshal(compiled)
        self._check(L.simon_snapshot_upload(self.h, C.byref(self.snap)))
        self._check(L.simon_pods_upload(self.h, C.byref(self.pods)))
        if getattr(compiled, "storage", None) is not None:      # Open-Local LVM volumes (compile_cluster(open_local=True))
            # the marshalled structs stay usable for a later re-upload: their arrays are kept with them
            self.storage, self._storage_keep = abi.marshal_storage(compiled.storage)
            self._check(L.simon_storage_upload(self.h, C.byref(self.storage)))
            if compiled.storage.devices:                        # SSD / HDD devices (compile_cluster(local_devices=True))
                self.devices, self._devices_keep = abi.marshal_devices(compiled.storage)
                self._check(L.simon_devices_upload(self.h, C.byref(self.devices)))

    def _check(self, rc: int):
        if rc != 0:
            msg = lib().simon_last_error(self.h)
            raise RuntimeError(f"simon engine error {rc}: {msg.decode() if msg else ''}")

    def close(self):
        if getattr(self, "h", None):
            lib().simon_ctx_destroy(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset(self):
        self._check(lib().simon_state_reset(self.h))

    def explain_set(self, pods, top_k: int = 3):
        """simon_explain_set: later schedule / schedule_resume calls also explain these pods (ascending pod indices; [] clears the
        set), listing the best top_k feasible nodes of each; explanations() reads the records."""
        a = np.ascontiguousarray(pods, dtype=np.uint32)
        self._check(lib().simon_explain_set(self.h, a.ctypes.data if len(a) else None, len(a), int(top_k)))
        self._explain = (len(a), int(top_k))

    def explanations(self):
        """The explained pods' records of the set, in its order: (records [n] of abi.EXPLAIN_RECORD_DTYPE, nodes [n][top_k] of
        abi.EXPLAIN_NODE_DTYPE); only the first records["n_top"] nodes of a record are filled."""
        n, k = getattr(self, "_explain", (0, 0))
        rec = np.zeros(max(n, 1), abi.EXPLAIN_RECORD_DTYPE)
        nodes = np.zeros((max(n, 1), max(k, 1)), abi.EXPLAIN_NODE_DTYPE)
        if n:
            self._check(lib().simon_explain_download(self.h, 0, n, rec.ctypes.data, nodes.ctypes.data))
        return rec[:n], nodes[:n, :k]

    def schedule(self, first: int = 0, count: Optional[int] = None, max_fail: Optional[int] = None, download: bool = True,
                 explain=None, top_k: int = 3):
        """Place pods [first, first+count). Returns (out_node, out_score, fail_counts, fail_pod).  explain: set the explained pods
        first (explain_set(explain, top_k)); None keeps the set as it is."""
        if explain is not None:
            self.explain_set(explain, top_k)
        P = self.c.pods_dims["n_pods"]
        count = P - first if count is None else count
        max_fail = count if max_fail is None else max_fail
        n_fail = C.c_uint32(0)
        if not download:
            self._check(lib().simon_schedule(self.h, first, count, None, None, None, None, 0, C.byref(n_fail)))
            return None, None, None, None
        out_node = np.full(count, -9, np.int32)
        out_score = np.zeros(count, np.int64)
        fail_counts = np.zeros((max(max_fail, 1), abi.N_FAIL_CODES), np.uint32)
        fail_pod = np.zeros(max(max_fail, 1), np.uint32)
        self._check(lib().simon_schedule(self.h, first, count, out_node.ctypes.data,
                                         out_score.ctypes.data if self.record_scores else None,
                                         fail_counts.ctypes.data, fail_pod.ctypes.data, max_fail, C.byref(n_fail)))
        nf = min(n_fail.value, max_fail)
        return out_node, out_score, fail_counts[:nf], fail_pod[:nf]

    def schedule_resume(self, prefix_node, max_fail: Optional[int] = None, explain=None, top_k: int = 3):
        """simon_schedule_resume: rebuild the state pods [0, len(prefix_node)) leave at the nodes an earlier call gave them (its
        out_node), then place the rest.  Returns (out_node, out_score, fail_counts, fail_pod) over ALL pods; the scores of the prefix
        pods are 0 (not recomputed) and the failures are those of the placed rest only.  explain: as schedule's."""
        if explain is not None:
            self.explain_set(explain, top_k)
        P = self.c.pods_dims["n_pods"]
        prefix = np.ascontiguousarray(prefix_node, dtype=np.int32)
        n_prefix = len(prefix)
        max_fail = max(P - n_prefix, 0) if max_fail is None else max_fail
        n_fail = C.c_uint32(0)
        out_node = np.full(max(P, 1), -9, np.int32)
        out_score = np.zeros(max(P, 1), np.int64)
        fail_counts = np.zeros((max(max_fail, 1), abi.N_FAIL_CODES), np.uint32)
        fail_pod = np.zeros(max(max_fail, 1), np.uint32)
        self._check(lib().simon_schedule_resume(self.h, prefix.ctypes.data if n_prefix else None, n_prefix, out_node.ctypes.data,
                                                out_score.ctypes.data if self.record_scores else None,
                                                fail_counts.ctypes.data, fail_pod.ctypes.data, max_fail, C.byref(n_fail)))
        nf = min(n_fail.value, max_fail)
        return out_node[:P], out_score[:P], fail_counts[:nf], fail_pod[:nf]

    def results(self, first: int = 0, count: Optional[int] = None):
        P = self.c.pods_dims["n_pods"]
        count = P - first if count is None else count
        out_node = np.full(count, -9, np.int32)
        self._check(lib().simon_results_download(self.h, first, count, out_node.ctypes.data, None))
        return out_node

    def replay(self, steps: int = 1) -> float:
        """steps x (reset + place every pod), device-timed; returns total ms. Results stay on the device."""
        ms = C.c_float(0)
        self._check(lib().simon_replay(self.h, steps, C.byref(ms)))
        return float(ms.value)

    def stats(self):
        a = np.zeros(32, np.uint64)
        self._check(lib().simon_stats(self.h, a.ctypes.data))
        return dict(decisions=int(a[0]), class_switches=int(a[1]), summary_rebuilds=int(a[2]), redone=int(a[3]), static_evals=int(a[4]), single_flip_fast=int(a[6]),
                    merged_decisions=int(a[7] & 0xffffffff), merged_redone=int(a[7] >> 32),
                    cycles=dict(zip(['loop', 'fixed', 'class_change_tail', 'r1', 'p1', 'reduce_steady', 'reduce_summary', 'p3', 'argmax', 'commit',
                                     'cc_pre', 'cc_sync', 'cc_blob', 'cc_entry', 'cc_static', 'pts_pass_steady'],
                                    [int(x) for x in a[8:24]])),
                    reductions=dict(zip(['allreduce_bar', 'allreduce_exchange', 'allreduce_n', 'argmax_bar', 'argmax_exchange', 'argmax_n'],
                                        [int(x) for x in a[24:30]])),
                    owner_commit=dict(cycles=int(a[30]), n=int(a[31])), spec_own=dict(cycles=int(a[27]), n=int(a[5])))

    def last_kernel_ms(self) -> float:
        return float(lib().simon_last_kernel_ms(self.h))

    def launch_count(self) -> int:
        return int(lib().simon_launch_count(self.h))

    def last_launch(self) -> dict:
        """The placement kernel the last schedule / schedule_resume / replay / run_scenarios call launched and its geometry;
        kernel "" when none ran."""
        li = abi.SimonLaunchInfo()
        self._check(lib().simon_last_launch(self.h, C.byref(li)))
        return dict(kernel=li.kernel.decode(), n_nodes=li.n_nodes, cluster_ctas=li.cluster_ctas, threads_per_cta=li.threads_per_cta,
                    node_slots=li.node_slots, n_scenarios=li.n_scenarios, large=bool(li.large), local=bool(li.local),
                    smem_bytes=int(li.smem_bytes))

    def _state(self, download, cols: slice = slice(0, 8)):
        """The node state through `download` (simon_state_download, simon_state_download_ext or simon_moves_plan_state_download),
        called with the host arrays of columns `cols` of (req_mcpu, req_mem, req_eph, nz_mcpu, nz_mem, num_pods, req_scalar [K][N],
        gpu_used [8][N]): -> (state() dict, state_ext() dict)."""
        N, K = self.c.n_nodes, int(self.c.snap_dims["n_scalars"])
        N1 = max(N, 1)
        arrs = [np.zeros(N1, np.int64) for _ in range(5)] + [np.zeros(N1, np.int32), np.zeros((max(K, 1), N1), np.int64),
                                                             np.zeros((8, N1), np.int64)]
        self._check(download(self.h, *[a.ctypes.data for a in arrs[cols]]))
        return (dict(zip(["req_mcpu", "req_mem", "req_eph", "nz_mcpu", "nz_mem", "num_pods"], [a[:N] for a in arrs[:6]])),
                dict(req_scalar=arrs[6][:K, :N], gpu_used=arrs[7][:, :N]))

    def state(self):
        return self._state(lib().simon_state_download, slice(0, 6))[0]

    def storage_state(self) -> np.ndarray:
        """Open-Local VG requested after scheduling, [V][N]."""
        V, N = self.c.storage.n_vgs, self.c.n_nodes
        a = np.zeros(max(V * N, 1), np.int64)
        self._check(lib().simon_storage_state_download(self.h, a.ctypes.data))
        return a[:V * N].reshape(V, N)

    def device_state(self) -> np.ndarray:
        """Open-Local allocated device slots after scheduling, [N] masks (bit s: slot s of storage.StorageTables)."""
        a = np.zeros(max(self.c.n_nodes, 1), np.uint32)
        self._check(lib().simon_devices_state_download(self.h, a.ctypes.data))
        return a[:self.c.n_nodes]

    def gpu_slot_words(self, first: int = 0, count: Optional[int] = None) -> np.ndarray:
        """GPU-share Reserve results as simon_gpu_slots_download packs them: per pod 4 bits per device = its slots there."""
        P = self.c.pods_dims["n_pods"]
        count = P - first if count is None else count
        a = np.zeros(max(count, 1), np.uint32)
        self._check(lib().simon_gpu_slots_download(self.h, first, count, a.ctypes.data))
        return a[:count]

    def gpu_slots(self, first: int = 0, count: Optional[int] = None):
        """GPU-share Reserve results: per pod a list of device ids (one per GPU slot, ascending), [] if none."""
        out = []
        for v in self.gpu_slot_words(first, count):
            v = int(v)
            out.append([d for d in range(8) for _ in range((v >> (4 * d)) & 15)])
        return out

    def state_ext(self):
        return self._state(lib().simon_state_download_ext, slice(6, 8))[1]

    def dump_pod(self, pod: int, placed: Optional[np.ndarray] = None):
        """From the EMPTY state, schedule up to and including `pod`; return (out_node of the range, per-node totals,
        per-node filter verdicts of that pod).  Leaves the context in that partial state.  placed: the out_node of an earlier run
        of this pod list - the pods before `pod` are then not placed again but rebuilt at those nodes (simon_schedule_resume), and
        the rest of the list is placed too."""
        if placed is not None:
            self._check(lib().simon_debug_set_dump_pod(self.h, pod))
            out = self.schedule_resume(np.asarray(placed)[:pod], max_fail=0)[0][:pod + 1]
        else:
            self.reset()
            self._check(lib().simon_debug_set_dump_pod(self.h, pod))
            out = self.schedule(0, pod + 1)[0]
        self._check(lib().simon_debug_set_dump_pod(self.h, 0xffffffff))
        N = self.c.n_nodes
        tot = np.zeros(max(N, 1), np.int64)
        code = np.zeros(max(N, 1), np.int32)
        self._check(lib().simon_debug_dump_read(self.h, tot.ctypes.data, code.ctypes.data))
        return out, tot[:N], code[:N]

    # ---- candidate-move scoring (config 5) ----
    def moves_upload(self, moves: np.ndarray, move_base: int = 0):
        """moves: uint32 array [n, 2] of (pod index, target node)."""
        a = np.ascontiguousarray(moves, dtype=np.uint32).reshape(-1, 2)
        self._moves_keep = a
        self._check(lib().simon_moves_upload(self.h, a.ctypes.data, len(a), move_base))
        return len(a)

    def moves_set_scope(self, scope: int):
        """Admit GPU-share classes (abi.MOVES_SCOPE_GPU_SHARE) and / or classes with DoNotSchedule spread constraints
        (abi.MOVES_SCOPE_HARD_SPREAD) as move candidates in later runs; 0 = the default scoring."""
        self._check(lib().simon_moves_set_scope(self.h, scope))

    def moves_run(self, k: int = 0, want_arrays: bool = True, want_per_pod: bool = False, want_gpu_slots: bool = False):
        """-> dict(best_key, n_feasible, kernel_ms, gain, code, best_per_pod, topk=[(move, gain)...]); with want_gpu_slots (the
        scope must include GPU share) also gpu_slots: per move the target's device slots, 4 bits per device, 0 if none."""
        n = len(self._moves_keep)
        gain = np.zeros(max(n, 1), np.int32) if want_arrays else None
        code = np.zeros(max(n, 1), np.uint32) if want_arrays else None
        bpp = np.zeros(max(self.c.pods_dims["n_pods"], 1), np.uint64) if want_per_pod else None
        topk = np.zeros((max(k, 1), 2), np.int32)
        res = abi.SimonMovesResult()
        self._check(lib().simon_moves_run(self.h, k, gain.ctypes.data if want_arrays else None, code.ctypes.data if want_arrays else None,
                                          bpp.ctypes.data if want_per_pod else None, topk.ctypes.data if k else None, C.byref(res)))
        out = dict(best_key=int(res.best_key), n_feasible=int(res.n_feasible), kernel_ms=float(res.kernel_ms),
                   gain=None if gain is None else gain[:n], code=None if code is None else code[:n],
                   best_per_pod=bpp, topk=[(int(topk[q, 0]) & 0xffffffff, int(topk[q, 1])) for q in range(res.n_topk)])
        if want_gpu_slots:
            slots = np.zeros(max(n, 1), np.uint32)
            self._check(lib().simon_moves_gpu_slots_download(self.h, 0, n, slots.ctypes.data))
            out["gpu_slots"] = slots[:n]
        return out

    def moves_replay(self, steps: int = 1) -> float:
        ms = C.c_float(0)
        self._check(lib().simon_moves_replay(self.h, steps, C.byref(ms)))
        return float(ms.value)

    def moves_plan(self, max_moves: int, min_gain: int = 1):
        """A migration plan over the uploaded move list (move_base 0) on the live state, under the current move scope
        (simon_moves_plan): -> dict(steps: structured array of abi.PLAN_STEP_DTYPE, stop_reason, excluded, kernel_ms).
        The live state is not changed."""
        steps = np.zeros(max(max_moves, 1), abi.PLAN_STEP_DTYPE)
        res = abi.SimonMovesPlanResult()
        self._check(lib().simon_moves_plan(self.h, max_moves, min_gain, steps.ctypes.data, C.byref(res)))
        return dict(steps=steps[:res.n_steps].copy(), stop_reason=int(res.stop_reason), excluded=int(res.n_excluded),
                    pdb_blocked=int(res.n_pdb_blocked), kernel_ms=float(res.kernel_ms))

    def moves_plan_download(self):
        """After moves_plan: (placement [P] int32, GPU slot words [P] uint32) of the plan's end state."""
        P = self.c.pods_dims["n_pods"]
        pl = np.zeros(max(P, 1), np.int32)
        sl = np.zeros(max(P, 1), np.uint32)
        self._check(lib().simon_moves_plan_download(self.h, pl.ctypes.data, sl.ctypes.data))
        return pl[:P], sl[:P]

    def moves_plan_state(self):
        """After moves_plan: the plan's end state as (state(), state_ext()) dicts."""
        return self._state(lib().simon_moves_plan_state_download)

    def run_scenarios(self, scenarios: List[np.ndarray], want_nodes: bool = False):
        """scenarios: list of uint32 arrays (active node indices in scenario order)."""
        return self._run_scenarios(scenarios, want_nodes, False)

    def run_scenarios_local(self, scenarios: List[np.ndarray], want_nodes: bool = False):
        """run_scenarios for a cluster compiled with open_local=True: every scenario places its pods on its own copy of the
        uploaded VG and device state; each result also carries vg_requested / vg_capacity, the sums over the scenario's
        annotated nodes after the run (satisfyResourceSetting's MaxVG input)."""
        return self._run_scenarios(scenarios, want_nodes, True)

    @staticmethod
    def _scenario_array(node_lists):
        """(SimonScenario array over node_lists, the uint32 arrays it points into: keep them alive for the call)."""
        arr = (abi.SimonScenario * len(node_lists))()
        keep = [np.ascontiguousarray(nodes, dtype=np.uint32) for nodes in node_lists]
        for s, a in zip(arr, keep):
            s.n_nodes = len(a)
            s.nodes = a.ctypes.data if len(a) else None
        return arr, keep

    def _run_scenarios(self, scenarios, want_nodes, local):
        n = len(scenarios)
        arr, keep = self._scenario_array(scenarios)
        res = (abi.SimonScenarioResult * n)()
        P = self.c.pods_dims["n_pods"]
        out_node = np.full((n, P), -9, np.int32) if want_nodes else None
        if local:
            loc = (abi.SimonScenarioLocalResult * n)()
            self._check(lib().simon_scenarios_run_local(self.h, arr, n, res, loc, out_node.ctypes.data if want_nodes else None))
        else:
            self._check(lib().simon_scenarios_run(self.h, arr, n, res, out_node.ctypes.data if want_nodes else None))
        out = [dict(n_unscheduled=r.n_unscheduled, n_scheduled=r.n_scheduled, req_mcpu=r.req_mcpu, alloc_mcpu=r.alloc_mcpu,
                    req_mem=r.req_mem, alloc_mem=r.alloc_mem, elapsed_ms=r.elapsed_ms) for r in res]
        if local:
            for o, r in zip(out, loc):
                o["vg_requested"], o["vg_capacity"] = int(r.vg_requested), int(r.vg_capacity)
        return out, out_node

    def scenario_storage_state(self, i: int):
        """Scenario i of the last run_scenarios_local batch, or drain i of the last batch (chunk) of the last
        drain_run(..., local=True): (VG requested [V][N], allocated device slot masks [N] or None without devices), node-indexed like
        the snapshot.  A drain's removed nodes keep their live values."""
        V, N = self.c.storage.n_vgs, self.c.n_nodes
        vg = np.zeros(max(V * N, 1), np.int64)
        dev = np.zeros(max(N, 1), np.uint32) if self.c.storage.devices else None
        self._check(lib().simon_scenarios_storage_download(self.h, i, vg.ctypes.data, None if dev is None else dev.ctypes.data))
        return vg[:V * N].reshape(V, N), None if dev is None else dev[:N]

    # ---- PodDisruptionBudgets (simon_pdbs_upload) ----
    def pdbs_upload(self, tables):
        """Upload disruption.PdbTables of this pod list (None or no PDB: clear the table).  Later drains, move runs and plans honour
        them; a new pod upload drops them."""
        if tables is None:
            self.pdbs, self._pdbs_keep = abi.SimonPdbs(0, self.c.pods_dims["n_pods"], None, None, None), []
        else:
            self.pdbs, self._pdbs_keep = abi.marshal_pdbs(tables)
        self.n_pdbs = int(self.pdbs.n_pdbs)
        self._check(lib().simon_pdbs_upload(self.h, C.byref(self.pdbs)))

    def pdbs_allowed(self) -> np.ndarray:
        """Per uploaded PDB: the disruptions it allows on the live placement, max(0, placed members - desired)."""
        n = getattr(self, "n_pdbs", 0)
        a = np.zeros(max(n, 1), np.int32)
        self._check(lib().simon_pdbs_allowed(self.h, a.ctypes.data))
        return a[:n]

    # ---- node drains (simon_drain_run) ----
    # share of the memory simon_drain_budget reports that one batch's pooled state may take: the rest is the margin for what the
    # per-scenario bytes do not count (per-evicted-pod outputs, failure records, the large-cluster variant's node arrays)
    DRAIN_MEM_FRACTION = 0.5

    def drain_budget(self):
        """(device bytes of one drain scenario's pooled state, bytes a batch may use now)."""
        per, free = C.c_uint64(0), C.c_uint64(0)
        self._check(lib().simon_drain_budget(self.h, C.byref(per), C.byref(free)))
        return int(per.value), int(free.value)

    def _chunked(self, n: int, chunk: Optional[int], times, run, extra: int = 0):
        """Entries [0, n) in batches of `chunk` entries, or of as many as fit: drain_budget()'s per-scenario bytes plus `extra` per
        entry, in DRAIN_MEM_FRACTION of the free bytes.  run(b, m) runs entries [b, b + m) as one batch and returns their dicts; after
        it, times(h, &setup_ms, &place_ms) reads the batch's device times.  -> (the dicts of every entry, dict(chunks,
        scenario_bytes, chunk, setup_ms / place_ms summed over the batches, launches: last_launch() of each batch))."""
        per, free = self.drain_budget()
        per += extra
        if chunk is None:
            chunk = max(1, int(free * self.DRAIN_MEM_FRACTION) // max(per, 1))
        out = []
        info = dict(chunks=0, scenario_bytes=per, chunk=chunk, setup_ms=0.0, place_ms=0.0, launches=[])
        for b in range(0, n, chunk):
            out.extend(run(b, min(chunk, n - b)))
            su, pm = C.c_float(0), C.c_float(0)
            self._check(times(self.h, C.byref(su), C.byref(pm)))
            info["chunks"] += 1
            info["setup_ms"] += float(su.value)
            info["place_ms"] += float(pm.value)
            info["launches"].append(self.last_launch())
        return out, info

    def _download(self, fn, i: int, *specs):
        """fn(h, i, *arrays) into zero arrays, one per spec (rows, dtype) or (rows, dtype, columns), each at least one row long: -> the
        arrays cut to their rows."""
        arrs = [np.zeros((max(s[0], 1),) + tuple(s[2:]), s[1]) for s in specs]
        self._check(fn(self.h, i, *[a.ctypes.data for a in arrs]))
        return [a[:s[0]] for a, s in zip(arrs, specs)]

    def drain_run(self, placed, remain_lists: List[np.ndarray], detail: bool = True, chunk: Optional[int] = None, local: bool = False):
        """Drains on the live state `placed` (out_node of a full placement of the pod list): each entry of remain_lists lists the
        nodes that remain, in their nodeTree.list() order.  The list runs in batches (chunks) sized so that one batch's pooled state
        fits the device: chunk scenarios of simon_drain_budget's per-scenario bytes in DRAIN_MEM_FRACTION of what it reports free
        (chunk: an explicit batch size).  Returns one dict per drain: n_evicted, n_placed, n_unscheduled, n_blocked, n_vanished and
        the sums req_mcpu / alloc_mcpu / req_mem / alloc_mem over the remaining nodes, and n_pdb_violated (with a PDB table); with
        detail also evicted (pod indices in pod order), node (per evicted pod, -1 unschedulable), gpu_slots, score, blocked,
        fail_counts [n_unscheduled][24], fail_pod, and pdb_violated / pdb_evicted (the violated PDBs ascending, their evicted
        members).  self.last_drain: chunks, scenario_bytes, setup_ms / place_ms (device time summed over the batches).
        local=True (a cluster compiled with open_local=True): simon_drain_run_local, so pods with Open-Local volumes are evicted and
        provisioned again on the remaining nodes instead of blocking the drain, and every result also carries vg_requested /
        vg_capacity, the VG sums over the remaining annotated nodes after the placement (satisfyResourceSetting's MaxVG input);
        scenario_storage_state(i) then describes drain i of the last chunk."""
        L = lib()
        pl = np.ascontiguousarray(placed, dtype=np.int32)

        def run(b, m):
            arr, keep = self._scenario_array(remain_lists[b:b + m])
            res = (abi.SimonDrainResult * m)()
            if local:
                loc = (abi.SimonScenarioLocalResult * m)()
                self._check(L.simon_drain_run_local(self.h, pl.ctypes.data, arr, m, res, loc))
            else:
                self._check(L.simon_drain_run(self.h, pl.ctypes.data, arr, m, res))
            return self._drain_results(res, loc if local else None, detail)
        out, self.last_drain = self._chunked(len(remain_lists), chunk, L.simon_drain_times, run)
        return out

    def _drain_results(self, res, loc, detail: bool) -> List[dict]:
        """The dicts drain_run returns, of the last drain or wave batch's results `res` (and Open-Local sums `loc`, or None)."""
        L = lib()
        out = []
        for i, r in enumerate(res):
            d = dict(n_evicted=r.n_evicted, n_placed=r.n_placed, n_unscheduled=r.n_unscheduled, n_blocked=r.n_blocked,
                     n_vanished=r.n_vanished, n_pdb_violated=r.n_pdb_violated, req_mcpu=r.req_mcpu, alloc_mcpu=r.alloc_mcpu,
                     req_mem=r.req_mem, alloc_mem=r.alloc_mem)
            if loc is not None:
                d["vg_requested"], d["vg_capacity"] = int(loc[i].vg_requested), int(loc[i].vg_capacity)
            if detail:
                ne, nb, nf, nv = r.n_evicted, r.n_blocked, r.n_unscheduled, r.n_pdb_violated
                d.update(zip(("evicted", "node", "gpu_slots", "score", "blocked", "fail_counts", "fail_pod"),
                             self._download(L.simon_drain_download, i, (ne, np.uint32), (ne, np.int32), (ne, np.uint32), (ne, np.int64),
                                            (nb, np.uint32), (nf, np.uint32, abi.N_FAIL_CODES), (nf, np.uint32))))
                d.update(zip(("pdb_violated", "pdb_evicted"), self._download(L.simon_drain_pdb_download, i, (nv, np.uint32), (nv, np.uint32))))
            out.append(d)
        return out

    # ---- rolling maintenance waves (simon_wave_*) ----
    def wave_begin(self, placed, present=None):
        """simon_wave_begin: the wave base is the live state `placed` (out_node of a full placement of the pod list) leaves.
        present (bool per node): simon_wave_begin_pool, the nodes that are in the cluster; the others are absent until a wave joins
        them."""
        pl = np.ascontiguousarray(placed, dtype=np.int32)
        if present is None:
            self._check(lib().simon_wave_begin(self.h, pl.ctypes.data))
        else:
            pr = np.ascontiguousarray(np.asarray(present, dtype=bool).astype(np.uint8))
            self._check(lib().simon_wave_begin_pool(self.h, pl.ctypes.data, pr.ctypes.data if pr.size else None))
        self._wave = None
        self.last_wave = dict(batches=0, setup_ms=0.0, place_ms=0.0, commits=0, commit_ms=0.0, launches=[])

    def wave_run(self, remain_lists: List[np.ndarray], joins: Optional[List[np.ndarray]] = None, detail: bool = True,
                 chunk: Optional[int] = None) -> List[dict]:
        """Drains from the wave base, one dict per entry of remain_lists as drain_run returns them; in batches sized as drain_run
        sizes them (chunk: an explicit batch size).  self.last_wave sums the device times of every batch and commit since wave_begin.
        joins (simon_wave_run_join): entry i also joins the absent nodes joins[i]; each dict then also carries n_join,
        n_join_placed, n_join_unscheduled and, with detail, join_pods, join_node, join_gpu_slots, join_score, join_fail_counts and
        join_fail_pod."""
        L = lib()

        def run(b, m):
            arr, keep = self._scenario_array(remain_lists[b:b + m])
            res = (abi.SimonDrainResult * m)()
            if joins is None:
                self._check(L.simon_wave_run(self.h, arr, m, res))
            else:
                jarr, jkeep = self._scenario_array(joins[b:b + m])
                jres = (abi.SimonJoinResult * m)()
                self._check(L.simon_wave_run_join(self.h, arr, jarr, m, res, jres))
            self._wave = (list(remain_lists), None if joins is None else list(joins), b, m)
            part_out = self._drain_results(res, None, detail)
            if joins is not None:
                for i, (d, r) in enumerate(zip(part_out, jres)):
                    nj, nf = r.n_join, r.n_unscheduled
                    d.update(n_join=nj, n_join_placed=r.n_placed, n_join_unscheduled=nf)
                    if detail:
                        d.update(zip(("join_pods", "join_node", "join_gpu_slots", "join_score", "join_fail_counts", "join_fail_pod"),
                                     self._download(L.simon_wave_join_download, i, (nj, np.uint32), (nj, np.int32), (nj, np.uint32),
                                                    (nj, np.int64), (nf, np.uint32, abi.N_FAIL_CODES), (nf, np.uint32))))
            return part_out
        out, info = self._chunked(len(remain_lists), chunk, lambda h, su, pm: L.simon_wave_times(h, su, pm, None), run)
        self.last_wave["batches"] += info["chunks"]
        self.last_wave["setup_ms"] += info["setup_ms"]
        self.last_wave["place_ms"] += info["place_ms"]
        self.last_wave["launches"] += info["launches"]
        return out

    def wave_commit(self, i: int, retire: bool = False):
        """simon_wave_commit of entry i of the last wave_run's remain_lists: it becomes the next base.  When entry i was not in the last
        batch it is run again alone first.  retire (simon_wave_commit_retire): its joined nodes become present and its drained nodes
        leave for good instead of returning."""
        lists, joins, b, m = self._wave if self._wave is not None else (None, None, 0, 0)
        if lists is not None and not b <= i < b + m:
            self.wave_run([lists[i]], joins=None if joins is None else [joins[i]], detail=False, chunk=1)
            self._wave = (lists, joins, i, 1)
            b = i
        self._check((lib().simon_wave_commit_retire if retire else lib().simon_wave_commit)(self.h, i - b))
        self._wave = None
        cm = C.c_float(0)
        self._check(lib().simon_wave_times(self.h, None, None, C.byref(cm)))
        self.last_wave["commits"] += 1
        self.last_wave["commit_ms"] += float(cm.value)

    def wave_placement(self):
        """The wave base's placement: (node per pod, GPU slot word per pod)."""
        P = self.c.pods_dims["n_pods"]
        pl = np.zeros(max(P, 1), np.int32)
        sl = np.zeros(max(P, 1), np.uint32)
        self._check(lib().simon_wave_download(self.h, pl.ctypes.data, sl.ctypes.data))
        return pl[:P], sl[:P]

    def wave_presence(self) -> np.ndarray:
        """The wave base's node states: 0 absent, 1 present, 2 retired."""
        N = self.c.n_nodes
        st = np.zeros(max(N, 1), np.uint8)
        self._check(lib().simon_wave_presence(self.h, st.ctypes.data))
        return st[:N]

    # ---- headroom probes (simon_probe_run) ----
    def probe_run(self, placed, probes, detail: bool = True, chunk: Optional[int] = None):
        """Headroom probes on the live state `placed` (out_node of a full placement of the pod list): each entry of probes is (pod,
        max_replicas), and places replicas of that pod one at a time on the state the ones before it leave, until one does not fit or
        max_replicas are placed.  The list runs in batches sized as drain_run sizes them (chunk: an explicit batch size).  Refused
        before any device work: n_pods + max_replicas past compiled.class_pod_limit of the pod's class (the int32 bounds of its
        tables).  Returns one dict per probe: n_placed, stop_reason (abi.PROBE_STOP_*) and the sums req_mcpu / alloc_mcpu / req_mem /
        alloc_mem over all nodes after the replicas, vg_requested / vg_capacity on a cluster compiled with open_local=True; with
        detail also node and gpu_slots and score per replica [n_placed] and fail_counts [24], the histogram of the replica that stopped
        it (zeros on MaxReplicas).  self.last_probe: chunks, scenario_bytes, setup_ms / place_ms (device time summed over the batches),
        launches.  scenario_storage_state(i) then describes probe i of the last chunk."""
        L = lib()
        pl = np.ascontiguousarray(placed, dtype=np.int32)
        probes = [(int(q), int(r)) for q, r in probes]
        P = self.c.pods_dims["n_pods"]
        limit = self.c.class_pod_limit
        cls = self.c.pods["pod_class"]
        for i, (q, r) in enumerate(probes):
            if limit is not None and 0 <= q < P and r > 0 and P + r > limit[int(cls[q])]:
                raise RuntimeError(f"probe {i}: {P} pods + {r} replicas of pod {q} exceed its class's int32 bounds "
                                   f"({limit[int(cls[q])]} pods)")
        local = getattr(self.c, "storage", None) is not None

        def run(b, m):
            part = probes[b:b + m]
            arr = (abi.SimonProbe * max(m, 1))(*[abi.SimonProbe(q, r) for q, r in part])
            res = (abi.SimonProbeResult * max(m, 1))()
            loc = (abi.SimonScenarioLocalResult * max(m, 1))() if local else None
            self._check(L.simon_probe_run(self.h, pl.ctypes.data, arr, m, res, loc))
            out = []
            for i in range(m):
                r = res[i]
                d = dict(n_placed=r.n_placed, stop_reason=r.stop_reason, req_mcpu=r.req_mcpu, alloc_mcpu=r.alloc_mcpu,
                         req_mem=r.req_mem, alloc_mem=r.alloc_mem)
                if local:
                    d["vg_requested"], d["vg_capacity"] = int(loc[i].vg_requested), int(loc[i].vg_capacity)
                if detail:
                    k = r.n_placed
                    d.update(zip(("node", "gpu_slots", "score", "fail_counts"),
                                 self._download(L.simon_probe_download, i, (k, np.int32), (k, np.uint32), (k, np.int64),
                                                (abi.N_FAIL_CODES, np.uint32))))
                out.append(d)
            return out
        out, self.last_probe = self._chunked(len(probes), chunk, L.simon_probe_times, run)
        if not probes:
            run(0, 0)           # no batch, but simon_probe_run still checks `placed` and drops the last batch
        return out

    # ---- grow batches (simon_grow_run) ----
    def grow_run(self, placed, n_prefix: int, scenarios: List[np.ndarray], detail: bool = True, chunk: Optional[int] = None):
        """Grow scenarios on the live state placed[:n_prefix] (out_node of the prefix pods): each entry of scenarios lists its active
        nodes in their nodeTree.list() order, and places the tail pods [n_prefix, n_pods) on them from the live state.  The list runs
        in batches sized as drain_run sizes them, where one scenario also holds its per-tail-pod outputs and failure records (16 + 4 x 24 + 4
        = 116 bytes per tail pod); chunk: an explicit batch size.  Returns one dict per scenario: n_scheduled / n_unscheduled over its
        existing tail pods that reach the scheduler and the sums req_mcpu / alloc_mcpu / req_mem / alloc_mem over its active nodes,
        vg_requested / vg_capacity on a cluster compiled with open_local=True; with detail also node, gpu_slots and score per tail pod
        [n_pods - n_prefix] (node -3: the pod does not exist in the scenario), and fail_counts [n_unscheduled][24] and fail_pod.
        self.last_grow: chunks, scenario_bytes, setup_ms / place_ms (device time summed over the batches), launches.
        scenario_storage_state(i) then describes scenario i of the last chunk."""
        L = lib()
        pl = np.ascontiguousarray(np.asarray(placed)[:n_prefix], dtype=np.int32)
        P = self.c.pods_dims["n_pods"]
        T = max(P - int(n_prefix), 0)
        local = getattr(self.c, "storage", None) is not None

        def run(b, m):
            arr, keep = self._scenario_array(scenarios[b:b + m])
            res = (abi.SimonScenarioResult * m)()
            loc = (abi.SimonScenarioLocalResult * m)() if local else None
            self._check(L.simon_grow_run(self.h, pl.ctypes.data if n_prefix else None, int(n_prefix), arr, m, res, loc))
            out = []
            for i, r in enumerate(res):
                d = dict(n_unscheduled=r.n_unscheduled, n_scheduled=r.n_scheduled, req_mcpu=r.req_mcpu, alloc_mcpu=r.alloc_mcpu,
                         req_mem=r.req_mem, alloc_mem=r.alloc_mem)
                if local:
                    d["vg_requested"], d["vg_capacity"] = int(loc[i].vg_requested), int(loc[i].vg_capacity)
                if detail:
                    nf = r.n_unscheduled
                    d.update(zip(("node", "gpu_slots", "score", "fail_counts", "fail_pod"),
                                 self._download(L.simon_grow_download, i, (T, np.int32), (T, np.uint32), (T, np.int64),
                                                (nf, np.uint32, abi.N_FAIL_CODES), (nf, np.uint32))))
                out.append(d)
            return out
        out, self.last_grow = self._chunked(len(scenarios), chunk, L.simon_grow_times, run, extra=(16 + 4 * abi.N_FAIL_CODES + 4) * T)
        return out

    # ---- trace replay (simon_trace_run) ----
    def trace_run(self, placed, n_prefix: int, events, scenarios: Optional[List[np.ndarray]] = None, samples=None, detail: bool = True,
                  chunk: Optional[int] = None) -> List[dict]:
        """Replay `events` ((op, pod) pairs, op abi.TRACE_CREATE / abi.TRACE_DELETE) on the live state placed[:n_prefix] in each scenario
        (scenarios: node lists as grow_run takes them; None: one scenario on every node in index order).  samples: ascending event
        indices after which the state is recorded.  The scenarios run in batches sized as grow_run sizes them (chunk: an explicit batch
        size).  Returns one dict per scenario: n_scheduled / n_unscheduled (creates placed and failed), n_removed (deletes that took a
        pod off a node), n_running and the sums req_mcpu / alloc_mcpu / req_mem / alloc_mem after the last event, samples (a structured
        array of abi.TRACE_POINT_DTYPE); with detail also node, gpu_slots and score per tail pod [n_pods - n_prefix], and fail_counts
        [n_unscheduled][24] and fail_pod.  self.last_trace: chunks, scenario_bytes, setup_ms / place_ms (device time summed over the
        batches), runs and launches of the runs and samples (summed), launches (last_launch() of each batch)."""
        L = lib()
        pl = np.ascontiguousarray(np.asarray(placed)[:n_prefix], dtype=np.int32)
        P = self.c.pods_dims["n_pods"]
        T = max(P - int(n_prefix), 0)
        ev = np.ascontiguousarray(np.asarray(events, dtype=np.uint32).reshape(-1, 2))
        sm = np.ascontiguousarray(np.asarray([] if samples is None else samples, dtype=np.uint32))
        ns = len(sm)
        single = scenarios is None
        n_scen = 1 if single else len(scenarios)
        info = dict(runs=0, run_launches=0)

        def run(b, m):
            arr, keep = (None, None) if single else self._scenario_array(scenarios[b:b + m])
            res = (abi.SimonTraceResult * max(m, 1))()
            self._check(L.simon_trace_run(self.h, pl.ctypes.data if n_prefix else None, int(n_prefix), ev.ctypes.data if len(ev) else None,
                                          len(ev), arr, m, sm.ctypes.data if ns else None, ns, res))
            nr, nl = C.c_uint32(0), C.c_uint64(0)
            self._check(L.simon_trace_times(self.h, None, None, C.byref(nr), C.byref(nl)))
            info["runs"] += nr.value
            info["run_launches"] += nl.value
            out = []
            for i in range(m):
                r = res[i]
                d = dict(n_scheduled=r.n_scheduled, n_unscheduled=r.n_unscheduled, n_removed=r.n_removed, n_running=r.n_running,
                         req_mcpu=r.req_mcpu, alloc_mcpu=r.alloc_mcpu, req_mem=r.req_mem, alloc_mem=r.alloc_mem)
                pts = np.zeros(max(ns, 1), abi.TRACE_POINT_DTYPE)
                self._check(L.simon_trace_samples_download(self.h, i, pts.ctypes.data))
                d["samples"] = pts[:ns]
                if detail:
                    nf = r.n_unscheduled
                    d.update(zip(("node", "gpu_slots", "score", "fail_counts", "fail_pod"),
                                 self._download(L.simon_trace_download, i, (T, np.int32), (T, np.uint32), (T, np.int64),
                                                (nf, np.uint32, abi.N_FAIL_CODES), (nf, np.uint32))))
                out.append(d)
            return out
        out, self.last_trace = self._chunked(n_scen, 1 if single else chunk, lambda h, su, pm: L.simon_trace_times(h, su, pm, None, None),
                                             run, extra=(16 + 4 * abi.N_FAIL_CODES + 4) * T + C.sizeof(abi.SimonTracePoint) * ns)
        self.last_trace.update(info)
        return out
