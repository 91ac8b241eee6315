// simon_trace.cu — trace replay (simon_trace_run, include/simon_gpu.h): the removal of a run of deleted pods and the samples.
//
// The creates of a trace are placed by the scenario-batch placement kernels, one launch per run of creates over its pod range; the
// deletes between them are removed here, one thread per (scenario, deleted pod), from the scenario's own state on the device.  A
// removal is the inverse of what the import and the placement kernel's commit add: requests, non-zero requests, pod count, scalars,
// the class's counter increments (eligibility-conditional ones as simon_import_kernel counts them) and the GPU-share memory the slot
// word states.  The deletes of one run may share a node, so every subtraction is an atomic.
//
// What a removal leaves stale in the placement kernel's per-class caches:
//   own-score cache (ocache[cls * N + g]): keyed by the node's pod count + 1, which a delete followed by a create on the same node
//     returns to while the node's requests differ.  Every class's entry of a node a delete touches is dropped (0 = empty).
//   feasible-set summaries (csum) and their feasibility bits (fbits): a summary is a function of the feasible set its bits describe,
//     and every decision re-evaluates every node's feasibility against the restored bits in both directions; a node that became
//     feasible after a delete is a flip like any other and rebuilds the summary.  Nothing to drop.
//   predicted topology sizes (in csum): exact for the stored bits, or verified by the summary rebuild.  Nothing to drop.
//
// This file is a translation unit of its own, linked into libsimon_gpu.so next to simon_api.cu, so that the main module keeps exactly
// the kernels it had; simon_api.cu reaches these through the launch functions of simon_trace.cuh.
#include <cuda_runtime.h>

#include <algorithm>

#include "simon_kernel.cuh"
#include "simon_trace.cuh"
namespace {      // the main module defines the same helpers with external linkage
#include "simon_select.cuh"
}  // namespace

// the counts of the scenario's last create run into its accumulator, and its record pointers past that run's failure records
__device__ __forceinline__ void trace_fold(SkScenario &SC, SkTraceAcc &a) {
    const uint32_t nf = *SC.n_fail, ns = *SC.n_sched;
    a.sched += ns;
    a.fail += nf;
    *SC.n_fail = 0;
    *SC.n_sched = 0;
    SC.fail_counts += (uint64_t)nf * SIMON_N_FAIL_CODES;
    SC.fail_pod += nf;
}

__device__ __forceinline__ void sub64(int64_t *p, int64_t v) {
    if (v) atomicAdd((unsigned long long *)p, (unsigned long long)(-v));
}

__global__ void __launch_bounds__(256) simon_trace_remove(const __grid_constant__ SkParams P, SkScenario *scen, uint32_t n, const uint32_t *pods,
                                                          uint32_t nd, const int32_t *prefix_node, const uint32_t *prefix_gpu,
                                                          uint32_t n_prefix, const int32_t *tail_node, const uint32_t *tail_gpu,
                                                          uint32_t stride, SkTraceAcc *acc) {
    const ReqCtx RC{P.label_bits, P.N, -1};
    const uint32_t N = P.N, K = P.K;
    for (uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; j < (uint64_t)n * nd; j += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t s = (uint32_t)(j / nd), k = (uint32_t)(j % nd);
        SkScenario &SC = scen[s];
        if (k == 0) trace_fold(SC, acc[s]);
        const uint32_t q = pods[k];
        const uint64_t at = (uint64_t)s * stride + q;
        const int32_t g = q < n_prefix ? prefix_node[q] : tail_node[at];
        if (g < 0) continue;
        const uint32_t w = q < n_prefix ? prefix_gpu[q] : tail_gpu[at];
        const int64_t *cw = P.class_blob + P.class_off[P.pod_class[q]];
        sub64(&SC.req_mcpu[g], cw[SCW_REQ_MCPU]); sub64(&SC.req_mem[g], cw[SCW_REQ_MEM]); sub64(&SC.req_eph[g], cw[SCW_REQ_EPH]);
        sub64(&SC.nz_mcpu[g], cw[SCW_NZ_MCPU]); sub64(&SC.nz_mem[g], cw[SCW_NZ_MEM]);
        atomicSub(&SC.num_pods[g], 1);
        const int64_t *sc = cw + cw[SCW_OFF_SCALARS];
        for (uint32_t r = 0; r < K; r++) sub64(&SC.req_scalar[(uint64_t)r * N + g], sc[r]);
        const int64_t *inc = cw + cw[SCW_OFF_INC];
        for (int64_t u = 0; u < cw[SCW_N_INC]; u++) {
            const int64_t c = inc[3 * u], t = inc[3 * u + 1], sig = inc[3 * u + 2];
            const int32_t d = P.topo_dom[(uint64_t)t * N + g];
            if (d < 0) continue;
            if (sig >= 0 && !elig_eval(P, sig, RC, (uint32_t)g)) continue;
            atomicSub(&SC.cnt[P.cnt_off[c] + d], 1);
            atomicSub(&SC.cnt_total[c], 1);
        }
        if (cw[SCW_GPU_MEM] > 0)
            for (int d = 0; d < SIMON_MAX_GPU_DEV; d++) sub64(&SC.gpu_used[(uint64_t)d * N + g], (int64_t)((w >> (4 * d)) & 15u) * cw[SCW_GPU_MEM]);
        for (uint32_t c = 0; c < P.n_classes; c++) SC.ocache[(uint64_t)c * N + g] = 0ull;
        atomicAdd(&acc[s].removed, 1u);
    }
}

// One CTA of 256 threads per scenario: the sums over its active nodes, as simon_scen_reduce computes them, and its GPU-share devices.
__global__ void __launch_bounds__(256) simon_trace_sample(const __grid_constant__ SkParams P, SkScenario *scen, SkTraceAcc *acc,
                                                          uint32_t placed_prefix, uint32_t event, simon_trace_point *out, uint32_t n_samples,
                                                          uint32_t at) {
    SkScenario &SC = scen[blockIdx.x];
    const uint32_t N = P.N;
    long long v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (uint32_t r = threadIdx.x; r < SC.n_active; r += blockDim.x) {
        const uint32_t g = SC.order ? SC.order[r] : r;
        v[0] += SC.req_mcpu[g]; v[1] += P.alloc_mcpu[g]; v[2] += SC.req_mem[g]; v[3] += P.alloc_mem[g];
        const int32_t nd = P.gpu_count ? P.gpu_count[g] : 0;
        const int64_t cap = P.gpu_dev_mem[g];
        for (int32_t d = 0; d < nd && d < SIMON_MAX_GPU_DEV; d++) {
            const int64_t u = SC.gpu_used[(uint64_t)d * N + g];
            v[4] += u; v[5] += cap;
            v[6] += u == 0; v[7] += u > 0 && u < cap;
        }
    }
    __shared__ long long part[8][8];
#pragma unroll
    for (int q = 0; q < 8; q++) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[q] += __shfl_down_sync(0xffffffffu, v[q], o);
        if ((threadIdx.x & 31) == 0) part[q][threadIdx.x >> 5] = v[q];
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        long long t[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        for (int q = 0; q < 8; q++)
            for (unsigned w = 0; w < (blockDim.x + 31) / 32; w++) t[q] += part[q][w];
        SkTraceAcc &a = acc[blockIdx.x];
        trace_fold(SC, a);
        simon_trace_point o;
        o.event = event;
        o.n_running = placed_prefix + a.sched - a.removed;
        o.n_failed = a.fail;
        o.idle_devices = (uint32_t)t[6]; o.partial_devices = (uint32_t)t[7]; o.reserved = 0;
        o.req_mcpu = t[0]; o.alloc_mcpu = t[1]; o.req_mem = t[2]; o.alloc_mem = t[3]; o.gpu_used = t[4]; o.gpu_total = t[5];
        out[(uint64_t)blockIdx.x * n_samples + at] = o;
    }
}

cudaError_t simon_trace_launch_remove(cudaStream_t st, uint32_t grid_cap, const SkParams &P, SkScenario *scen, uint32_t n,
                                      const uint32_t *pods, uint32_t nd, const int32_t *prefix_node, const uint32_t *prefix_gpu,
                                      uint32_t n_prefix, const int32_t *tail_node, const uint32_t *tail_gpu, uint32_t stride,
                                      SkTraceAcc *acc) {
    const uint64_t total = (uint64_t)n * nd;
    const uint32_t grid = (uint32_t)std::min<uint64_t>((total + 255) / 256, grid_cap);
    simon_trace_remove<<<grid ? grid : 1, 256, 0, st>>>(P, scen, n, pods, nd, prefix_node, prefix_gpu, n_prefix, tail_node, tail_gpu, stride, acc);
    return cudaGetLastError();
}

cudaError_t simon_trace_launch_sample(cudaStream_t st, const SkParams &P, SkScenario *scen, uint32_t n, SkTraceAcc *acc,
                                      uint32_t placed_prefix, uint32_t event, simon_trace_point *out, uint32_t n_samples, uint32_t at) {
    simon_trace_sample<<<n, 256, 0, st>>>(P, scen, acc, placed_prefix, event, out, n_samples, at);
    return cudaGetLastError();
}
