// simon_pdb.cu — PodDisruptionBudgets for drains, move scoring and migration plans (simon_pdbs_upload, include/simon_gpu.h).
//
// The table is two CSRs uploaded once per pod list: pod -> its PDBs (ascending) and PDB -> its member pods, plus each PDB's
// desired healthy count (computed by the host compiler, simon_b200/disruption.py).  On a placement:
//   healthy[j] = members of j that are placed,  allowed[j] = max(0, healthy[j] - desired[j]).
// Drains compare each drain's evicted members per PDB with `allowed` on the host (simon_drain_run); move runs and plans mark the pods
// of PDBs without budget never movable in their packed SmvPod records, so the scoring kernels skip them unchanged.  In a plan every
// applied step spends one unit of each PDB of the moved pod (simon_pdb_step); a PDB that reaches 0 marks its members
// (simon_pdb_mark_hit).  None of these kernels runs without a table.
//
// This file is a translation unit of its own, linked into libsimon_gpu.so next to simon_api.cu: the library's main module keeps
// exactly the kernels it had before PDBs existed, and simon_api.cu reaches these through the launch functions of simon_pdb.cuh.
#include <cuda_runtime.h>

#include "../../include/simon_gpu.h"
#include "simon_moves.cuh"
#include "simon_pdb.cuh"

// healthy[j] += 1 for each PDB j of each placed pod (healthy cleared by the caller)
__global__ void simon_pdb_healthy(uint32_t n_pods, const int32_t *placement, const uint32_t *pod_off, const uint32_t *pod_pdb,
                                  int32_t *healthy) {
    for (uint32_t q = blockIdx.x * blockDim.x + threadIdx.x; q < n_pods; q += gridDim.x * blockDim.x) {
        if (placement[q] < 0) continue;
        for (uint32_t k = pod_off[q]; k < pod_off[q + 1]; k++) atomicAdd(healthy + pod_pdb[k], 1);
    }
}

// in place: healthy -> allowed = max(0, healthy - desired)
__global__ void simon_pdb_allowed(uint32_t n_pdbs, const int32_t *desired, int32_t *healthy) {
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n_pdbs; j += gridDim.x * blockDim.x)
        healthy[j] = max(0, healthy[j] - desired[j]);
}

// Pods with a PDB whose remaining budget is 0 become never movable.  blocked (may be NULL) counts the placed ones that nothing else
// had made never movable (pinned, Open-Local, excluded GPU-share pods): simon_moves_plan_result.n_pdb_blocked.
__global__ void simon_pdb_mark(uint32_t n_pods, const uint32_t *pod_off, const uint32_t *pod_pdb, const int32_t *remaining,
                               SmvPod *pods, uint32_t *blocked) {
    for (uint32_t q = blockIdx.x * blockDim.x + threadIdx.x; q < n_pods; q += gridDim.x * blockDim.x) {
        bool out = false;
        for (uint32_t k = pod_off[q]; k < pod_off[q + 1] && !out; k++) out = remaining[pod_pdb[k]] <= 0;
        if (!out) continue;
        const SmvPod r = pods[q];
        pods[q].bits = r.bits | SMC_NOT_MOVABLE | SMC_NEVER;
        if (blocked && r.node >= 0 && !(r.bits & SMC_NEVER)) atomicAdd(blocked, 1u);
    }
}

// After simon_moves_plan_apply (one warp).  pctl[0]: steps this kernel has seen, pctl[1]: PDBs that reached 0 at the last step (their
// ids in hit).  A step recorded since the last call spends one unit of every PDB of its pod.
__global__ void __launch_bounds__(32) simon_pdb_step(const uint32_t *ctl, const simon_plan_step *steps, const uint32_t *pod_off,
                                                     const uint32_t *pod_pdb, int32_t *remaining, uint32_t *pctl, uint32_t *hit) {
    const uint32_t lane = threadIdx.x, s = ctl[0], seen = pctl[0];
    __syncwarp();
    if (lane == 0) pctl[1] = 0u;
    __syncwarp();
    if (s == seen) return;
    const uint32_t p = steps[s - 1].pod;
    for (uint32_t k = pod_off[p] + lane; k < pod_off[p + 1]; k += 32) {
        const uint32_t j = pod_pdb[k];
        if (atomicSub(remaining + j, 1) == 1) hit[atomicAdd(pctl + 1, 1u)] = j;
    }
    if (lane == 0) pctl[0] = s;
}

// The members of the PDBs simon_pdb_step found at 0 become never movable; returns at once when there are none.
__global__ void simon_pdb_mark_hit(const uint32_t *pctl, const uint32_t *hit, const uint32_t *pdb_off, const uint32_t *pdb_pod,
                                   SmvPod *pods) {
    const uint32_t n = pctl[1];
    for (uint32_t h = 0; h < n; h++) {
        const uint32_t j = hit[h], b = pdb_off[j], e = pdb_off[j + 1];
        for (uint32_t k = b + blockIdx.x * blockDim.x + threadIdx.x; k < e; k += gridDim.x * blockDim.x)
            pods[pdb_pod[k]].bits |= SMC_NOT_MOVABLE | SMC_NEVER;
    }
}

// ---- launch functions (simon_pdb.cuh) ----
static unsigned grid_for(uint32_t n, uint32_t cap) { return n ? ((n + 255) / 256 < cap ? (n + 255) / 256 : cap) : 1u; }

cudaError_t simon_pdb_launch_allowed(cudaStream_t st, uint32_t grid_cap, uint32_t n_pods, const int32_t *placement, const uint32_t *pod_off,
                                     const uint32_t *pod_pdb, uint32_t n_pdbs, const int32_t *desired, int32_t *allowed) {
    cudaError_t e = cudaMemsetAsync(allowed, 0, 4ull * n_pdbs, st);
    if (e != cudaSuccess) return e;
    simon_pdb_healthy<<<grid_for(n_pods, grid_cap), 256, 0, st>>>(n_pods, placement, pod_off, pod_pdb, allowed);
    simon_pdb_allowed<<<grid_for(n_pdbs, grid_cap), 256, 0, st>>>(n_pdbs, desired, allowed);
    return cudaGetLastError();
}

cudaError_t simon_pdb_launch_mark(cudaStream_t st, uint32_t grid_cap, uint32_t n_pods, const uint32_t *pod_off, const uint32_t *pod_pdb,
                                  const int32_t *remaining, SmvPod *pods, uint32_t *blocked) {
    simon_pdb_mark<<<grid_for(n_pods, grid_cap), 256, 0, st>>>(n_pods, pod_off, pod_pdb, remaining, pods, blocked);
    return cudaGetLastError();
}

cudaError_t simon_pdb_launch_step(cudaStream_t st, uint32_t grid_cap, const uint32_t *ctl, const simon_plan_step *steps, const uint32_t *pod_off,
                                  const uint32_t *pod_pdb, int32_t *remaining, uint32_t *pctl, uint32_t *hit, uint32_t max_members,
                                  const uint32_t *pdb_off, const uint32_t *pdb_pod, SmvPod *pods) {
    simon_pdb_step<<<1, 32, 0, st>>>(ctl, steps, pod_off, pod_pdb, remaining, pctl, hit);
    simon_pdb_mark_hit<<<grid_for(max_members, grid_cap), 256, 0, st>>>(pctl, hit, pdb_off, pdb_pod, pods);
    return cudaGetLastError();
}
