// simon_pdb.cuh — launch functions of the PodDisruptionBudget kernels (simon_pdb.cu, its own translation unit).  Each enqueues on
// `st`; grids are capped at grid_cap CTAs of 256 threads.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/simon_gpu.h"
#include "simon_moves.cuh"

// allowed[j] = max(0, placed members of j - desired[j]) on `placement` (two launches)
cudaError_t simon_pdb_launch_allowed(cudaStream_t st, uint32_t grid_cap, uint32_t n_pods, const int32_t *placement, const uint32_t *pod_off,
                                     const uint32_t *pod_pdb, uint32_t n_pdbs, const int32_t *desired, int32_t *allowed);
// pods of PDBs at remaining <= 0 become never movable in their SmvPod; blocked (may be NULL) counts the placed ones nothing else
// had made never movable (one launch)
cudaError_t simon_pdb_launch_mark(cudaStream_t st, uint32_t grid_cap, uint32_t n_pods, const uint32_t *pod_off, const uint32_t *pod_pdb,
                                  const int32_t *remaining, SmvPod *pods, uint32_t *blocked);
// after a plan step's apply: spend the moved pod's PDBs and mark the members of those that reach 0 (two launches)
cudaError_t simon_pdb_launch_step(cudaStream_t st, uint32_t grid_cap, const uint32_t *ctl, const simon_plan_step *steps, const uint32_t *pod_off,
                                  const uint32_t *pod_pdb, int32_t *remaining, uint32_t *pctl, uint32_t *hit, uint32_t max_members,
                                  const uint32_t *pdb_off, const uint32_t *pdb_pod, SmvPod *pods);
