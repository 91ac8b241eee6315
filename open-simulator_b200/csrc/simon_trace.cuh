// simon_trace.cuh — launch functions of the trace-replay kernels (simon_trace.cu, its own translation unit).  Each enqueues one launch
// on `st`.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "simon_kernel.cuh"

// Per scenario of a trace batch, on the device: creates placed and failed, and deletes that took a pod off a node, summed over the
// runs folded so far.  The placement kernel writes each create run's counts into the scenario's n_sched / n_fail and its failure
// records from the scenario's fail_counts / fail_pod; the next removal or sample launch folds them into these words, zeroes the
// counts and moves the record pointers past the run's records, so the next create run writes after them.
struct SkTraceAcc {
    uint32_t sched, fail, removed, pad;
};

// One delete run on n scenarios: pods[0 .. nd) leave the nodes they hold in each scenario.  A prefix pod's node and slot word are
// prefix_node / prefix_gpu; tail pod q's in scenario s are tail_node / tail_gpu[s * stride + q].
cudaError_t simon_trace_launch_remove(cudaStream_t st, uint32_t grid_cap, const SkParams &P, SkScenario *scen, uint32_t n,
                                      const uint32_t *pods, uint32_t nd, const int32_t *prefix_node, const uint32_t *prefix_gpu,
                                      uint32_t n_prefix, const int32_t *tail_node, const uint32_t *tail_gpu, uint32_t stride,
                                      SkTraceAcc *acc);
// One sample on n scenarios: record s of out[s * n_samples + at] describes scenario s after event `event`; placed_prefix is the
// number of prefix pods on nodes in the live state.
cudaError_t simon_trace_launch_sample(cudaStream_t st, const SkParams &P, SkScenario *scen, uint32_t n, SkTraceAcc *acc,
                                      uint32_t placed_prefix, uint32_t event, simon_trace_point *out, uint32_t n_samples, uint32_t at);
