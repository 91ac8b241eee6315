// simon_select.cuh — node-selection programs and spreading eligibility on the device (include/simon_gpu.h, SCW_OFF_SEL): shared by
// the placement kernel and the trace-removal kernel (simon_trace.cu), which is a translation unit of its own.
#pragma once
#include "simon_kernel.cuh"

struct ReqCtx {
    const uint64_t *label_bits;
    uint32_t N;
    int32_t pin;        // pin node of the pod being evaluated (simon_podset.pod_pin_node), -1 none: what REQ_NODE_IS payload -3 means
};

__device__ inline bool req_eval(const int64_t *&p, const ReqCtx &c, uint32_t g) {
    int64_t head = *p++;
    int op = (int)(head & 0xff);
    if (op == SIMON_REQ_NODE_IS || op == SIMON_REQ_NODE_ISNOT) {
        int64_t idx = *p++;
        if (idx == -3) idx = c.pin;          // the pod's own pin (DaemonSet pods, pkg/utils/utils.go:770-815)
        return op == SIMON_REQ_NODE_IS ? ((int64_t)g == idx) : ((int64_t)g != idx);
    }
    int nw = (int)((head >> 8) & 0xff);
    bool any = false;
    #pragma unroll 1
    for (int i = 0; i < nw; i++) {
        int64_t wi = *p++;
        uint64_t mask = (uint64_t)*p++;
        if (__ldg(c.label_bits + (uint64_t)wi * c.N + g) & mask) any = true;
    }
    return op == SIMON_REQ_ANY ? any : !any;
}

__device__ inline bool term_eval(const int64_t *&p, const ReqCtx &c, uint32_t g) {
    int64_t nreq = *p++;
    bool ok = true;
    #pragma unroll 1
    for (int64_t i = 0; i < nreq; i++)
        if (!req_eval(p, c, g)) ok = false;
    return ok;
}

// PodMatchesNodeSelectorAndAffinityTerms (helper/node_affinity.go:27-71) over the compiled program
__device__ inline bool selection_ok(const int64_t *cw, const ReqCtx &c, uint32_t g) {
    const int64_t *p = cw + cw[SCW_OFF_SEL];
    bool ok = true;
    int64_t n_ns = *p++;
    #pragma unroll 1
    for (int64_t q = 0; q < n_ns; q++)
        if (!req_eval(p, c, g)) ok = false;
    int64_t has_required = *p++, n_terms = *p++;
    bool any = false;
    #pragma unroll 1
    for (int64_t q = 0; q < n_terms; q++)
        if (term_eval(p, c, g)) any = true;
    if (has_required && !any) ok = false;
    return ok;
}

// eligibility of node g for the spreading counts of class `sig` (scoring.go:140-148)
__device__ __noinline__ bool elig_eval(const SkParams &P, int64_t sig, const ReqCtx &c, uint32_t g) {
    const int64_t *cw = P.class_blob + P.class_off[sig];
    if (!selection_ok(cw, c, g)) return false;
    const int64_t *soft = cw + cw[SCW_OFF_PTS_SOFT];
    #pragma unroll 1
    for (int64_t j = 0; j < cw[SCW_N_PTS_SOFT]; j++)
        if (P.topo_dom[(uint64_t)soft[5 * j + 1] * P.N + g] < 0) return false;
    return true;
}
