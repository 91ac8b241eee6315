/*
 * trace_oracle.c — CPU checker of trace replays (simon_trace_run, include/simon_gpu.h).  TEST INFRASTRUCTURE ONLY.
 *
 * The move-scope checker (and through it the CPU oracle) is compiled into this library unchanged.  One scenario is replayed one event at
 * a time with the oracle's own primitives, by a different mechanism from the engine's (runs of creates in one launch, runs of deletes
 * in another, state rebuilt once and copied):
 *   1. reset; the scenario's nodes become the active set, in their order; every placed prefix pod is committed on its node in pod order,
 *      with Reserve for the pods that went through the scheduler (as the grow checker does);
 *   2. a create is simon_oracle_schedule of that one pod on the active nodes;
 *   3. a delete of a pod that holds a node is uncommit() there plus the release of its device memory as its slot word states it (as the
 *      migration-plan checker does); a pod that holds no node leaves nothing;
 *   4. after every event, the sums the samples report over the active nodes.
 */
#include "moves_scope_oracle.c"

#define TRACE_SAMPLE_W 10   /* running, failed, idle devices, partial devices, req / alloc mcpu, req / alloc mem, gpu used / total */

/* events: n_events pairs (op, pod).  Per tail pod out_node / out_score / out_slots; the failed creates in event order (out_fail_counts
 * [n][SIMON_N_FAIL_CODES], out_fail_pod); counts[4] = scheduled, failed, removed, running; samples (may be NULL) [n_events][10]. */
int simon_oracle_trace(simon_oracle *o, const int32_t *placed, uint32_t n_prefix, const uint32_t *nodes, uint32_t n_nodes,
                       const uint32_t *events, uint32_t n_events, int32_t *out_node, int64_t *out_score, uint32_t *out_slots,
                       uint32_t *out_fail_counts, uint32_t *out_fail_pod, uint32_t *counts, int64_t *samples) {
    const uint32_t P = o->p.n_pods, N = o->N;
    if (n_prefix > P) return SIMON_ERR_INVALID;
    simon_oracle_reset(o);
    simon_oracle_set_active(o, nodes, n_nodes);
    int32_t *where = (int32_t *)malloc(4ull * (P + 1));
    uint32_t *slot = (uint32_t *)calloc(P + 1, 4);
    uint32_t sched = 0, failed = 0, removed = 0, running = 0;
    for (uint32_t q = 0; q < P; q++) where[q] = -1;
    for (uint32_t q = 0; q < n_prefix; q++) {
        const int32_t g = placed[q];
        if (g < 0) continue;
        if ((uint32_t)g >= N || !o->active[g]) { free(where); free(slot); return SIMON_ERR_INVALID; }
        const int32_t fixed = o->p.pod_fixed_node[q];
        o->cur_pin = o->p.pod_pin_node ? o->p.pod_pin_node[q] : -1;
        const uint32_t pack = commit(o, CW(o, (uint32_t)o->p.pod_class[q]), (uint32_t)g, fixed == -1);
        slot[q] = fixed == -1 ? pack : 0;
        where[q] = g;
        running++;
    }
    for (uint32_t e = 0; e < n_events; e++) {
        const uint32_t op = events[2 * e], q = events[2 * e + 1];
        if (q >= P) { free(where); free(slot); return SIMON_ERR_INVALID; }
        const int64_t *cw = CW(o, (uint32_t)o->p.pod_class[q]);
        if (op == SIMON_TRACE_CREATE) {
            if (q < n_prefix) { free(where); free(slot); return SIMON_ERR_INVALID; }
            int32_t node;
            int64_t score = 0;
            uint32_t f = 0;
            const int rc = simon_oracle_schedule(o, q, 1, &node, &score, out_fail_counts + (uint64_t)failed * SIMON_N_FAIL_CODES,
                                                 out_fail_pod + failed, 1, &f);
            if (rc) { free(where); free(slot); return rc; }
            out_node[q - n_prefix] = node;
            out_score[q - n_prefix] = score;
            out_slots[q - n_prefix] = o->gpu_slots[q];
            failed += f;
            if (node >= 0) { where[q] = node; slot[q] = o->gpu_slots[q]; running++; if (o->p.pod_fixed_node[q] == -1) sched++; }
        } else if (op == SIMON_TRACE_DELETE) {
            const int32_t g = where[q];
            if (g >= 0) {
                uncommit(o, cw, (uint32_t)g);
                if (cw[SCW_GPU_MEM] > 0)
                    for (int d = 0; d < SIMON_MAX_GPU_DEV; d++) o->gpu_used[(uint64_t)d * N + g] -= (int64_t)((slot[q] >> (4 * d)) & 15u) * cw[SCW_GPU_MEM];
                where[q] = -1;
                removed++;
                running--;
            }
        } else {
            free(where); free(slot); return SIMON_ERR_INVALID;
        }
        if (samples) {
            int64_t *s = samples + (uint64_t)e * TRACE_SAMPLE_W;
            memset(s, 0, 8 * TRACE_SAMPLE_W);
            s[0] = running; s[1] = failed;
            for (uint32_t r = 0; r < n_nodes; r++) {
                const uint32_t g = nodes[r];
                s[4] += o->req_mcpu[g]; s[5] += o->s.alloc_mcpu[g]; s[6] += o->req_mem[g]; s[7] += o->s.alloc_mem[g];
                const int32_t nd = o->s.gpu_count ? o->s.gpu_count[g] : 0;
                for (int32_t d = 0; d < nd && d < SIMON_MAX_GPU_DEV; d++) {
                    const int64_t u = o->gpu_used[(uint64_t)d * N + g], cap = o->s.gpu_dev_mem[g];
                    s[8] += u; s[9] += cap;
                    s[2] += u == 0; s[3] += u > 0 && u < cap;
                }
            }
        }
    }
    counts[0] = sched; counts[1] = failed; counts[2] = removed; counts[3] = running;
    free(where); free(slot);
    return SIMON_OK;
}
