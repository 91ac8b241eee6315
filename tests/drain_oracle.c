/*
 * drain_oracle.c — CPU checker of node drains (simon_drain_run, include/simon_gpu.h).  TEST INFRASTRUCTURE ONLY, like the oracle
 * it is built on.
 *
 * The CPU oracle (oracle/simon_oracle.c) is compiled into this library unchanged.  One drain is evaluated by a different mechanism
 * from the engine's (live state copied into every scenario, then the removed pods taken out of the counters): the state is built up
 * from empty on the remaining nodes only.
 *   1. reset; 2. the remaining nodes become the active set, in their order;
 *   3. every placed pod that sits on a remaining node is committed there in pod order - Reserve (GPU-share devices) for the pods
 *      that went through the scheduler, none for pre-bound ones, as simon_oracle_schedule does;
 *   4. the pods of removed nodes are classified (vanished: DaemonSet pods of a removed node; blocked: bound by spec.nodeName or of
 *      a class with Open-Local volumes; evicted: the rest) and each evicted pod is scheduled in pod order.
 */
#include "../oracle/simon_oracle.c"

/* counts[5]: evicted, placed, unscheduled, blocked, vanished.  Per evicted pod in pod order (arrays of n_pods entries suffice):
 * out_evicted (pod index), out_node (-1 unschedulable), out_score, out_slots (4 bits per device); out_blocked: blocked pods in
 * pod order; failures in order: out_fail_counts [n][SIMON_N_FAIL_CODES], out_fail_pod.  class_local: NULL, or per class 1 = Open-Local
 * volumes.  The oracle's state afterwards is the drain's end state (simon_oracle_state / _state_ext). */
int simon_oracle_drain(simon_oracle *o, const int32_t *placed, const uint32_t *remain, uint32_t n_remain, const uint8_t *class_local,
                       uint32_t *counts, uint32_t *out_evicted, int32_t *out_node, int64_t *out_score, uint32_t *out_slots,
                       uint32_t *out_blocked, uint32_t *out_fail_counts, uint32_t *out_fail_pod) {
    const uint32_t P = o->p.n_pods, N = o->N;
    simon_oracle_reset(o);
    simon_oracle_set_active(o, remain, n_remain);
    memset(counts, 0, 5 * sizeof(uint32_t));
    uint32_t *ev = (uint32_t *)malloc(4ull * (P + 1));
    uint32_t n_ev = 0;
    for (uint32_t q = 0; q < P; q++) {
        const int32_t g = placed[q];
        if (g < 0) continue;
        if ((uint32_t)g >= N) { free(ev); return SIMON_ERR_INVALID; }
        const uint32_t cls = (uint32_t)o->p.pod_class[q];
        const int64_t *cw = CW(o, cls);
        const int32_t fixed = o->p.pod_fixed_node[q];
        if (o->active[g]) {
            const uint32_t pack = commit(o, cw, (uint32_t)g, fixed == -1);
            o->gpu_slots[q] = fixed == -1 ? pack : 0;
            continue;
        }
        int64_t guard = cw[SCW_GUARD_NODE];
        if (guard == -3) guard = o->p.pod_pin_node ? o->p.pod_pin_node[q] : -1;
        if (guard >= 0 && !o->active[guard]) counts[4]++;
        else if (fixed >= 0 || (class_local && class_local[cls])) out_blocked[counts[3]++] = q;
        else ev[n_ev++] = q;
    }
    uint32_t n_fail = 0;
    for (uint32_t j = 0; j < n_ev; j++) {
        const uint32_t q = ev[j], cls = (uint32_t)o->p.pod_class[q];
        const int64_t *cw = CW(o, cls);
        o->cur_pin = o->p.pod_pin_node ? o->p.pod_pin_node[q] : -1;
        uint32_t hist[SIMON_N_FAIL_CODES];
        int64_t score = 0;
        const int64_t n = schedule_one(o, cls, &score, hist);
        if (n == -2) { free(ev); return SIMON_ERR_LIMIT; }
        out_evicted[j] = q;
        out_node[j] = (int32_t)n;
        out_slots[j] = 0;
        if (n >= 0) {
            out_slots[j] = commit(o, cw, (uint32_t)n, 1);
            o->gpu_slots[q] = out_slots[j];
            counts[1]++;
        } else {
            memcpy(out_fail_counts + (uint64_t)n_fail * SIMON_N_FAIL_CODES, hist, sizeof(hist));
            out_fail_pod[n_fail++] = q;
            score = 0;
        }
        out_score[j] = score;
    }
    counts[0] = n_ev;
    counts[2] = n_fail;
    free(ev);
    return SIMON_OK;
}
