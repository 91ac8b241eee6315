/*
 * replace_oracle.c — CPU checker of node-pool replacement waves (simon_wave_run_join / simon_wave_commit_retire, include/simon_gpu.h).
 * TEST INFRASTRUCTURE ONLY, like the oracle it is built on.
 *
 * The rolling-wave checker (and through it the move-scope checker and the CPU oracle) is compiled into this library unchanged.  The
 * oracle's state is the wave base.  One wave is applied with the oracle's own primitives, by a different mechanism from the engine's
 * (base copied into a slot, counters of the drained pods taken out, one pod list per scenario, state copied back):
 *   1. every pod of a node missing from `remain` is uncommitted there in pod order, its device memory released as its slot word
 *      states, and classified as simon_drain_run classifies it (vanished, blocked, evicted);
 *   2. the remaining nodes (the joined ones among them) become the active set, in their order;
 *   3. the join pods (whose DaemonSet guard joins) are scheduled in pod order, committed with Reserve;
 *   4. the evicted pods are scheduled in pod order, committed with Reserve;
 *   5. apply: the joined nodes become present, the drained present nodes retired, and the vanished pods and the pending DaemonSet
 *      pods of the drained nodes do not exist (-3).  Without
 *      apply the base is restored.
 */
#include "rolling_oracle.c"

/* One wave from the base the oracle holds (placement / slots / state: its placement, slot words and node states 0 absent, 1 present,
 * 2 retired).  counts[7]: evicted, placed, unscheduled, blocked, vanished, join pods, unscheduled join pods; per evicted pod in pod
 * order out_evicted, out_node, out_score, out_slots; out_blocked; per join pod out_join, out_jnode, out_jscore, out_jslots; failures in
 * list order (join pods, then evicted pods) out_fail_counts [n][SIMON_N_FAIL_CODES], out_fail_pod; sums[2]: requested mcpu and memory
 * over the remaining nodes.  apply (SIMON_ERR_INVALID for a wave with a blocked or unscheduled pod): the oracle, placement, slots and
 * state become the next base. */
int simon_oracle_replace(simon_oracle *o, int32_t *placement, uint32_t *slots, uint8_t *state, const uint32_t *remain, uint32_t n_remain,
                         const uint32_t *join, uint32_t n_join, int apply, uint32_t *counts, uint32_t *out_evicted, int32_t *out_node,
                         int64_t *out_score, uint32_t *out_slots, uint32_t *out_blocked, uint32_t *out_join, int32_t *out_jnode,
                         int64_t *out_jscore, uint32_t *out_jslots, uint32_t *out_fail_counts, uint32_t *out_fail_pod, int64_t *sums) {
    const uint32_t P = o->p.n_pods, N = o->N;
    saved_state sv;
    state_io(o, &sv, 1);
    uint8_t *rm = (uint8_t *)malloc(N + 1), *jn = (uint8_t *)calloc(N + 1, 1);
    memset(rm, 1, N + 1);
    for (uint32_t i = 0; i < n_remain; i++) rm[remain[i]] = 0;
    for (uint32_t i = 0; i < n_join; i++) jn[join[i]] = 1;
    uint32_t *vanished = (uint32_t *)malloc(4ull * (P + 1));
    uint32_t n_van = 0, n_ev = 0, n_fail = 0, n_j = 0;
    memset(counts, 0, 7 * sizeof(uint32_t));
    for (uint32_t q = 0; q < P; q++) {
        const int32_t g = placement[q];
        if (g < 0 || !rm[g]) continue;
        const uint32_t cls = (uint32_t)o->p.pod_class[q];
        const int64_t *cw = CW(o, cls);
        uncommit(o, cw, (uint32_t)g);
        if (cw[SCW_GPU_MEM] > 0)
            for (int d = 0; d < SIMON_MAX_GPU_DEV; d++) o->gpu_used[(uint64_t)d * N + g] -= (int64_t)((slots[q] >> (4 * d)) & 15u) * cw[SCW_GPU_MEM];
        const int64_t guard = guard_of(o, cw, q);
        if (guard >= 0 && rm[guard]) vanished[n_van++] = q;
        else if (o->p.pod_fixed_node[q] >= 0 || class_local(o, cls)) out_blocked[counts[3]++] = q;
        else out_evicted[n_ev++] = q;
    }
    counts[4] = n_van;
    simon_oracle_set_active(o, remain, n_remain);
    int rc = SIMON_OK;
    for (int pass = 0; pass < 2 && rc == SIMON_OK; pass++) {
        const uint32_t n_list = pass == 0 ? P : n_ev;
        for (uint32_t x = 0; x < n_list; x++) {
            uint32_t q;
            if (pass == 0) {
                q = x;
                const int64_t guard = guard_of(o, CW(o, (uint32_t)o->p.pod_class[q]), q);
                if (guard < 0 || !jn[guard]) continue;
            } else {
                q = out_evicted[x];
            }
            const uint32_t cls = (uint32_t)o->p.pod_class[q];
            o->cur_pin = o->p.pod_pin_node ? o->p.pod_pin_node[q] : -1;
            uint32_t hist[SIMON_N_FAIL_CODES];
            int64_t score = 0;
            const int64_t n = schedule_one(o, cls, &score, hist);
            if (n == -2) { rc = SIMON_ERR_LIMIT; break; }
            uint32_t pack = 0;
            if (n >= 0) pack = commit(o, CW(o, cls), (uint32_t)n, 1);
            else {
                memcpy(out_fail_counts + (uint64_t)n_fail * SIMON_N_FAIL_CODES, hist, sizeof(hist));
                out_fail_pod[n_fail++] = q;
                score = 0;
            }
            if (pass == 0) {
                out_join[n_j] = q; out_jnode[n_j] = (int32_t)n; out_jscore[n_j] = score; out_jslots[n_j] = pack;
                n_j++;
                if (n < 0) counts[6]++;
            } else {
                out_node[x] = (int32_t)n; out_score[x] = score; out_slots[x] = pack;
                if (n >= 0) counts[1]++;
                else counts[2]++;
            }
        }
    }
    counts[0] = n_ev;
    counts[5] = n_j;
    sums[0] = sums[1] = 0;
    for (uint32_t i = 0; i < n_remain; i++) { sums[0] += o->req_mcpu[remain[i]]; sums[1] += o->req_mem[remain[i]]; }
    if (rc == SIMON_OK && apply && (n_fail || counts[3])) rc = SIMON_ERR_INVALID;
    if (rc == SIMON_OK && apply) {
        for (uint32_t j = 0; j < n_ev; j++) { placement[out_evicted[j]] = out_node[j]; slots[out_evicted[j]] = out_slots[j]; }
        for (uint32_t j = 0; j < n_j; j++) { placement[out_join[j]] = out_jnode[j]; slots[out_join[j]] = out_jslots[j]; }
        for (uint32_t j = 0; j < n_van; j++) { placement[vanished[j]] = -3; slots[vanished[j]] = 0; }
        /* the pending DaemonSet pods of the retiring nodes stop existing as well */
        for (uint32_t q = 0; q < P; q++) {
            const int64_t guard = guard_of(o, CW(o, (uint32_t)o->p.pod_class[q]), q);
            if (guard >= 0 && rm[guard] && state[guard] == 1 && placement[q] == -1) { placement[q] = -3; slots[q] = 0; }
        }
        for (uint32_t g = 0; g < N; g++) {
            if (jn[g]) state[g] = 1;
            else if (rm[g] && state[g] == 1) state[g] = 2;
        }
    } else {
        state_io(o, &sv, 0);
    }
    free(sv.i64); free(sv.i32); free(sv.slots); free(rm); free(jn); free(vanished);
    return rc;
}
