/*
 * rolling_oracle.c — CPU checker of rolling-maintenance waves (simon_wave_run / simon_wave_commit, include/simon_gpu.h).  TEST
 * INFRASTRUCTURE ONLY, like the oracle it is built on.
 *
 * The move-scope checker (and through it the CPU oracle) is compiled into this library unchanged, for uncommit().  The oracle's state
 * is the wave base.  One wave is applied with the oracle's own primitives, by a different mechanism from the engine's (base copied into
 * a slot, counters of the removed pods taken out, state copied back, nodes reset):
 *   1. every pod of a removed node is uncommitted there in pod order, its device memory released as its slot word states, and
 *      classified as simon_drain_run classifies it (vanished, blocked, evicted);
 *   2. the remaining nodes become the active set, in their order;
 *   3. the evicted pods are scheduled in pod order, committed with Reserve;
 *   4. apply: all nodes active again, in index order, and the vanished pods (the DaemonSet pods of the returned nodes) committed on
 *      their nodes in pod order, with Reserve for the ones that went through the scheduler.  Without apply the base is restored.
 */
#include "moves_scope_oracle.c"

typedef struct {
    int64_t *i64;
    int32_t *i32;
    uint32_t *slots;
    size_t n64, n32;
} saved_state;

/* the oracle's dynamic state, in one buffer per type */
static void state_io(simon_oracle *o, saved_state *s, int save) {
    const size_t N = o->N, K = o->s.n_scalars, nc = o->p.n_counters, cw = o->cnt_off[nc], P = o->p.n_pods;
    int64_t *cols64[5] = {o->req_mcpu, o->req_mem, o->req_eph, o->nz_mcpu, o->nz_mem};
    if (save) {
        s->n64 = 5 * N + K * N + SIMON_MAX_GPU_DEV * N + nc;
        s->n32 = N + cw;
        s->i64 = (int64_t *)malloc(8 * (s->n64 + 1));
        s->i32 = (int32_t *)malloc(4 * (s->n32 + 1));
        s->slots = (uint32_t *)malloc(4 * (P + 1));
    }
#define IO(dst, src, bytes) do { if (save) memcpy(dst, src, bytes); else memcpy(src, dst, bytes); } while (0)
    int64_t *a = s->i64;
    for (int c = 0; c < 5; c++, a += N) IO(a, cols64[c], 8 * N);
    IO(a, o->req_scalar, 8 * K * N); a += K * N;
    IO(a, o->gpu_used, 8 * SIMON_MAX_GPU_DEV * N); a += SIMON_MAX_GPU_DEV * N;
    IO(a, o->cnt_total, 8 * nc);
    IO(s->i32, o->num_pods, 4 * N);
    IO(s->i32 + N, o->cnt, 4 * cw);
    IO(s->slots, o->gpu_slots, 4 * P);
#undef IO
}

static int64_t guard_of(const simon_oracle *o, const int64_t *cw, uint32_t q) {
    const int64_t g = cw[SCW_GUARD_NODE];
    return g == -3 ? (o->p.pod_pin_node ? o->p.pod_pin_node[q] : -1) : g;
}

/* One wave from the base the oracle holds, whose placement is placement / slots.  counts[5]: evicted, placed, unscheduled, blocked,
 * vanished; per evicted pod in pod order out_evicted, out_node (-1 unschedulable), out_score, out_slots; out_blocked; failures in
 * order out_fail_counts [n][SIMON_N_FAIL_CODES], out_fail_pod; sums[2]: requested mcpu and memory over the remaining nodes after the
 * placement.  apply (only for a wave with no blocked or unscheduled pod, else
 * SIMON_ERR_INVALID): the oracle, placement and slots become the next base; else they are left as they were. */
int simon_oracle_wave(simon_oracle *o, int32_t *placement, uint32_t *slots, const uint32_t *remain, uint32_t n_remain, int apply,
                      uint32_t *counts, uint32_t *out_evicted, int32_t *out_node, int64_t *out_score, uint32_t *out_slots,
                      uint32_t *out_blocked, uint32_t *out_fail_counts, uint32_t *out_fail_pod, int64_t *sums) {
    const uint32_t P = o->p.n_pods, N = o->N;
    saved_state sv;
    state_io(o, &sv, 1);
    uint8_t *rm = (uint8_t *)malloc(N + 1);
    memset(rm, 1, N + 1);
    for (uint32_t i = 0; i < n_remain; i++) rm[remain[i]] = 0;
    uint32_t *vanished = (uint32_t *)malloc(4ull * (P + 1));
    uint32_t n_van = 0, n_ev = 0, n_fail = 0;
    memset(counts, 0, 5 * sizeof(uint32_t));
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
    for (uint32_t j = 0; j < n_ev; j++) {
        const uint32_t q = out_evicted[j], cls = (uint32_t)o->p.pod_class[q];
        o->cur_pin = o->p.pod_pin_node ? o->p.pod_pin_node[q] : -1;
        uint32_t hist[SIMON_N_FAIL_CODES];
        int64_t score = 0;
        const int64_t n = schedule_one(o, cls, &score, hist);
        if (n == -2) { rc = SIMON_ERR_LIMIT; break; }
        out_node[j] = (int32_t)n;
        out_slots[j] = 0;
        if (n >= 0) {
            out_slots[j] = commit(o, CW(o, cls), (uint32_t)n, 1);
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
    sums[0] = sums[1] = 0;
    for (uint32_t i = 0; i < n_remain; i++) { sums[0] += o->req_mcpu[remain[i]]; sums[1] += o->req_mem[remain[i]]; }
    uint32_t *all = (uint32_t *)malloc(4ull * (N + 1));
    for (uint32_t g = 0; g < N; g++) all[g] = g;
    simon_oracle_set_active(o, all, N);
    if (rc == SIMON_OK && apply && (n_fail || counts[3])) rc = SIMON_ERR_INVALID;
    if (rc == SIMON_OK && apply) {
        for (uint32_t j = 0; j < n_ev; j++) { placement[out_evicted[j]] = out_node[j]; slots[out_evicted[j]] = out_slots[j]; }
        for (uint32_t j = 0; j < n_van; j++) {
            const uint32_t q = vanished[j];
            const int reserve = o->p.pod_fixed_node[q] == -1;
            o->cur_pin = o->p.pod_pin_node ? o->p.pod_pin_node[q] : -1;
            const uint32_t pack = commit(o, CW(o, (uint32_t)o->p.pod_class[q]), (uint32_t)placement[q], reserve);
            slots[q] = reserve ? pack : 0;
        }
    } else {
        state_io(o, &sv, 0);
    }
    free(sv.i64); free(sv.i32); free(sv.slots); free(rm); free(vanished); free(all);
    return rc;
}
