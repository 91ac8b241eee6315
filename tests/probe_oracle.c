/*
 * probe_oracle.c — CPU checker of headroom probes (simon_probe_run, include/simon_gpu.h).  TEST INFRASTRUCTURE ONLY, like the oracle
 * it is built on.
 *
 * The CPU oracle (oracle/simon_oracle.c) is compiled into this library unchanged.  One probe is evaluated by a different mechanism
 * from the engine's (live state rebuilt once and copied into every scenario): the state is built up from empty in the oracle.
 *   1. reset;
 *   2. every placed pod is committed on its node in pod order - Reserve (GPU-share devices) and, with storage, Open-Local's Bind for
 *      the pods that went through the scheduler, neither for pre-bound ones, as simon_oracle_schedule does;
 *   3. replicas of the probe pod's class are scheduled (schedule_one) and committed one at a time until one fails or max_replicas.
 */
#include "../oracle/simon_oracle.c"

/* Probe (pod, max_replicas) on the live placement `placed`: *n_placed replicas placed; per replica out_node, out_score, out_slots
 * (4 bits per device); out_fail_counts [SIMON_N_FAIL_CODES]: the histogram of the replica that failed (zeros if none did).  The
 * oracle's state afterwards is the probe's end state (simon_oracle_state / _state_ext / _storage_state). */
int simon_oracle_probe(simon_oracle *o, const int32_t *placed, uint32_t pod, uint32_t max_replicas, uint32_t *n_placed, int32_t *out_node,
                       int64_t *out_score, uint32_t *out_slots, uint32_t *out_fail_counts) {
    const uint32_t P = o->p.n_pods, N = o->N;
    if (pod >= P) return SIMON_ERR_INVALID;
    simon_oracle_reset(o);
    for (uint32_t q = 0; q < P; q++) {
        const int32_t g = placed[q];
        if (g < 0) continue;
        if ((uint32_t)g >= N) return SIMON_ERR_INVALID;
        const int32_t fixed = o->p.pod_fixed_node[q];
        o->cur_pin = o->p.pod_pin_node ? o->p.pod_pin_node[q] : -1;
        const uint32_t pack = commit(o, CW(o, (uint32_t)o->p.pod_class[q]), (uint32_t)g, fixed == -1);
        o->gpu_slots[q] = fixed == -1 ? pack : 0;
    }
    const uint32_t cls = (uint32_t)o->p.pod_class[pod];
    const int64_t *cw = CW(o, cls);
    memset(out_fail_counts, 0, SIMON_N_FAIL_CODES * sizeof(uint32_t));
    *n_placed = 0;
    o->cur_pin = o->p.pod_pin_node ? o->p.pod_pin_node[pod] : -1;
    for (uint32_t k = 0; k < max_replicas; k++) {
        uint32_t hist[SIMON_N_FAIL_CODES];
        int64_t score = 0;
        const int64_t n = schedule_one(o, cls, &score, hist);
        if (n == -2) return SIMON_ERR_LIMIT;
        if (n < 0) {
            memcpy(out_fail_counts, hist, sizeof(hist));
            break;
        }
        out_node[k] = (int32_t)n;
        out_score[k] = score;
        out_slots[k] = commit(o, cw, (uint32_t)n, 1);
        (*n_placed)++;
    }
    return SIMON_OK;
}
