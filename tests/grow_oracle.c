/*
 * grow_oracle.c — CPU checker of grow batches (simon_grow_run, include/simon_gpu.h).  TEST INFRASTRUCTURE ONLY, like the oracle it
 * is built on.
 *
 * The CPU oracle (oracle/simon_oracle.c) is compiled into this library unchanged.  One scenario is evaluated by a different mechanism
 * from the engine's (live state rebuilt once and copied into every scenario): the state is built up from empty in the oracle.
 *   1. reset; 2. the scenario's nodes become the active set, in their order;
 *   3. every placed prefix pod is committed on its node in pod order - Reserve (GPU-share devices) and, with storage, Open-Local's Bind
 *      for the pods that went through the scheduler, neither for pre-bound ones, as simon_oracle_schedule does;
 *   4. simon_oracle_schedule places the tail [n_prefix, n_pods), where a pod whose guard node is inactive does not exist (-3).
 */
#include "../oracle/simon_oracle.c"

/* Scenario `nodes` on the live placement placed[n_prefix]: per tail pod out_node / out_score / out_slots (4 bits per device); the
 * failures of the tail in order (out_fail_counts [n][SIMON_N_FAIL_CODES], out_fail_pod, *n_fail).  The oracle's state afterwards is the
 * scenario's end state (simon_oracle_state / _state_ext / _storage_state). */
int simon_oracle_grow(simon_oracle *o, const int32_t *placed, uint32_t n_prefix, const uint32_t *nodes, uint32_t n_nodes, int32_t *out_node,
                      int64_t *out_score, uint32_t *out_slots, uint32_t *out_fail_counts, uint32_t *out_fail_pod, uint32_t *n_fail) {
    const uint32_t P = o->p.n_pods, N = o->N;
    if (n_prefix > P) return SIMON_ERR_INVALID;
    simon_oracle_reset(o);
    simon_oracle_set_active(o, nodes, n_nodes);
    for (uint32_t q = 0; q < n_prefix; q++) {
        const int32_t g = placed[q];
        if (g < 0) continue;
        if ((uint32_t)g >= N || !o->active[g]) return SIMON_ERR_INVALID;
        const int32_t fixed = o->p.pod_fixed_node[q];
        o->cur_pin = o->p.pod_pin_node ? o->p.pod_pin_node[q] : -1;
        const uint32_t pack = commit(o, CW(o, (uint32_t)o->p.pod_class[q]), (uint32_t)g, fixed == -1);
        o->gpu_slots[q] = fixed == -1 ? pack : 0;
    }
    const uint32_t T = P - n_prefix;
    const int rc = simon_oracle_schedule(o, n_prefix, T, out_node, out_score, out_fail_counts, out_fail_pod, T, n_fail);
    if (rc) return rc;
    return simon_oracle_gpu_slots(o, n_prefix, T, out_slots);
}
