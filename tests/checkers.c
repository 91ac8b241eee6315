/*
 * checkers.c — the CPU checkers of the device features (include/simon_gpu.h), one library: build/libsimon_checkers.so.
 * TEST INFRASTRUCTURE ONLY, like the oracle it is built on.
 *
 * The CPU oracle (oracle/simon_oracle.c) is compiled into this library unchanged, so that every checker evaluates pods with the
 * oracle's own scheduling-cycle stages and its own commit(), rather than with a third restatement of the filters.  Below the oracle
 * come the primitives the checkers share, then one section per checker.  Each checker reaches the engine's answer by a mechanism of
 * its own, which its section's comment describes.
 */
#include "../oracle/simon_oracle.c"

/* ---- shared primitives ---- */

/* the inverse of commit(o, cw, n, 0) */
static void uncommit(simon_oracle *o, const int64_t *cw, uint32_t n) {
    const uint32_t N = o->N;
    o->req_mcpu[n] -= cw[SCW_REQ_MCPU]; o->req_mem[n] -= cw[SCW_REQ_MEM]; o->req_eph[n] -= cw[SCW_REQ_EPH];
    o->nz_mcpu[n] -= cw[SCW_NZ_MCPU]; o->nz_mem[n] -= cw[SCW_NZ_MEM];
    o->num_pods[n] -= 1;
    const int64_t *sc = cw + cw[SCW_OFF_SCALARS];
    for (uint32_t k = 0; k < o->s.n_scalars; k++) o->req_scalar[(uint64_t)k * N + n] -= sc[k];
    const int64_t *inc = cw + cw[SCW_OFF_INC];
    for (int64_t i = 0; i < cw[SCW_N_INC]; i++) {
        int64_t k = inc[3 * i], t = inc[3 * i + 1], sig = inc[3 * i + 2];
        int32_t d = dom_of(o, t, n);
        if (sig >= 0) continue;
        if (d >= 0) { o->cnt[o->cnt_off[k] + (uint32_t)d] -= 1; o->cnt_total[k] -= 1; }
    }
}

/* Take pod q off its node n: uncommit() there, then release its GPU-share device memory as its slot word `slot` states. */
static void take_off(simon_oracle *o, uint32_t q, uint32_t n, uint32_t slot) {
    const int64_t *cw = CW(o, (uint32_t)o->p.pod_class[q]);
    uncommit(o, cw, n);
    if (cw[SCW_GPU_MEM] > 0)
        for (int d = 0; d < SIMON_MAX_GPU_DEV; d++) o->gpu_used[(uint64_t)d * o->N + n] -= (int64_t)((slot >> (4 * d)) & 15u) * cw[SCW_GPU_MEM];
}

/* Commit every placed pod q < n_pods of the live placement `placed` on its node in pod order - Reserve (GPU-share devices) and, with
 * storage, Open-Local's Bind for the pods that went through the scheduler, neither for pre-bound ones, as simon_oracle_schedule
 * does.  slots[q] gets the pod's slot word.  A pod on a node outside the active set is SIMON_ERR_INVALID, or left out with
 * active_only. */
static int commit_live(simon_oracle *o, const int32_t *placed, uint32_t n_pods, int active_only, uint32_t *slots) {
    for (uint32_t q = 0; q < n_pods; q++) {
        const int32_t g = placed[q];
        if (g < 0) continue;
        if ((uint32_t)g >= o->N) return SIMON_ERR_INVALID;
        if (!o->active[g]) {
            if (active_only) continue;
            return SIMON_ERR_INVALID;
        }
        const int32_t fixed = o->p.pod_fixed_node[q];
        o->cur_pin = o->p.pod_pin_node ? o->p.pod_pin_node[q] : -1;
        const uint32_t pack = commit(o, CW(o, (uint32_t)o->p.pod_class[q]), (uint32_t)g, fixed == -1);
        slots[q] = fixed == -1 ? pack : 0;
    }
    return SIMON_OK;
}

/* the node whose presence pod q's existence depends on (a DaemonSet pod's), -1: none */
static int64_t guard_of(const simon_oracle *o, uint32_t q) {
    const int64_t g = CW(o, (uint32_t)o->p.pod_class[q])[SCW_GUARD_NODE];
    return g == -3 ? (o->p.pod_pin_node ? o->p.pod_pin_node[q] : -1) : g;
}

/* A pod of a removed node, with the remaining nodes active, as simon_drain_run classifies it: vanished (a DaemonSet pod of a removed
 * node), blocked (bound by spec.nodeName, or `local`: of a class with Open-Local volumes) or evicted. */
enum { POD_VANISHED, POD_BLOCKED, POD_EVICTED };
static int removed_pod_kind(const simon_oracle *o, uint32_t q, int local) {
    const int64_t guard = guard_of(o, q);
    if (guard >= 0 && !o->active[guard]) return POD_VANISHED;
    if (o->p.pod_fixed_node[q] >= 0 || local) return POD_BLOCKED;
    return POD_EVICTED;
}

/* Schedule the pods list[0, n) in order on the active nodes, each one that fits committed with Reserve: per pod out_node (-1
 * unschedulable), out_score (0 when unschedulable), out_slots, and pod_slots[q] (may be NULL) for the placed ones; each failure appended
 * to out_fail_counts [.][SIMON_N_FAIL_CODES] / out_fail_pod at *n_fail.  *n_placed counts the placed pods. */
static int schedule_list(simon_oracle *o, const uint32_t *list, uint32_t n, int32_t *out_node, int64_t *out_score, uint32_t *out_slots,
                         uint32_t *pod_slots, uint32_t *out_fail_counts, uint32_t *out_fail_pod, uint32_t *n_fail, uint32_t *n_placed) {
    for (uint32_t j = 0; j < n; j++) {
        const uint32_t q = list[j], cls = (uint32_t)o->p.pod_class[q];
        o->cur_pin = o->p.pod_pin_node ? o->p.pod_pin_node[q] : -1;
        uint32_t hist[SIMON_N_FAIL_CODES];
        int64_t score = 0;
        const int64_t g = schedule_one(o, cls, &score, hist);
        if (g == -2) return SIMON_ERR_LIMIT;
        out_node[j] = (int32_t)g;
        out_slots[j] = 0;
        if (g >= 0) {
            out_slots[j] = commit(o, CW(o, cls), (uint32_t)g, 1);
            if (pod_slots) pod_slots[q] = out_slots[j];
            (*n_placed)++;
        } else {
            memcpy(out_fail_counts + (uint64_t)*n_fail * SIMON_N_FAIL_CODES, hist, sizeof(hist));
            out_fail_pod[(*n_fail)++] = q;
            score = 0;
        }
        out_score[j] = score;
    }
    return SIMON_OK;
}

/* ---- explained placement decisions (simon_explain_set) ----
 * The oracle's per-node detail of the last scheduled pod (simon_oracle_last_detail: filter stage and the ten score words) names the
 * failing stage of each node, not every reason its verdict carries; this exports those reasons (the bitmask of simon_fail_code the
 * oracle's filter stage builds for each node). */

/* The filter verdict of every node for the last pod that reached the scheduler: 0 feasible, else a bitmask of simon_fail_code. */
void simon_oracle_last_reasons(simon_oracle *o, uint32_t *out) { memcpy(out, o->reasons, 4ull * o->N); }

/* ---- node drains (simon_drain_run) ----
 * One drain is evaluated by a different mechanism from the engine's (live state copied into every scenario, then the removed pods
 * taken out of the counters): the state is built up from empty on the remaining nodes only.
 *   1. reset; 2. the remaining nodes become the active set, in their order;
 *   3. every placed pod that sits on a remaining node is committed there in pod order - Reserve (GPU-share devices) for the pods
 *      that went through the scheduler, none for pre-bound ones (commit_live);
 *   4. the pods of removed nodes are classified (removed_pod_kind: vanished, blocked, evicted) and each evicted pod is scheduled in
 *      pod order. */

/* counts[5]: evicted, placed, unscheduled, blocked, vanished.  Per evicted pod in pod order (arrays of n_pods entries suffice):
 * out_evicted (pod index), out_node (-1 unschedulable), out_score, out_slots (4 bits per device); out_blocked: blocked pods in
 * pod order; failures in order: out_fail_counts [n][SIMON_N_FAIL_CODES], out_fail_pod.  class_local: NULL, or per class 1 = Open-Local
 * volumes.  The oracle's state afterwards is the drain's end state (simon_oracle_state / _state_ext). */
int simon_oracle_drain(simon_oracle *o, const int32_t *placed, const uint32_t *remain, uint32_t n_remain, const uint8_t *class_local,
                       uint32_t *counts, uint32_t *out_evicted, int32_t *out_node, int64_t *out_score, uint32_t *out_slots,
                       uint32_t *out_blocked, uint32_t *out_fail_counts, uint32_t *out_fail_pod) {
    const uint32_t P = o->p.n_pods;
    simon_oracle_reset(o);
    simon_oracle_set_active(o, remain, n_remain);
    memset(counts, 0, 5 * sizeof(uint32_t));
    const int rc = commit_live(o, placed, P, 1, o->gpu_slots);
    if (rc) return rc;
    for (uint32_t q = 0; q < P; q++) {
        if (placed[q] < 0 || o->active[placed[q]]) continue;
        const uint32_t cls = (uint32_t)o->p.pod_class[q];
        const int kind = removed_pod_kind(o, q, class_local && class_local[cls]);
        if (kind == POD_VANISHED) counts[4]++;
        else if (kind == POD_BLOCKED) out_blocked[counts[3]++] = q;
        else out_evicted[counts[0]++] = q;
    }
    return schedule_list(o, out_evicted, counts[0], out_node, out_score, out_slots, o->gpu_slots, out_fail_counts, out_fail_pod,
                         &counts[2], &counts[1]);
}

/* ---- grow batches (simon_grow_run) ----
 * One scenario is evaluated by a different mechanism from the engine's (live state rebuilt once and copied into every scenario): the
 * state is built up from empty in the oracle.
 *   1. reset; 2. the scenario's nodes become the active set, in their order;
 *   3. every placed prefix pod is committed on its node in pod order - Reserve (GPU-share devices) and, with storage, Open-Local's Bind
 *      for the pods that went through the scheduler, neither for pre-bound ones (commit_live);
 *   4. simon_oracle_schedule places the tail [n_prefix, n_pods), where a pod whose guard node is inactive does not exist (-3). */

/* Scenario `nodes` on the live placement placed[n_prefix]: per tail pod out_node / out_score / out_slots (4 bits per device); the
 * failures of the tail in order (out_fail_counts [n][SIMON_N_FAIL_CODES], out_fail_pod, *n_fail).  The oracle's state afterwards is the
 * scenario's end state (simon_oracle_state / _state_ext / _storage_state). */
int simon_oracle_grow(simon_oracle *o, const int32_t *placed, uint32_t n_prefix, const uint32_t *nodes, uint32_t n_nodes, int32_t *out_node,
                      int64_t *out_score, uint32_t *out_slots, uint32_t *out_fail_counts, uint32_t *out_fail_pod, uint32_t *n_fail) {
    const uint32_t P = o->p.n_pods;
    if (n_prefix > P) return SIMON_ERR_INVALID;
    simon_oracle_reset(o);
    simon_oracle_set_active(o, nodes, n_nodes);
    int rc = commit_live(o, placed, n_prefix, 0, o->gpu_slots);
    if (rc) return rc;
    const uint32_t T = P - n_prefix;
    rc = simon_oracle_schedule(o, n_prefix, T, out_node, out_score, out_fail_counts, out_fail_pod, T, n_fail);
    if (rc) return rc;
    return simon_oracle_gpu_slots(o, n_prefix, T, out_slots);
}

/* ---- headroom probes (simon_probe_run) ----
 * One probe is evaluated by a different mechanism from the engine's (live state rebuilt once and copied into every scenario): the
 * state is built up from empty in the oracle.
 *   1. reset; every node active, in index order, as the engine's probes run;
 *   2. every placed pod is committed on its node in pod order - Reserve (GPU-share devices) and, with storage, Open-Local's Bind for
 *      the pods that went through the scheduler, neither for pre-bound ones (commit_live);
 *   3. replicas of the probe pod's class are scheduled (schedule_one) and committed one at a time until one fails or max_replicas. */

/* Probe (pod, max_replicas) on the live placement `placed`: *n_placed replicas placed; per replica out_node, out_score, out_slots
 * (4 bits per device); out_fail_counts [SIMON_N_FAIL_CODES]: the histogram of the replica that failed (zeros if none did).  The
 * oracle's state afterwards is the probe's end state (simon_oracle_state / _state_ext / _storage_state). */
int simon_oracle_probe(simon_oracle *o, const int32_t *placed, uint32_t pod, uint32_t max_replicas, uint32_t *n_placed, int32_t *out_node,
                       int64_t *out_score, uint32_t *out_slots, uint32_t *out_fail_counts) {
    const uint32_t P = o->p.n_pods;
    if (pod >= P) return SIMON_ERR_INVALID;
    simon_oracle_reset(o);
    simon_oracle_set_active(o, NULL, 0);
    const int rc = commit_live(o, placed, P, 0, o->gpu_slots);
    if (rc) return rc;
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

/* ---- trace replays (simon_trace_run) ----
 * One scenario is replayed one event at a time with the oracle's own primitives, by a different mechanism from the engine's (runs of
 * creates in one launch, runs of deletes in another, state rebuilt once and copied):
 *   1. reset; the scenario's nodes become the active set, in their order; every placed prefix pod is committed on its node in pod order
 *      (commit_live, as the grow checker does);
 *   2. a create is simon_oracle_schedule of that one pod on the active nodes;
 *   3. a delete of a pod that holds a node is take_off() there (as the migration-plan checker does); a pod that holds no node leaves
 *      nothing;
 *   4. after every event, the sums the samples report over the active nodes. */

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
    if (commit_live(o, placed, n_prefix, 0, slot)) { free(where); free(slot); return SIMON_ERR_INVALID; }
    for (uint32_t q = 0; q < P; q++) {
        where[q] = q < n_prefix && placed[q] >= 0 ? placed[q] : -1;
        running += where[q] >= 0;
    }
    for (uint32_t e = 0; e < n_events; e++) {
        const uint32_t op = events[2 * e], q = events[2 * e + 1];
        if (q >= P) { free(where); free(slot); return SIMON_ERR_INVALID; }
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
                take_off(o, q, (uint32_t)g, slot[q]);
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

/* ---- the move scope (simon_moves_set_scope; the scoped instantiation of open-simulator_b200/csrc/simon_moves.cu) ----
 * A move of a class the scope admits is evaluated by the oracle's own scheduling-cycle stages:
 *   take p off its node a (uncommit: requests, non-zero requests, pod count, scalars and its unconditional counter increments), run
 *   ST_SEL / ST_HARDREG / the hard minimum / ST_FILTER for p's class on the target b, then commit p back on a.  The first failing
 *   filter's reasons are the code; the gain is that of simon_oracle_moves_score.
 * Every other move, and every move under scope 0, is simon_oracle_moves_score's own answer. */

/* per class, for the duration of one call: node selection verdicts over all nodes, registered domains of each hard constraint
 * (static), and the hard minimum with p removed, per source domain of p's count (slot max_dom: p holds no count) */
typedef struct {
    uint8_t *sel;
    uint8_t *reg;        /* [n_hard][max_dom] */
    int64_t *min_at;     /* [n_hard][max_dom + 1], INT64_MIN: not computed yet */
} scope_class;

static void ctx_init(simon_oracle *o, sched_ctx *c, const int64_t *cw) {
    memset(c, 0, sizeof(*c));
    c->o = o; c->cw = cw;
    c->N = o->N; c->NA = o->n_active; c->K = o->s.n_scalars; c->WT = o->s.n_taint_words;
    c->flags = (uint32_t)cw[SCW_FLAGS];
    c->tol = cw + cw[SCW_OFF_TOL];
    c->sc_req = cw + cw[SCW_OFF_SCALARS];
    c->n_hard = cw[SCW_N_PTS_HARD]; c->n_soft = cw[SCW_N_PTS_SOFT];
    c->hard = cw + cw[SCW_OFF_PTS_HARD]; c->soft = cw + cw[SCW_OFF_PTS_SOFT];
    c->n_aff = cw[SCW_N_IPA_AFF]; c->n_anti = cw[SCW_N_IPA_ANTI]; c->n_exist = cw[SCW_N_IPA_EXIST];
    c->aff = cw + cw[SCW_OFF_IPA_AFF]; c->anti = cw + cw[SCW_OFF_IPA_ANTI]; c->exist = cw + cw[SCW_OFF_IPA_EXIST];
    c->n_isc = cw[SCW_N_IPA_SCORE]; c->isc = cw + cw[SCW_OFF_IPA_SCORE];
    c->n_ports = cw[SCW_N_PORTS]; c->ports = cw + cw[SCW_OFF_PORTS];
}

static scope_class *class_tables(simon_oracle *o, sched_ctx *c, scope_class *S) {
    if (S->sel) return S;
    const uint32_t N = o->N, md = o->max_dom;
    S->sel = (uint8_t *)malloc(N + 1);
    S->reg = (uint8_t *)calloc((uint64_t)(c->n_hard ? c->n_hard : 1) * md, 1);
    S->min_at = (int64_t *)malloc(8ull * (c->n_hard ? c->n_hard : 1) * (md + 1));
    for (uint64_t q = 0; q < (uint64_t)(c->n_hard ? c->n_hard : 1) * (md + 1); q++) S->min_at[q] = INT64_MIN;
    stage_run(c, 0, c->NA, 0);                        /* c->stage == ST_SEL: every node (the moves path has them all active) */
    memcpy(S->sel, o->sel_ok, N);
    c->stage = ST_HARDREG;
    for (int64_t j = 0; j < c->n_hard; j++) {
        c->j = (int)j;
        stage_run(c, 0, c->NA, 0);                    /* thread 0's table of constraint j */
        memcpy(S->reg + (uint64_t)j * md, o->t_flag + (uint64_t)j * md, o->s.topo_ndom[c->hard[4 * j + 1]]);
    }
    return S;
}

#define SCOPE_GPU 1u
#define SCOPE_HARD 2u

/* Scoped moves on the oracle's current state (see include/simon_gpu.h, simon_moves_set_scope).  class_local (NULL: none) flags the
 * classes with Open-Local volumes, which the engine never moves; without it, scope 0 returns exactly simon_oracle_moves_score.
 * out_gpu_slots (may be NULL): per move the target's device slots of a feasible GPU-share move (4 bits per device), else 0. */
int simon_oracle_moves_score_scoped(simon_oracle *o, uint32_t scope, uint32_t n_moves, const uint32_t *moves, const int32_t *placement,
                                    const uint8_t *class_local, int32_t *out_gain, uint32_t *out_code, uint32_t *out_gpu_slots) {
    if (scope & ~(SCOPE_GPU | SCOPE_HARD)) return SIMON_ERR_INVALID;
    if (o->n_active != o->N) return SIMON_ERR_STATE;
    int rc = simon_oracle_moves_score(o, n_moves, moves, placement, out_gain, out_code);
    if (rc) return rc;
    if (out_gpu_slots) memset(out_gpu_slots, 0, 4ull * n_moves);
    const uint32_t C = o->p.n_classes, md = o->max_dom;
    scope_class *tabs = (scope_class *)calloc(C ? C : 1, sizeof(scope_class));
    sched_ctx *c = (sched_ctx *)malloc(sizeof(sched_ctx));
    for (uint32_t m = 0; m < n_moves; m++) {
        const uint32_t pod = moves[2 * m], b = moves[2 * m + 1];
        const uint32_t cls = (uint32_t)o->p.pod_class[pod < o->p.n_pods ? pod : 0];
        const int64_t *cw = CW(o, cls);
        if (class_local && class_local[cls] && out_code[m] != SMV_BAD_INDEX && out_code[m] != SMV_NOT_PLACED && out_code[m] != SMV_NOOP) {
            out_code[m] = SMV_NOT_MOVABLE; out_gain[m] = 0;
            continue;
        }
        if (out_code[m] != SMV_NOT_MOVABLE || (cw[SCW_FLAGS] & SIMON_CLS_PINNED)) continue;
        const uint32_t need = (cw[SCW_GPU_MEM] > 0 ? SCOPE_GPU : 0u) | (cw[SCW_N_PTS_HARD] > 0 ? SCOPE_HARD : 0u);
        if (need & ~scope) continue;
        const uint32_t a = (uint32_t)placement[pod];
        ctx_init(o, c, cw);
        if (c->n_hard > 16) { rc = SIMON_ERR_LIMIT; break; }
        o->cur_pin = -1;
        c->stage = ST_SEL;
        scope_class *S = class_tables(o, c, &tabs[cls]);
        uncommit(o, cw, a);
        const int64_t *inc = cw + cw[SCW_OFF_INC];
        for (int64_t j = 0; j < c->n_hard; j++) {
            const int64_t k = c->hard[4 * j], t = c->hard[4 * j + 1];
            const int32_t da = dom_of(o, t, a);
            const uint32_t key = (da >= 0 && own_inc(o, inc, cw[SCW_N_INC], k, t, a, da)) ? (uint32_t)da : md;
            const uint8_t *reg = S->reg + (uint64_t)j * md;
            int64_t *mn = S->min_at + (uint64_t)j * (md + 1) + key;
            if (*mn == INT64_MIN) {                   /* schedule_one's minimum, on the state with p removed */
                *mn = INT32_MAX;
                for (uint32_t d = 0; d < o->s.topo_ndom[t]; d++)
                    if (reg[d] && cnt_at(o, k, (int32_t)d) < *mn) *mn = cnt_at(o, k, (int32_t)d);
            }
            c->hard_reg[j] = (uint8_t *)reg;
            c->hard_min[j] = *mn;
        }
        c->aff_total = 0;
        for (int64_t j = 0; j < c->n_aff; j++) c->aff_total += o->cnt_total[c->aff[2 * j]];
        o->sel_ok[b] = S->sel[b];
        uint32_t *order = o->order, one = b;
        o->order = &one;
        c->stage = ST_FILTER;
        stage_run(c, 0, 1, 0);
        o->order = order;
        const uint32_t code = o->code[b] ? o->reasons[b] : 0u;
        int32_t gain = 0;
        if (!code) {
            int64_t on_b = own_score(o->s.alloc_mcpu[b], o->s.alloc_mem[b], o->nz_mcpu[b], o->nz_mem[b], cw[SCW_SCORE_MCPU], cw[SCW_SCORE_MEM]);
            int64_t on_a = own_score(o->s.alloc_mcpu[a], o->s.alloc_mem[a], o->nz_mcpu[a], o->nz_mem[a], cw[SCW_SCORE_MCPU], cw[SCW_SCORE_MEM]);
            gain = (int32_t)(on_b - on_a);
            if (out_gpu_slots && cw[SCW_GPU_MEM] > 0) {
                int slots[64];
                const int ns = gpu_allocate(o, cw, b, slots);
                uint32_t pack = 0;
                for (int q = 0; q < ns && q < 64; q++)
                    if (((pack >> (4 * slots[q])) & 15u) < 15u) pack += 1u << (4 * slots[q]);
                out_gpu_slots[m] = pack;
            }
        }
        commit(o, cw, a, 0);
        out_code[m] = code;
        out_gain[m] = gain;
    }
    for (uint32_t q = 0; q < C; q++) { free(tabs[q].sel); free(tabs[q].reg); free(tabs[q].min_at); }
    free(tabs);
    free(c);
    return rc;
}

/* GPU-share device memory in use, [SIMON_MAX_GPU_DEV][N] */
void simon_oracle_gpu_used(simon_oracle *o, int64_t *out) {
    memcpy(out, o->gpu_used, 8ull * SIMON_MAX_GPU_DEV * o->N);
}

/* ---- migration plans (simon_moves_plan, with an optional PodDisruptionBudget table from simon_pdbs_upload) ----
 * Every step scores all candidate moves with simon_oracle_moves_score_scoped on the oracle's current state and placement, skips the
 * moves of pods that already moved, of excluded pods and of pods with a PDB at remaining 0, takes the best remaining feasible move by
 * (gain descending, move index ascending), and applies it with the oracle's own primitives: take_off() on the source, commit() with
 * Reserve on the target.
 *
 * The PDB table is the pod -> PDB CSR pdb_off / pdb_ids and each PDB's `allowed` on the live placement: remaining[j] starts at
 * allowed[j]; each applied step decrements remaining of every PDB of the moved pod.  *out_pdb_blocked counts the placed pods, other
 * than pinned, Open-Local and excluded ones, that a PDB at 0 keeps in place at the start.  With n_pdbs 0 the tables are not read
 * (they may be NULL) and no pod is kept in place by a PDB. */

/* out_steps: 6 words per step (move, pod, from, to, gain, gpu slots); placement and slots (the live slot words) are updated in place.
 * out_pdb_blocked may be NULL.  Returns 0, or 1 when Reserve on the target gives other slots than the scoring reported, or an error
 * of the scoring. */
int simon_oracle_moves_plan(simon_oracle *o, uint32_t scope, uint32_t n_moves, const uint32_t *moves, int32_t *placement, uint32_t *slots,
                            const uint8_t *class_local, uint32_t max_moves, int32_t min_gain, uint32_t n_pdbs, const uint32_t *pdb_off,
                            const uint32_t *pdb_ids, const int32_t *allowed, int32_t *out_steps, uint32_t *out_n, uint32_t *out_stop,
                            uint32_t *out_excluded, uint32_t *out_pdb_blocked) {
    const uint32_t P = o->p.n_pods;
    uint8_t *skip = (uint8_t *)calloc(P + 1, 1);
    int64_t *remaining = (int64_t *)malloc(8ull * (n_pdbs + 1));
    for (uint32_t j = 0; j < n_pdbs; j++) remaining[j] = allowed[j];
    uint32_t pdb_blocked = 0;
    int32_t *gain = (int32_t *)malloc(4ull * (n_moves + 1));
    uint32_t *code = (uint32_t *)malloc(4ull * (n_moves + 1)), *sl = (uint32_t *)malloc(4ull * (n_moves + 1));
    uint32_t excluded = 0, n = 0, stop = 0;
    int rc = 0;
    for (uint32_t q = 0; q < P; q++) {
        const uint32_t cls = (uint32_t)o->p.pod_class[q];
        const int64_t *cw = CW(o, cls);
        if (cw[SCW_GPU_MEM] <= 0 || (cw[SCW_FLAGS] & SIMON_CLS_PINNED) || (class_local && class_local[cls]) || placement[q] < 0) continue;
        for (int d = 0; d < SIMON_MAX_GPU_DEV; d++)
            if (((slots[q] >> (4 * d)) & 15u) == 15u) { skip[q] = 1; excluded++; break; }
    }
    for (uint32_t q = 0; n_pdbs && q < P; q++) {
        int out = 0;
        for (uint32_t k = pdb_off[q]; k < pdb_off[q + 1]; k++) out |= remaining[pdb_ids[k]] <= 0;
        if (!out) continue;
        const uint32_t cls = (uint32_t)o->p.pod_class[q];
        if (placement[q] >= 0 && !skip[q] && !(CW(o, cls)[SCW_FLAGS] & SIMON_CLS_PINNED) && !(class_local && class_local[cls])) pdb_blocked++;
        skip[q] = 1;
    }
    while (!stop) {
        rc = simon_oracle_moves_score_scoped(o, scope, n_moves, moves, placement, class_local, gain, code, sl);
        if (rc) break;
        int64_t best = -1;
        for (uint32_t m = 0; m < n_moves; m++)
            if (code[m] == 0 && !skip[moves[2 * m]] && (best < 0 || gain[m] > gain[best])) best = m;
        if (best < 0 || gain[best] < min_gain) { stop = SIMON_PLAN_STOP_NO_MOVE; break; }
        const uint32_t p = moves[2 * best], b = moves[2 * best + 1], a = (uint32_t)placement[p];
        const int64_t *cw = CW(o, o->p.pod_class[p]);
        take_off(o, p, a, slots[p]);
        const uint32_t pack = commit(o, cw, b, 1);
        if (cw[SCW_GPU_MEM] > 0) {
            if (pack != ((scope & SCOPE_GPU) ? sl[best] : 0u)) { rc = 1; break; }
            slots[p] = pack;
        }
        placement[p] = (int32_t)b;
        skip[p] = 1;
        for (uint32_t k = 0; n_pdbs && k < pdb_off[p + 1] - pdb_off[p]; k++) {
            const uint32_t j = pdb_ids[pdb_off[p] + k];
            if (--remaining[j] > 0) continue;
            for (uint32_t q = 0; q < P; q++)          /* the members of a PDB at 0 (a plain scan: this is a checker) */
                for (uint32_t u = pdb_off[q]; u < pdb_off[q + 1]; u++)
                    if (pdb_ids[u] == j) skip[q] = 1;
        }
        int32_t *s = out_steps + 6ull * n;
        s[0] = (int32_t)best; s[1] = (int32_t)p; s[2] = (int32_t)a; s[3] = (int32_t)b; s[4] = gain[best]; s[5] = (int32_t)pack;
        if (++n >= max_moves) stop = SIMON_PLAN_STOP_MAX_MOVES;
    }
    *out_n = n; *out_stop = stop; *out_excluded = excluded;
    if (out_pdb_blocked) *out_pdb_blocked = pdb_blocked;
    free(skip); free(gain); free(code); free(sl); free(remaining);
    return rc;
}

/* ---- rolling-maintenance and node-pool replacement waves (simon_wave_run / simon_wave_run_join / simon_wave_commit) ----
 * The oracle's state is the wave base.  One wave is applied with the oracle's own primitives, by a different mechanism from the
 * engine's (base copied into a slot, counters of the drained pods taken out, one pod list per scenario, state copied back):
 *   1. the remaining nodes (the joined ones among them) become the active set, in their order;
 *   2. every pod of a node missing from `remain` is take_off() there in pod order and classified (removed_pod_kind);
 *   3. the join pods (whose DaemonSet guard joins) are scheduled in pod order, committed with Reserve;
 *   4. the evicted pods are scheduled in pod order, committed with Reserve;
 *   5. apply without retire: the drained nodes come back, and the vanished pods (the DaemonSet pods of the returned nodes) are
 *      committed on their nodes in pod order, with Reserve for the ones that went through the scheduler;
 *      apply with retire: the joined nodes become present, the drained present nodes retired, and the vanished pods and the pending
 *      DaemonSet pods of the drained nodes do not exist (-3).
 *   Without apply the base is restored.  Every node is active again afterwards, in index order. */

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

/* One wave from the base the oracle holds (placement / slots / state: its placement, slot words and node states 0 absent, 1 present,
 * 2 retired; state NULL: every node present).  counts[7]: evicted, placed, unscheduled, blocked, vanished, join pods, unscheduled join
 * pods; per evicted pod in pod order out_evicted, out_node (-1 unschedulable), out_score, out_slots; out_blocked; per join pod
 * out_join, out_jnode, out_jscore, out_jslots; failures in list order (join pods, then evicted pods) out_fail_counts
 * [n][SIMON_N_FAIL_CODES], out_fail_pod; sums[2]: requested mcpu and memory over the remaining nodes after the placement.  apply: the
 * oracle, placement, slots and (with retire) state become the next base; SIMON_ERR_INVALID for a wave with a blocked or unscheduled
 * pod, for a wave that joined nodes without retire, and for retire without node states. */
int simon_oracle_wave(simon_oracle *o, int32_t *placement, uint32_t *slots, uint8_t *state, const uint32_t *remain, uint32_t n_remain,
                      const uint32_t *join, uint32_t n_join, int apply, int retire, uint32_t *counts, uint32_t *out_evicted,
                      int32_t *out_node, int64_t *out_score, uint32_t *out_slots, uint32_t *out_blocked, uint32_t *out_join,
                      int32_t *out_jnode, int64_t *out_jscore, uint32_t *out_jslots, uint32_t *out_fail_counts, uint32_t *out_fail_pod,
                      int64_t *sums) {
    const uint32_t P = o->p.n_pods, N = o->N;
    saved_state sv;
    state_io(o, &sv, 1);
    uint8_t *jn = (uint8_t *)calloc(N + 1, 1);
    for (uint32_t i = 0; i < n_join; i++) jn[join[i]] = 1;
    uint32_t *vanished = (uint32_t *)malloc(4ull * (P + 1));
    uint32_t n_van = 0, n_fail = 0;
    memset(counts, 0, 7 * sizeof(uint32_t));
    simon_oracle_set_active(o, remain, n_remain);
    for (uint32_t q = 0; q < P; q++) {
        const int32_t g = placement[q];
        if (g < 0 || o->active[g]) continue;
        take_off(o, q, (uint32_t)g, slots[q]);
        const int kind = removed_pod_kind(o, q, class_local(o, (uint32_t)o->p.pod_class[q]));
        if (kind == POD_VANISHED) vanished[n_van++] = q;
        else if (kind == POD_BLOCKED) out_blocked[counts[3]++] = q;
        else out_evicted[counts[0]++] = q;
    }
    counts[4] = n_van;
    for (uint32_t q = 0; q < P; q++) {
        const int64_t guard = guard_of(o, q);
        if (guard >= 0 && jn[guard]) out_join[counts[5]++] = q;
    }
    uint32_t n_jplaced = 0;
    int rc = schedule_list(o, out_join, counts[5], out_jnode, out_jscore, out_jslots, NULL, out_fail_counts, out_fail_pod, &n_fail,
                           &n_jplaced);
    counts[6] = n_fail;
    if (rc == SIMON_OK)
        rc = schedule_list(o, out_evicted, counts[0], out_node, out_score, out_slots, NULL, out_fail_counts, out_fail_pod, &n_fail,
                           &counts[1]);
    counts[2] = n_fail - counts[6];
    sums[0] = sums[1] = 0;
    for (uint32_t i = 0; i < n_remain; i++) { sums[0] += o->req_mcpu[remain[i]]; sums[1] += o->req_mem[remain[i]]; }
    if (rc == SIMON_OK && apply && (n_fail || counts[3] || (n_join && !retire) || (retire && !state))) rc = SIMON_ERR_INVALID;
    if (rc == SIMON_OK && apply) {
        for (uint32_t j = 0; j < counts[0]; j++) { placement[out_evicted[j]] = out_node[j]; slots[out_evicted[j]] = out_slots[j]; }
        for (uint32_t j = 0; j < counts[5]; j++) { placement[out_join[j]] = out_jnode[j]; slots[out_join[j]] = out_jslots[j]; }
        if (!retire) {
            for (uint32_t j = 0; j < n_van; j++) {
                const uint32_t q = vanished[j];
                const int reserve = o->p.pod_fixed_node[q] == -1;
                o->cur_pin = o->p.pod_pin_node ? o->p.pod_pin_node[q] : -1;
                const uint32_t pack = commit(o, CW(o, (uint32_t)o->p.pod_class[q]), (uint32_t)placement[q], reserve);
                slots[q] = reserve ? pack : 0;
            }
        } else {
            for (uint32_t j = 0; j < n_van; j++) { placement[vanished[j]] = -3; slots[vanished[j]] = 0; }
            /* the pending DaemonSet pods of the retiring nodes stop existing as well */
            for (uint32_t q = 0; q < P; q++) {
                const int64_t guard = guard_of(o, q);
                if (guard >= 0 && !o->active[guard] && state[guard] == 1 && placement[q] == -1) { placement[q] = -3; slots[q] = 0; }
            }
            for (uint32_t g = 0; g < N; g++) {
                if (jn[g]) state[g] = 1;
                else if (!o->active[g] && state[g] == 1) state[g] = 2;
            }
        }
    } else {
        state_io(o, &sv, 0);
    }
    simon_oracle_set_active(o, NULL, 0);
    free(sv.i64); free(sv.i32); free(sv.slots); free(jn); free(vanished);
    return rc;
}
