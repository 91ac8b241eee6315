/*
 * moves_scope_oracle.c — CPU checker of the move scope (simon_moves_set_scope; the scoped instantiation of
 * open-simulator_b200/csrc/simon_moves.cu).  TEST INFRASTRUCTURE ONLY, like the oracle it is built on.
 *
 * The CPU oracle (oracle/simon_oracle.c) is compiled into this library unchanged, so that a move of a class the scope admits is
 * evaluated by the oracle's own scheduling-cycle stages rather than by a third restatement of the filters:
 *   take p off its node a (the inverse of commit() for requests, non-zero requests, pod count, scalars and its unconditional
 *   counter increments), run ST_SEL / ST_HARDREG / the hard minimum / ST_FILTER for p's class on the target b, then commit p
 *   back on a.  The first failing filter's reasons are the code; the gain is that of simon_oracle_moves_score.
 * Every other move, and every move under scope 0, is simon_oracle_moves_score's own answer.
 */
#include "../oracle/simon_oracle.c"

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
