/*
 * moves_plan_pdb_oracle.c — CPU checker of migration plans with a PodDisruptionBudget table (simon_moves_plan after
 * simon_pdbs_upload, include/simon_gpu.h).  TEST INFRASTRUCTURE ONLY.
 *
 * The plan of tests/moves_plan_oracle.c, restated with the PDB rules: the move-scope checker (and through it the CPU oracle) is
 * compiled in unchanged; every step scores all candidate moves with simon_oracle_moves_score_scoped on the oracle's current state,
 * skips the moves of pods that already moved, of excluded pods and of pods with a PDB at remaining 0, takes the best remaining feasible
 * move by (gain descending, move index ascending), and applies it with the oracle's own primitives (uncommit() on the source, the
 * pod's device memory released as its slot word states, commit() with Reserve on the target).
 *
 * The PDB table is the pod -> PDB CSR pdb_off / pdb_ids and each PDB's `allowed` on the live placement: remaining[j] starts at
 * allowed[j]; each applied step decrements remaining of every PDB of the moved pod.  *out_pdb_blocked counts the placed pods, other
 * than pinned, Open-Local and excluded ones, that a PDB at 0 keeps in place at the start.
 */
#include "moves_scope_oracle.c"

/* out_steps: 6 words per step (move, pod, from, to, gain, gpu slots); placement and slots (the live slot words) are updated in place.
 * Returns 0, or 1 when Reserve on the target gives other slots than the scoring reported, or an error of the scoring. */
int simon_oracle_moves_plan_pdb(simon_oracle *o, uint32_t scope, uint32_t n_moves, const uint32_t *moves, int32_t *placement, uint32_t *slots,
                                const uint8_t *class_local, uint32_t max_moves, int32_t min_gain, uint32_t n_pdbs, const uint32_t *pdb_off,
                                const uint32_t *pdb_ids, const int32_t *allowed, int32_t *out_steps, uint32_t *out_n, uint32_t *out_stop,
                                uint32_t *out_excluded, uint32_t *out_pdb_blocked) {
    const uint32_t P = o->p.n_pods, N = o->N;
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
        uncommit(o, cw, a);
        uint32_t pack = 0;
        if (cw[SCW_GPU_MEM] > 0) {
            for (int d = 0; d < SIMON_MAX_GPU_DEV; d++) o->gpu_used[(uint64_t)d * N + a] -= (int64_t)((slots[p] >> (4 * d)) & 15u) * cw[SCW_GPU_MEM];
            pack = commit(o, cw, b, 1);
            if (pack != ((scope & SCOPE_GPU) ? sl[best] : 0u)) { rc = 1; break; }
            slots[p] = pack;
        } else {
            commit(o, cw, b, 1);
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
