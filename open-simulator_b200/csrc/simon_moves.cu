// simon_moves.cu — candidate-move scoring for defragmentation / rebalancing (BASELINE config 5, SURVEY 8e row 3).
//
// The reference has no implementation of this path (README.md:16 names the use case only); what it offers is the
// primitive a rebalancer needs, NodeInfo.RemovePod (vendor/k8s.io/kubernetes/pkg/scheduler/framework/types.go:539-585),
// and the scheduling path restated by this engine.  The definition below is therefore this repository's (DESIGN.md
// section 5) and parity is against oracle/simon_oracle.c:simon_oracle_moves_score.
//
// A move m = (pod p, target node b) is evaluated on the LIVE state the context holds after simon_schedule, with p taken
// off its current node a = placement[p] (RemovePod: requests, non-zero requests, pod count and p's own increments of the
// class's counters at a's domains):
//   code  = first failing filter of this path for p's class on b, in the path's order: static verdict (NodeUnschedulable,
//           NodeName, TaintToleration, NodeAffinity), NodePorts, NodeResourcesFit, InterPodAffinity (required affinity,
//           required anti-affinity, existing pods' anti-affinity), or SMV_* for moves that are not candidates;
//   gain  = [LeastAllocated + BalancedAllocation of b for p]  -  [the same of a for p, with p removed first]
//           i.e. how much better the scheduler's own node-local score likes p on b than where it sits.
// Every move is independent: one thread per move over a read-only snapshot.  Node columns are packed per launch into one
// 96-byte record per node (three 32-byte sectors) so that the two random gathers per move (target, source) cost six
// sectors instead of two dozen; the move list itself streams through coalesced 8-byte loads.
//
// Move scope (simon_moves_set_scope): classes with a GPU-share request and / or DoNotSchedule spread constraints are refused
// (SMV_NOT_MOVABLE) unless the scope admits them; then the scoped instantiation of the kernel adds, in the placement kernel's
// filter order, PodTopologySpread (hard) after NodeResourcesFit and Open-Gpu-Share after InterPodAffinity.  Its inputs are
// built per scoped launch: simon_moves_hard_prep gives every (admitted class, hard constraint) its registered-domain bitmap
// and the minimum of the live counter over those domains, simon_moves_pack_gpu one 96-byte record of free device memory per
// node.  The default instantiation compiles none of it.
#pragma once

struct __align__(32) SmvNode {          // 96 bytes = three 32-byte sectors, ordered by who needs them:
    int64_t alloc_mcpu, alloc_mem, nz_mcpu, nz_mem;      // sector 0: scoring inputs (target AND source node of a move)
    int64_t alloc_eph, req_mcpu, req_mem, req_eph;       // sector 1: NodeResourcesFit inputs (target only)
    int32_t alloc_pods, num_pods;                        // sector 2: pod count + domains (target; source only for classes that
    int32_t dom[6];                                      //           increment counters), topologies 1..6 (0 is the node itself)
};
static_assert(sizeof(SmvNode) == 96, "SmvNode layout");

// per-class header of the move kernel (64 bytes = two sectors), built at upload from the class record
struct __align__(32) SmvClass {
    int64_t score_mcpu, score_mem, nz_mcpu, nz_mem;      // sector 0: scoring
    int64_t req_mcpu, req_mem, req_eph;                  // sector 1: Fit
    uint32_t sig;                                        //           static signature
    uint32_t bits;                                       //           flags:8 | not movable:1 | has scalar request:1 | n_ports, low 5 bits | n_filter entries (aff+anti+exist):6 | own increments:1
                                                         //           | scope bits the class needs:2 | never movable:1 | n_hard:4 | n_ports, bit 5 (32 ports: SK_MAX_ENT)
};
static_assert(sizeof(SmvClass) == 64, "SmvClass layout");
#include "simon_moves.cuh"       // SmvPod and the SMC_* class bits (shared with simon_pdb.cu)
#define SMV_MAX_HARD 8                   // == SK_MAX_HARD: stride of the per-class rows of SmvParams::hs

// free memory per GPU-share device of a node (-1 past gpu_count) and its total gpu-mem: AllocateGpuId's input
struct __align__(32) SmvGpu {
    int64_t free_mem[SIMON_MAX_GPU_DEV];
    int64_t total, pad[3];
};
static_assert(sizeof(SmvGpu) == 96, "SmvGpu layout");

#define SMV_OK 0u
#define SMV_NOOP (1u << 24)            // target == current node
#define SMV_NOT_PLACED (1u << 25)      // the pod is not running anywhere (unscheduled / absent / bound outside the cluster)
#define SMV_NOT_MOVABLE (1u << 26)     // pinned (DaemonSet) or Open-Local class, or one with DoNotSchedule spread constraints / a GPU-share
                                       // request that the move scope does not admit: not a candidate
#define SMV_BAD_INDEX (1u << 27)
#define SMV_GAIN_BIAS 1000
#define SMV_NBINS 401                  // gains lie in [-200, 200]

struct SmvParams {
    uint32_t N, K, WT, T, n_pods, n_moves, use_scache, pad;
    const SmvNode *nodes;
    const int64_t *alloc_scalar, *req_scalar;
    const uint32_t *node_flags;
    const uint64_t *label_bits, *taint_hard;
    const int32_t *topo_dom;
    const uint64_t *class_off;
    const int64_t *class_blob;
    const SmvClass *classes;
    const SmvPod *pods;
    const int32_t *pod_class, *placement;
    const int32_t *cnt, *cnt_total;
    unsigned long long *scache;
    const uint2 *moves;                 // (pod, target)
    int32_t *out_gain;
    uint32_t *out_code;
    unsigned long long *best_per_pod;   // [n_pods] max over the pod's feasible moves of (gain + bias) << 32 | ~move index; 0 = none
    unsigned long long *best_global;    // [1]
    uint32_t *hist;                     // [SMV_NBINS] feasible moves per gain
    uint32_t move_base, pad2;           // global index of moves[0] (multi-GPU shards)
    // scoped instantiation only
    uint32_t scope, pad3;               // SIMON_MOVES_SCOPE_* of this launch
    const SmvGpu *gpu;                  // [N] (GPU share in scope)
    const int2 *hs;                     // [n_classes][SMV_MAX_HARD] (minimum over the registered domains, word offset in hreg)
    const uint32_t *hreg;               // registered-domain bitmaps
    uint32_t *out_slots;                // [n_moves] device slots of feasible GPU-share moves, or NULL
};

__global__ void simon_moves_pack(uint32_t N, uint32_t T, const int64_t *alloc_mcpu, const int64_t *alloc_mem, const int64_t *alloc_eph,
                                 const int32_t *alloc_pods, const int32_t *topo_dom, const int64_t *req_mcpu, const int64_t *req_mem,
                                 const int64_t *req_eph, const int64_t *nz_mcpu, const int64_t *nz_mem, const int32_t *num_pods, SmvNode *out,
                                 unsigned long long *best_per_pod, uint32_t n_pods, unsigned long long *best_global, uint32_t *hist,
                                 const int32_t *pod_class, const int32_t *placement, const SmvClass *classes, SmvPod *pods) {
    // the per-launch outputs are cleared here too (one launch instead of three memsets + a kernel)
    for (uint32_t q = blockIdx.x * blockDim.x + threadIdx.x; q < n_pods; q += gridDim.x * blockDim.x) {
        best_per_pod[q] = 0ull;
        const int32_t c = pod_class[q];
        SmvPod r;
        r.cls = c; r.node = placement[q]; r.sig = classes[c].sig; r.bits = classes[c].bits;
        pods[q] = r;
    }
    if (blockIdx.x == 0) {
        for (uint32_t q = threadIdx.x; q < SMV_NBINS; q += blockDim.x) hist[q] = 0u;
        if (threadIdx.x == 0) *best_global = 0ull;
    }
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= N) return;
    SmvNode r;
    r.alloc_mcpu = alloc_mcpu[g]; r.alloc_mem = alloc_mem[g]; r.alloc_eph = alloc_eph[g];
    r.req_mcpu = req_mcpu[g]; r.req_mem = req_mem[g]; r.req_eph = req_eph[g]; r.nz_mcpu = nz_mcpu[g]; r.nz_mem = nz_mem[g];
    r.alloc_pods = alloc_pods[g]; r.num_pods = num_pods[g];
#pragma unroll
    for (int t = 0; t < 6; t++) r.dom[t] = (uint32_t)(t + 1) < T ? topo_dom[(uint64_t)(t + 1) * N + g] : -1;
    out[g] = r;
}

// GPU record per node for scoped runs with GPU share in scope, from the live device memory in use
__global__ void simon_moves_pack_gpu(uint32_t N, const int32_t *gpu_count, const int64_t *dev_mem, const int64_t *total_mem,
                                     const int64_t *gpu_used, SmvGpu *out) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= N) return;
    const int nd = gpu_count ? gpu_count[g] : 0;
    SmvGpu r;
#pragma unroll
    for (int d = 0; d < SIMON_MAX_GPU_DEV; d++) r.free_mem[d] = d < nd ? dev_mem[g] - gpu_used[(uint64_t)d * N + g] : -1;
    r.total = total_mem ? total_mem[g] : 0;
    r.pad[0] = r.pad[1] = r.pad[2] = 0;
    out[g] = r;
}

// For scoped runs with hard spread in scope: one block per (admitted class, hard constraint j) pair (cls, j, word offset of its
// bitmap in hreg).  The registered domains of the constraint (filtering.go:221-243: nodes that pass the class's node selection and
// carry all of its hard topology keys) from the static verdict cache, or evaluated here where the cache has no record (cache
// disabled, or a record not stored); then the minimum of the live counter over them (INT32_MAX: none), into hs[cls][j].
__global__ void __launch_bounds__(256) simon_moves_hard_prep(uint32_t N, uint32_t use_scache, const unsigned long long *scache,
                                                             const uint64_t *label_bits, const int32_t *topo_dom, const uint32_t *topo_ndom,
                                                             const uint64_t *class_off, const int64_t *class_blob, const int32_t *cnt,
                                                             const uint4 *pairs, uint32_t *hreg, int2 *hs) {
    __shared__ int32_t s_min[8];
    const uint4 pr = pairs[blockIdx.x];
    const int64_t *cw = class_blob + class_off[pr.x];
    const int64_t *r = cw + cw[SCW_OFF_ENT] + 8ull * (uint64_t)(cw[SCW_N_PORTS] + pr.y);
    const int64_t t = r[ER_T];
    const uint32_t nd = topo_ndom[t], nw = (nd + 31) / 32;
    uint32_t *reg = hreg + pr.z;
    for (uint32_t w = threadIdx.x; w < nw; w += blockDim.x) reg[w] = 0u;
    __syncthreads();
    const ReqCtx RC{label_bits, N};
    const uint64_t sig = (uint64_t)cw[SCW_STATIC_SIG];
    const int64_t *hard = cw + cw[SCW_OFF_PTS_HARD];
    for (uint32_t g = threadIdx.x; g < N; g += blockDim.x) {
        const unsigned long long rec = use_scache ? __ldcg(scache + sig * N + g) : 0ull;
        bool elig;
        if (rec & (1ull << 24)) elig = ((rec >> 8) & (NF_SEL_OK | NF_HARDKEYS)) == (NF_SEL_OK | NF_HARDKEYS);
        else {
            elig = selection_ok(cw, RC, g);
            for (int64_t q = 0; q < cw[SCW_N_PTS_HARD]; q++)
                if (topo_dom[(uint64_t)hard[4 * q + 1] * N + g] < 0) elig = false;
        }
        if (elig) {
            const int32_t d = topo_dom[(uint64_t)t * N + g];
            atomicOr(reg + (d >> 5), 1u << (d & 31));
        }
    }
    __syncthreads();
    int32_t mn = INT32_MAX;
    for (uint32_t d = threadIdx.x; d < nd; d += blockDim.x)
        if ((__ldcg(reg + (d >> 5)) >> (d & 31)) & 1u) mn = min(mn, cnt[(uint32_t)r[ER_BASE] + d]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    if ((threadIdx.x & 31) == 0) s_min[threadIdx.x >> 5] = mn;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (uint32_t w = 1; w < blockDim.x / 32; w++) mn = min(mn, s_min[w]);
        hs[(uint64_t)pr.x * SMV_MAX_HARD + pr.y] = make_int2(mn, (int32_t)pr.z);
    }
}

// AllocateGpuId (cache/gpunodeinfo.go:232-290) on a node's free device memory, in registers: the slots in the 4-bits-per-device
// format of simon_gpu_slots_download (saturating at 15), 0 = no assignment.  One GPU: the device of least free memory that holds the
// request, first on ties.  Several: the greedy scan fills device d while it holds the request, then moves on to d + 1, so it can fail
// with enough memory free in total.
__device__ __forceinline__ uint32_t smv_gpu_fit(const SmvGpu &n, int64_t req, int64_t num) {
    if (req <= 0 || num <= 0) return 0u;
    if (num == 1) {
        int cand = -1;
        int64_t cm = 0;
#pragma unroll
        for (int d = 0; d < SIMON_MAX_GPU_DEV; d++)
            if (n.free_mem[d] >= req && (cand < 0 || n.free_mem[d] < cm)) { cand = d; cm = n.free_mem[d]; }
        return cand < 0 ? 0u : 1u << (4 * cand);
    }
    uint32_t out = 0;
    int64_t got = 0;
#pragma unroll 1
    for (int d = 0; d < SIMON_MAX_GPU_DEV && got < num; d++) {
        int64_t take = 0;
        for (int64_t av = n.free_mem[d]; av >= req && got + take < num; av -= req) take++;
        got += take;
        out |= (uint32_t)(take < 15 ? take : 15) << (4 * d);
    }
    return got == num ? out : 0u;
}

// one 32-byte sector as two 128-bit loads (sm_90 has no wider global load; both halves fall in the same sector, so the
// memory traffic is one sector), read-only path
__device__ __forceinline__ void smv_ld_sector(void *dst, const void *src) {
    unsigned long long *d = reinterpret_cast<unsigned long long *>(dst);
    const unsigned long long *s = reinterpret_cast<const unsigned long long *>(src);
    asm volatile("ld.global.nc.v2.b64 {%0,%1}, [%2];" : "=l"(d[0]), "=l"(d[1]) : "l"(s));
    asm volatile("ld.global.nc.v2.b64 {%0,%1}, [%2];" : "=l"(d[2]), "=l"(d[3]) : "l"(s + 2));
}
// sector mask: bit s = load the s-th 32-byte sector of the record (the others stay zero and are never read)
template <int MASK>
__device__ __forceinline__ SmvNode smv_load(const SmvNode *p) {
    SmvNode r;
    unsigned long long *d = reinterpret_cast<unsigned long long *>(&r);
#pragma unroll
    for (int sec = 0; sec < 3; sec++) {
        if ((MASK >> sec) & 1) smv_ld_sector(d + 4 * sec, reinterpret_cast<const unsigned long long *>(p) + 4 * sec);
        else { d[4 * sec] = 0; d[4 * sec + 1] = 0; d[4 * sec + 2] = 0; d[4 * sec + 3] = 0; }
    }
    return r;
}
__device__ __forceinline__ void smv_load_sector(SmvNode &r, const SmvNode *p, int sec) {
    smv_ld_sector(reinterpret_cast<unsigned long long *>(&r) + 4 * sec, reinterpret_cast<const unsigned long long *>(p) + 4 * sec);
}

// exact floor((cap - rq) * 100 / cap) for 0 <= rq <= cap, from the already computed fraction f = rq / cap (correctly rounded):
// the estimate (1 - f) * 100 is within 1e-13 of the true quotient, so one integer fix-up step makes it exact - no second
// division (the emulated 64-bit integer division costs ~100 instructions, an f64 division ~35)
__device__ __forceinline__ int64_t smv_la(int64_t cap, int64_t rq, double f) {
    const int64_t x = (cap - rq) * 100;
    int64_t q = (int64_t)((1.0 - f) * 100.0);
    const int64_t r = x - q * cap;
    if (r < 0) q--;
    else if (r >= cap) q++;
    return q;
}

// LeastAllocated + BalancedAllocation for a pod with scoring request (sc, sm) on a node whose NonZeroRequested is (nzc, nzm)
// (least_allocated.go:93-117, balanced_allocation.go:82-119); same values as the placement kernel's own_core
__device__ __forceinline__ int32_t smv_own(int64_t capc, int64_t capm, int64_t nzc, int64_t nzm, int64_t sc, int64_t sm) {
    const int64_t rqc = nzc + sc, rqm = nzm + sm;
    const double cf = capc == 0 ? 1.0 : (double)rqc / (double)capc;
    const double mf = capm == 0 ? 1.0 : (double)rqm / (double)capm;
    const int64_t s1 = (capc == 0 || rqc > capc) ? 0 : smv_la(capc, rqc, cf);
    const int64_t s2 = (capm == 0 || rqm > capm) ? 0 : smv_la(capm, rqm, mf);
    const int64_t la = (s1 + s2) / 2;
    int64_t ba = 0;
    if (!(cf >= 1.0 || mf >= 1.0)) ba = f2i((1.0 - fabs(cf - mf)) * 100.0);
    return (int32_t)(la + ba);
}

// domain of node g on topology t: topology 0 is the node itself, 1..6 travel in the packed record, 7 (rare) is gathered
__device__ __forceinline__ int32_t smv_dom(const SmvParams &P, const SmvNode &n, uint32_t g, int64_t t) {
    if (t == 0) return (int32_t)g;
    if (t <= 6) {
        int32_t d = n.dom[0];
#pragma unroll
        for (int q = 1; q < 6; q++) d = (t == q + 1) ? n.dom[q] : d;
        return d;
    }
    return __ldg(P.topo_dom + (uint64_t)t * P.N + g);
}

// SCOPED: the instantiation for runs whose scope admits a class (see the top of this file)
template <int MINB, bool SCOPED>
__global__ void __launch_bounds__(256, MINB) simon_moves_kernel(const __grid_constant__ SmvParams P) {
    __shared__ uint32_t s_hist[SMV_NBINS];
    for (uint32_t q = threadIdx.x; q < SMV_NBINS; q += blockDim.x) s_hist[q] = 0;
    __syncthreads();
    const ReqCtx RC{P.label_bits, P.N};
    unsigned long long my_best = 0;
    for (uint32_t m = blockIdx.x * blockDim.x + threadIdx.x; m < P.n_moves; m += gridDim.x * blockDim.x) {
        const uint2 mv = __ldg(P.moves + m);
        const uint32_t pod = mv.x, b = mv.y;
        uint32_t code = SMV_OK, slots = 0;
        int32_t gain = 0;
        int32_t a = -1;
        SmvPod pr;
        pr.cls = 0; pr.node = -1; pr.sig = 0; pr.bits = 0;
        if (pod >= P.n_pods || b >= P.N) code = SMV_BAD_INDEX;
        else {
            const int4 v = __ldg(reinterpret_cast<const int4 *>(P.pods + pod));
            pr.cls = v.x; pr.node = v.y; pr.sig = (uint32_t)v.z; pr.bits = (uint32_t)v.w;
            a = pr.node;
            if (a < 0 || (uint32_t)a >= P.N) code = SMV_NOT_PLACED;
            else if ((uint32_t)a == b) code = SMV_NOOP;
            else if ((pr.bits & SMC_NOT_MOVABLE) && (!SCOPED || (pr.bits & SMC_NEVER) || (SMC_NEED(pr.bits) & ~P.scope))) code = SMV_NOT_MOVABLE;
        }
        if (code == SMV_OK) {
            const int32_t cls = pr.cls;
            // the four gathers of a move are independent now: class header, static verdict record, target and source node
            unsigned long long rec = P.use_scache ? __ldcg(P.scache + (uint64_t)pr.sig * P.N + b) : 0ull;
            SmvClass kc;
            smv_ld_sector(&kc, P.classes + cls);
            smv_ld_sector(reinterpret_cast<unsigned long long *>(&kc) + 4, reinterpret_cast<const unsigned long long *>(P.classes + cls) + 4);
            const uint32_t bits = kc.bits, cflags = bits & 0xffu;
            {
                const uint32_t n_ports = SMC_NPORTS(bits), n_filt = SMC_NFILT(bits), n_hard = SCOPED ? SMC_NHARD(bits) : 0u;
                const bool need_ent = (n_ports | n_filt | n_hard) != 0;
                const SmvNode nb = smv_load<7>(P.nodes + b);
                SmvNode na = smv_load<1>(P.nodes + a);
                if (need_ent && (bits & SMC_OWN_INC)) smv_load_sector(na, P.nodes + a, 2);       // the source's domains: only to take p's own counts out
                // ---- static verdict of (class, b): cached per (static signature, node) by the placement kernel, or computed here
                uint32_t st_code;
                const int64_t *cw = nullptr;
                if (rec & (1ull << 24)) st_code = (uint32_t)(rec & 0xff);
                else {
                    cw = P.class_blob + __ldg(P.class_off + cls);
                    const bool ok = selection_ok(cw, RC, b);
                    const int64_t *tol = cw + cw[SCW_OFF_TOL];
                    st_code = 0;
                    if ((P.node_flags[b] & SIMON_NODE_UNSCHEDULABLE) && !(cflags & SIMON_CLS_TOL_UNSCHED)) st_code = 1;
                    if (!st_code && cw[SCW_NODE_NAME] != -1 && cw[SCW_NODE_NAME] != (int64_t)b) st_code = 2;
                    if (!st_code)
                        for (uint32_t w = 0; w < P.WT; w++)
                            if (P.taint_hard[(uint64_t)w * P.N + b] & ~(uint64_t)tol[w]) st_code = 3;
                    if (!st_code && !ok) st_code = 4;
                }
                if (st_code) code = 1u << SFC_STATIC;
                if (code == SMV_OK && need_ent && !cw) cw = P.class_blob + __ldg(P.class_off + cls);
                const int64_t *et = need_ent && cw ? cw + cw[SCW_OFF_ENT] : nullptr;
                // counter value of entry e at b's domain with p's own contribution (made from node a: its multiplicity in the
                // counter) removed
                auto val_at = [&](uint32_t e, int32_t d) -> int32_t {
                    const int64_t *r = et + 8ull * e;
                    int32_t v = __ldg(P.cnt + (uint32_t)r[ER_BASE] + (uint32_t)d);
                    if (r[ER_INC] && smv_dom(P, na, (uint32_t)a, r[ER_T]) == d) v -= (int32_t)r[ER_INC];
                    return v;
                };
                // ---- NodePorts
                if (code == SMV_OK)
                    for (uint32_t e = 0; e < n_ports; e++)
                        if (val_at(e, (int32_t)b) > 0) { code = 1u << SFC_PORTS; break; }
                // ---- NodeResourcesFit on b (p is not on b)
                if (code == SMV_OK) {
                    uint32_t rs = 0;
                    if (nb.num_pods + 1 > nb.alloc_pods) rs |= 1u << SFC_TOO_MANY_PODS;
                    if (cflags & SIMON_CLS_HAS_REQUEST) {
                        if (nb.alloc_mcpu < kc.req_mcpu + nb.req_mcpu) rs |= 1u << SFC_CPU;
                        if (nb.alloc_mem < kc.req_mem + nb.req_mem) rs |= 1u << SFC_MEM;
                        if (nb.alloc_eph < kc.req_eph + nb.req_eph) rs |= 1u << SFC_EPH;
                        if (bits & SMC_HAS_SCALAR) {
                            const int64_t *cw3 = cw ? cw : P.class_blob + __ldg(P.class_off + cls);
                            const int64_t *sc_req = cw3 + cw3[SCW_OFF_SCALARS];
                            for (uint32_t k = 0; k < P.K; k++)
                                if (sc_req[k] != 0 && P.alloc_scalar[(uint64_t)k * P.N + b] < sc_req[k] + P.req_scalar[(uint64_t)k * P.N + b]) rs |= 1u << (SFC_SCALAR0 + k);
                        }
                    }
                    code = rs;
                }
                // ---- PodTopologySpread, DoNotSchedule constraints (filtering.go:276-328) with p removed: b's count loses p's own
                // count if p's sits at b's domain (val_at), and the minimum over the registered domains becomes
                // min(min, cnt[dom_a] - m) when p's count m (its class's multiplicity in the counter) sits at a registered dom_a
                if (SCOPED && code == SMV_OK && n_hard) {
                    const int2 *hs = P.hs + (uint64_t)cls * SMV_MAX_HARD;
#pragma unroll 1
                    for (uint32_t j = 0; j < n_hard; j++) {
                        const int64_t *r = et + 8ull * (n_ports + j);
                        const int64_t t = r[ER_T];
                        const int32_t db = smv_dom(P, nb, b, t);
                        if (db < 0) { code = 1u << SFC_PTS_MISSING; break; }
                        const int2 h = __ldg(hs + j);
                        const uint32_t *reg = P.hreg + (uint32_t)h.y;
                        const int32_t match = ((__ldg(reg + (db >> 5)) >> (db & 31)) & 1u) ? val_at(n_ports + j, db) : 0;
                        int32_t mn = h.x;
                        if (r[ER_INC]) {
                            const int32_t da = smv_dom(P, na, (uint32_t)a, t);
                            if (da >= 0 && ((__ldg(reg + (da >> 5)) >> (da & 31)) & 1u))
                                mn = min(mn, __ldg(P.cnt + (uint32_t)r[ER_BASE] + (uint32_t)da) - (int32_t)r[ER_INC]);
                        }
                        if ((int64_t)match + r[ER_B] - (int64_t)mn > r[ER_A]) { code = 1u << SFC_PTS_SKEW; break; }
                    }
                }
                // ---- InterPodAffinity (filtering.go:317-401) on the counters, p's own increments taken out
                if (code == SMV_OK && n_filt) {
                    const uint32_t n_soft = (uint32_t)cw[SCW_N_PTS_SOFT], n_aff = (uint32_t)cw[SCW_N_IPA_AFF];
                    const uint32_t n_anti = (uint32_t)cw[SCW_N_IPA_ANTI], n_exist = (uint32_t)cw[SCW_N_IPA_EXIST];
                    const uint32_t e_aff = n_ports + n_hard + n_soft, e_anti = e_aff + n_aff, e_exist = e_anti + n_anti, e_end = e_exist + n_exist;
                    if (n_aff) {
                        bool pods_exist = true, missing = false;
                        long long aff_total = 0;
                        for (uint32_t e = e_aff; e < e_anti; e++) {
                            const int64_t *r = et + 8ull * e;
                            aff_total += __ldg(P.cnt_total + r[ER_K]);
                            if (r[ER_INC] && smv_dom(P, na, (uint32_t)a, r[ER_T]) >= 0) aff_total -= 1;
                            const int32_t d = smv_dom(P, nb, b, r[ER_T]);
                            if (d < 0) { missing = true; continue; }
                            if (val_at(e, d) <= 0) pods_exist = false;
                        }
                        bool ok = true;
                        if (missing) ok = false;
                        else if (!pods_exist) ok = aff_total == 0 && (cflags & SIMON_CLS_IPA_SELF_MATCH);
                        if (!ok) code = 1u << SFC_IPA_AFF;
                    }
                    if (code == SMV_OK)
                        for (uint32_t e = e_anti; e < e_exist; e++) {
                            const int32_t d = smv_dom(P, nb, b, (et + 8ull * e)[ER_T]);
                            if (d >= 0 && val_at(e, d) > 0) { code = 1u << SFC_IPA_ANTI; break; }
                        }
                    if (code == SMV_OK)
                        for (uint32_t e = e_exist; e < e_end; e++) {
                            const int32_t d = smv_dom(P, nb, b, (et + 8ull * e)[ER_T]);
                            if (d >= 0 && val_at(e, d) > 0) { code = 1u << SFC_IPA_EXIST; break; }
                        }
                }
                // ---- Open-Gpu-Share (open-gpu-share.go:51-81) on b's live device memory; p's devices on a do not matter (b != a)
                if (SCOPED && code == SMV_OK && (bits & SMC_NEED_GPU)) {
                    if (!cw) cw = P.class_blob + __ldg(P.class_off + cls);
                    const int64_t req = cw[SCW_GPU_MEM];
                    SmvGpu gr;
#pragma unroll
                    for (int sec = 0; sec < 3; sec++)
                        smv_ld_sector(reinterpret_cast<unsigned long long *>(&gr) + 4 * sec, reinterpret_cast<const unsigned long long *>(P.gpu + b) + 4 * sec);
                    slots = smv_gpu_fit(gr, req, cw[SCW_GPU_COUNT]);
                    if (gr.total < req || slots == 0u) { code = 1u << SFC_GPU; slots = 0u; }
                }
                if (code == SMV_OK) {
                    const int32_t on_b = smv_own(nb.alloc_mcpu, nb.alloc_mem, nb.nz_mcpu, nb.nz_mem, kc.score_mcpu, kc.score_mem);
                    const int32_t on_a = smv_own(na.alloc_mcpu, na.alloc_mem, na.nz_mcpu - kc.nz_mcpu, na.nz_mem - kc.nz_mem, kc.score_mcpu, kc.score_mem);
                    gain = on_b - on_a;
                }
            }
        }
        P.out_gain[m] = gain;
        P.out_code[m] = code;
        if (SCOPED && P.out_slots) P.out_slots[m] = slots;
        if (code == SMV_OK) {
            const uint32_t gm = P.move_base + m;
            const unsigned long long key = ((unsigned long long)(uint32_t)(gain + SMV_GAIN_BIAS) << 32) | (unsigned long long)(0xffffffffu - gm);
            asm volatile("red.global.max.u64 [%0], %1;" ::"l"(P.best_per_pod + pod), "l"(key) : "memory");
            my_best = key > my_best ? key : my_best;
            int bin = gain + 200;
            bin = bin < 0 ? 0 : (bin > SMV_NBINS - 1 ? SMV_NBINS - 1 : bin);
            asm volatile("red.shared.add.u32 [%0], 1;" ::"r"((uint32_t)__cvta_generic_to_shared(&s_hist[bin])) : "memory");
        }
    }
    my_best = warp_maxu64(my_best);
    if ((threadIdx.x & 31) == 0 && my_best) atomicMax(P.best_global, my_best);
    __syncthreads();
    for (uint32_t q = threadIdx.x; q < SMV_NBINS; q += blockDim.x)
        if (s_hist[q]) atomicAdd(P.hist + q, s_hist[q]);
}

// Static verdict records of EVERY (static signature, node) pair, computed densely (one thread per pair, the node index
// fastest: label / taint words are read coalesced) - what the placement kernel's class switch fills lazily on first use
// (same record format: code:8 | flags:8 | tt:8 | valid bit 24 | na:32).  A snapshot that was imported rather than placed
// (all pods pre-bound) has an empty cache; scoring a million moves against it would otherwise evaluate a selector program
// per move.  sig_class[s] = a class that carries signature s.
__global__ void __launch_bounds__(256) simon_static_fill(SkParams P, const uint32_t *sig_class, uint32_t n_sigs) {
    const ReqCtx RC{P.label_bits, P.N};
    const uint64_t total = (uint64_t)n_sigs * P.N;
    for (uint64_t q = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; q < total; q += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t sig = (uint32_t)(q / P.N), g = (uint32_t)(q % P.N);
        if (__ldcg(P.scache + q) & (1ull << 24)) continue;
        const int64_t *cw = P.class_blob + P.class_off[sig_class[sig]];
        const uint32_t cflags = (uint32_t)cw[SCW_FLAGS];
        const bool ok = selection_ok(cw, RC, g);
        uint8_t fl = ok ? NF_SEL_OK : 0, code = 0;
        const int64_t *tol = cw + cw[SCW_OFF_TOL];
        if ((P.node_flags[g] & SIMON_NODE_UNSCHEDULABLE) && !(cflags & SIMON_CLS_TOL_UNSCHED)) code = 1;
        if (!code && cw[SCW_NODE_NAME] != -1 && cw[SCW_NODE_NAME] != (int64_t)g) code = 2;
        if (!code)
            for (uint32_t w = 0; w < P.WT; w++)
                if (P.taint_hard[(uint64_t)w * P.N + g] & ~(uint64_t)tol[w]) code = 3;
        if (!code && !ok) code = 4;
        const int64_t *p = cw + cw[SCW_OFF_PREF];
        int64_t na64 = 0;
        for (int64_t z = 0; z < cw[SCW_N_PREF]; z++) { int64_t w = *p++; if (term_eval(p, RC, g)) na64 += w; }
        int32_t tt = 0;
        for (uint32_t w = 0; w < P.WT; w++) tt += __popcll(P.taint_soft[(uint64_t)w * P.N + g] & ~(uint64_t)tol[P.WT + w]);
        bool hk = true, ign = false;
        const int64_t *hard = cw + cw[SCW_OFF_PTS_HARD], *soft = cw + cw[SCW_OFF_PTS_SOFT];
        for (int64_t j = 0; j < cw[SCW_N_PTS_HARD]; j++) if (P.topo_dom[(uint64_t)hard[4 * j + 1] * P.N + g] < 0) hk = false;
        for (int64_t j = 0; j < cw[SCW_N_PTS_SOFT]; j++) if (P.topo_dom[(uint64_t)soft[5 * j + 1] * P.N + g] < 0) ign = true;
        if (hk) fl |= NF_HARDKEYS;
        if (ign) fl |= NF_IGNORED;
        if (tt < 256)
            P.scache[q] = (unsigned long long)code | ((unsigned long long)fl << 8) | ((unsigned long long)(uint32_t)tt << 16) | (1ull << 24) |
                          ((unsigned long long)(uint32_t)(int32_t)na64 << 32);
    }
}

// Top-k by (gain descending, move index ascending): one block scans the move list in index order and keeps every feasible
// move above the threshold gain plus the first `need_eq` moves exactly at it (the threshold comes from the histogram).
__global__ void __launch_bounds__(1024) simon_moves_collect(uint32_t n_moves, const int32_t *gain, const uint32_t *code, int32_t thr,
                                                            uint32_t need_eq, uint32_t k, uint32_t move_base, uint2 *out, uint32_t *out_n) {
    __shared__ uint32_t s_gt[32], s_eq[32];
    __shared__ uint32_t base_gt, base_eq;
    if (threadIdx.x == 0) { base_gt = 0; base_eq = 0; }
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (uint32_t m0 = 0; m0 < n_moves; m0 += blockDim.x) {
        const uint32_t m = m0 + threadIdx.x;
        bool gt = false, eq = false;
        int32_t g = 0;
        if (m < n_moves && code[m] == SMV_OK) { g = gain[m]; gt = g > thr; eq = g == thr; }
        const uint32_t bg = __ballot_sync(0xffffffffu, gt), be = __ballot_sync(0xffffffffu, eq);
        if (lane == 0) { s_gt[warp] = __popc(bg); s_eq[warp] = __popc(be); }
        __syncthreads();
        uint32_t og = 0, oe = 0;
        for (uint32_t w = 0; w < warp; w++) { og += s_gt[w]; oe += s_eq[w]; }
        const uint32_t rg = base_gt + og + __popc(bg & ((1u << lane) - 1u));
        const uint32_t re = base_eq + oe + __popc(be & ((1u << lane) - 1u));
        if (gt && rg < k) out[rg] = make_uint2(move_base + m, (uint32_t)g);
        if (eq && re < need_eq) out[k + re] = make_uint2(move_base + m, (uint32_t)g);       // ties are stored after the k "greater" slots
        __syncthreads();
        if (threadIdx.x == 0) {
            uint32_t tg = 0, te = 0;
            for (uint32_t w = 0; w < (blockDim.x >> 5); w++) { tg += s_gt[w]; te += s_eq[w]; }
            base_gt += tg; base_eq += te;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) { out_n[0] = base_gt < k ? base_gt : k; out_n[1] = base_eq < need_eq ? base_eq : need_eq; }
}

// ---- migration plans (simon_moves_plan, include/simon_gpu.h) ----------------------------------------------------------------------
// A plan runs the scoring kernels above unchanged on plan-owned copies of the dynamic columns; between two scoring passes the apply
// kernel below moves the winner and patches the packed records (SmvNode of a and b, SmvGpu of a and b, SmvPod of p) in place, so no
// pack runs after the setup.  Control words: ctl[0] steps recorded, ctl[1] stop reason (SMV_PLAN_ERROR: inconsistency), ctl[2] the
// inconsistency (SMV_PLAN_ERR_*), ctl[3] the excluded pods.
#define SMV_PLAN_ERROR 0xffu
#define SMV_PLAN_ERR_SLOTS 1u            // Reserve on the target gave other slots than the scoring reported
#define SMV_PLAN_ERR_NEGATIVE 2u         // a count of the source node would go negative

struct SmvPlan {
    uint32_t max_moves;
    int32_t min_gain;
    int64_t *req_mcpu, *req_mem, *req_eph, *nz_mcpu, *nz_mem, *req_scalar, *gpu_used;
    int32_t *num_pods, *cnt, *cnt_total, *place;
    uint32_t *slots;                    // [P] GPU slot word of every pod
    const uint2 *moves;
    const uint32_t *mv_slots;           // [n_moves] slots the scoring reported (GPU share in scope), or NULL
    unsigned long long *best_global;
    uint32_t *hist;
    SmvNode *nodes;
    SmvGpu *gpu;                        // NULL unless the scoring reads it
    SmvPod *pods;
    simon_plan_step *steps;
    uint32_t *ctl;
};

// After simon_moves_pack on the plan copies: the excluded pods (placed, of a GPU-share class that is neither pinned nor Open-Local,
// with a saturated nibble in the slot word) become never movable, and are counted
__global__ void simon_moves_plan_setup(uint32_t n_pods, const uint32_t *slots, SmvPod *pods, uint32_t *ctl) {
    for (uint32_t q = blockIdx.x * blockDim.x + threadIdx.x; q < n_pods; q += gridDim.x * blockDim.x) {
        const SmvPod r = pods[q];
        if (!(r.bits & SMC_NEED_GPU) || (r.bits & SMC_NEVER) || r.node < 0) continue;
        const uint32_t w = slots[q];
        bool sat = false;
#pragma unroll
        for (int d = 0; d < SIMON_MAX_GPU_DEV; d++) sat |= ((w >> (4 * d)) & 15u) == 15u;
        if (sat) {
            pods[q].bits = r.bits | SMC_NOT_MOVABLE | SMC_NEVER;
            atomicAdd(ctl + 3, 1u);
        }
    }
}

// One step's apply (one warp): the best key of the scoring pass, the stop conditions, then pod p moves from a to b on the plan
// columns - lane 0 the node sums and the devices, every lane a share of the scalars and of the commit list (eligibility-conditional
// entries as simon_import_kernel counts them) - and the packed records follow.  Clears the best key and the histogram for the next pass.
__global__ void __launch_bounds__(32) simon_moves_plan_apply(const __grid_constant__ SkParams P, const __grid_constant__ SmvPlan Q) {
    const uint32_t lane = threadIdx.x;
    if (Q.ctl[1]) return;                // stopped: the passes enqueued after the stop score for nothing
    const unsigned long long key = *Q.best_global;
    const int32_t gain = (int32_t)(uint32_t)(key >> 32) - SMV_GAIN_BIAS;
    __syncwarp();
    if (key == 0ull || gain < Q.min_gain) {
        if (lane == 0) Q.ctl[1] = SIMON_PLAN_STOP_NO_MOVE;
        return;
    }
    const uint32_t m = 0xffffffffu - (uint32_t)key;
    const uint2 mv = Q.moves[m];
    const uint32_t p = mv.x, b = mv.y, N = P.N;
    const uint32_t a = (uint32_t)Q.place[p];
    const int64_t *cw = P.class_blob + P.class_off[P.pod_class[p]];
    bool neg = false;
    uint32_t pack = 0, err = 0;
    if (lane == 0) {
        Q.req_mcpu[a] -= cw[SCW_REQ_MCPU]; Q.req_mem[a] -= cw[SCW_REQ_MEM]; Q.req_eph[a] -= cw[SCW_REQ_EPH];
        Q.nz_mcpu[a] -= cw[SCW_NZ_MCPU]; Q.nz_mem[a] -= cw[SCW_NZ_MEM]; Q.num_pods[a] -= 1;
        neg |= Q.req_mcpu[a] < 0 || Q.req_mem[a] < 0 || Q.req_eph[a] < 0 || Q.nz_mcpu[a] < 0 || Q.nz_mem[a] < 0 || Q.num_pods[a] < 0;
        Q.req_mcpu[b] += cw[SCW_REQ_MCPU]; Q.req_mem[b] += cw[SCW_REQ_MEM]; Q.req_eph[b] += cw[SCW_REQ_EPH];
        Q.nz_mcpu[b] += cw[SCW_NZ_MCPU]; Q.nz_mem[b] += cw[SCW_NZ_MEM]; Q.num_pods[b] += 1;
        if (cw[SCW_GPU_MEM] > 0) {
            // release on a what the slot word states (0 for a pre-bound pod), then Reserve on b
            const uint32_t w = Q.slots[p];
#pragma unroll 1
            for (int d = 0; d < SIMON_MAX_GPU_DEV; d++) {
                const int64_t n = (w >> (4 * d)) & 15u;
                if (!n) continue;
                Q.gpu_used[(uint64_t)d * N + a] -= n * cw[SCW_GPU_MEM];
                neg |= Q.gpu_used[(uint64_t)d * N + a] < 0;
            }
            SkScenario SC{};
            SC.gpu_used = Q.gpu_used;
            pack = gpu_reserve(P, SC, cw, b);
            if (pack != (Q.mv_slots ? Q.mv_slots[m] : 0u)) err = SMV_PLAN_ERR_SLOTS;
        }
    }
    const int64_t *sc = cw + cw[SCW_OFF_SCALARS];
    for (uint32_t k = lane; k < P.K; k += 32) {
        if (sc[k] == 0) continue;
        Q.req_scalar[(uint64_t)k * N + a] -= sc[k];
        neg |= Q.req_scalar[(uint64_t)k * N + a] < 0;
        Q.req_scalar[(uint64_t)k * N + b] += sc[k];
    }
    const ReqCtx RC{P.label_bits, N, -1};
    const int64_t *inc = cw + cw[SCW_OFF_INC];
    for (int64_t u = lane; u < cw[SCW_N_INC]; u += 32) {
        const int64_t k = inc[3 * u], t = inc[3 * u + 1], sig = inc[3 * u + 2];
        const int32_t da = P.topo_dom[(uint64_t)t * N + a], db = P.topo_dom[(uint64_t)t * N + b];
        if (da >= 0 && (sig < 0 || elig_eval(P, sig, RC, a))) {
            neg |= atomicSub(&Q.cnt[P.cnt_off[k] + da], 1) <= 0;
            neg |= atomicSub(&Q.cnt_total[k], 1) <= 0;
        }
        if (db >= 0 && (sig < 0 || elig_eval(P, sig, RC, b))) {
            atomicAdd(&Q.cnt[P.cnt_off[k] + db], 1);
            atomicAdd(&Q.cnt_total[k], 1);
        }
    }
    if (__any_sync(0xffffffffu, neg) && !err) err = SMV_PLAN_ERR_NEGATIVE;
    for (uint32_t q = lane; q < SMV_NBINS; q += 32) Q.hist[q] = 0u;
    if (lane != 0) return;
    if (err) {
        Q.ctl[2] = err;
        Q.ctl[1] = SMV_PLAN_ERROR;
        return;
    }
    Q.place[p] = (int32_t)b;
    if (cw[SCW_GPU_MEM] > 0) Q.slots[p] = pack;
    const uint32_t ends[2] = {a, b};
#pragma unroll
    for (int e = 0; e < 2; e++) {
        const uint32_t g = ends[e];
        SmvNode &r = Q.nodes[g];
        r.req_mcpu = Q.req_mcpu[g]; r.req_mem = Q.req_mem[g]; r.req_eph = Q.req_eph[g];
        r.nz_mcpu = Q.nz_mcpu[g]; r.nz_mem = Q.nz_mem[g]; r.num_pods = Q.num_pods[g];
        if (Q.gpu) {
            const int nd = P.gpu_count ? P.gpu_count[g] : 0;
#pragma unroll 1
            for (int d = 0; d < SIMON_MAX_GPU_DEV; d++) Q.gpu[g].free_mem[d] = d < nd ? P.gpu_dev_mem[g] - Q.gpu_used[(uint64_t)d * N + g] : -1;
        }
    }
    Q.pods[p].node = (int32_t)b;
    Q.pods[p].bits |= SMC_NOT_MOVABLE | SMC_NEVER;          // each pod moves at most once
    const uint32_t s = Q.ctl[0];
    simon_plan_step st;
    st.move = m; st.pod = p; st.from = (int32_t)a; st.to = (int32_t)b; st.gain = gain; st.gpu_slots = pack;
    Q.steps[s] = st;
    Q.ctl[0] = s + 1;
    if (s + 1 >= Q.max_moves) Q.ctl[1] = SIMON_PLAN_STOP_MAX_MOVES;
    *Q.best_global = 0ull;
}
