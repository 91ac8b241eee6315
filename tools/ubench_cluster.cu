// micro-benchmark: cost of cluster barriers and of the engine's all-reduce primitives on a 16-CTA cluster
// build (from the repository root):
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o tools/ubench_cluster tools/ubench_cluster.cu
#include <cstdio>
#include "../open-simulator_b200/csrc/simon_kernel.cuh"

extern "C" __global__ void k_sync(long long *out, int iters, int mode) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    cg::cluster_group cluster = cg::this_cluster();
    SkSmem S;
    const uint32_t NW = (blockDim.x + 31) >> 5;
    sk_carve(S, smem_raw, blockDim.x, 2, 4, 64, cluster.num_blocks());
    for (uint32_t q = threadIdx.x; q < (B_N32 + 2 + 4) * blockDim.x; q += blockDim.x) S.a32[q] = (int32_t)q;
    for (uint32_t q = threadIdx.x; q < C_N8 * blockDim.x; q += blockDim.x) S.a8[q] = (uint8_t)q;
    if (threadIdx.x < 2) ((uint32_t *)(S.wpart + 200))[threadIdx.x] = 0;
    SkRed R{&S, &cluster, cluster.block_rank(), cluster.num_blocks(), 0, nullptr};
    sk_red_init(R);
    long long t0 = clock64();
    unsigned long long acc = threadIdx.x;
    for (int i = 0; i < iters; i++) {
        if (mode == 0) cluster.sync();
        else if (mode == 1) { unsigned long long v[5] = {acc, acc + 1, acc + 2, acc + 3, acc & 1}; const int op[5] = {OP_MINU, OP_MAXU, OP_MINU, OP_MAXU, OP_OR}; sk_allreduce<5>(R, v, op); acc += v[1]; }
        else if (mode == 2) { unsigned long long v[16]; for (int q = 0; q < 16; q++) { v[q] = acc + q; } const int opc[16] = {0,0,2,2,2,1,1,2,1,2,3,3,3,3,3,3}; sk_allreduce<16>(R, v, opc); acc += v[2]; }
        else if (mode == 3) { uint32_t who; unsigned long long k = sk_argmax(R, ((acc & 0xffff) << 24) | (0xFFFFFFu - (cluster.block_rank() * blockDim.x + threadIdx.x)), cluster.num_blocks() * blockDim.x, blockDim.x, who); acc += k + sk_wpay(S, who, 0) + sk_wpay(S, who, S.T); }
        else if (mode == 4) __syncthreads();
        else if (mode == 5) { __threadfence(); cluster.sync(); }
        else if (mode == 6) { unsigned x = (unsigned)acc; for (int q = 0; q < 10; q++) x = __reduce_max_sync(0xffffffffu, x + (threadIdx.x & 31)); acc += x; }
        else if (mode == 7) { unsigned long long x = acc; for (int q = 0; q < 10; q++) x = warp_maxu64(x + (threadIdx.x & 31)); acc += x; }
        else if (mode == 8) {   // one st.async round trip to the own CTA + mbarrier wait, all threads waiting
            const uint32_t ph = R.mph, buf = ph & 1, parity = (ph >> 1) & 1;
            if (threadIdx.x == 0) { sk_mbar_expect(&S.mbar[buf], 8u); sk_st_async(sk_mapa(sk_saddr(S.box + buf * 64), cluster.block_rank()), acc, sk_mapa(sk_saddr(&S.mbar[buf]), cluster.block_rank())); }
            sk_mbar_wait(&S.mbar[buf], parity); acc += S.box[buf * 64]; R.mph++;
        }
        else if (mode == 9) {   // same, to the NEXT CTA of the cluster (ring)
            const uint32_t ph = R.mph, buf = ph & 1, parity = (ph >> 1) & 1, nxt = (cluster.block_rank() + 1) % cluster.num_blocks();
            if (threadIdx.x == 0) { sk_mbar_expect(&S.mbar[buf], 8u); sk_st_async(sk_mapa(sk_saddr(S.box + buf * 64), nxt), acc, sk_mapa(sk_saddr(&S.mbar[buf]), nxt)); }
            sk_mbar_wait(&S.mbar[buf], parity); acc += S.box[buf * 64]; R.mph++;
        }
        else if (mode == 10) {  // CTA-level combine through 32-bit shared atomics + __syncthreads
            unsigned *a = (unsigned *)S.wpart;
            unsigned x = __reduce_max_sync(0xffffffffu, (unsigned)acc + threadIdx.x);
            if ((threadIdx.x & 31) == 0) atomicMax(&a[i & 1], x);
            __syncthreads(); acc += a[i & 1]; if (threadIdx.x == 0) a[(i + 1) & 1] = 0;
        }
        else if (mode == 12) { uint32_t v[6] = {(uint32_t)acc, (uint32_t)acc + 1, (uint32_t)acc + 2, (uint32_t)acc + 3, (uint32_t)acc & 1, 1u}; const int op[6] = {W_MIN, W_MAX, W_MIN, W_MAX, W_OR, W_SUM}; sk_allreduce_w<6>(R, v, op); acc += v[1] + v[5]; }
        else if (mode == 13) { uint32_t v[22]; for (int q = 0; q < 22; q++) v[q] = (uint32_t)acc + q; const int op[22] = {0,0,2,2,2,1,1,2,1,2,3,3,3,3,3,3,3,3,3,3,3,3}; sk_allreduce_w<22>(R, v, op); acc += v[2] + v[0]; }
        else if (mode == 14) {  // allreduce_w<7> followed by the arg-max
            uint32_t who; uint32_t xw[7] = {(uint32_t)acc, (uint32_t)acc + 1, (uint32_t)acc + 2, (uint32_t)acc + 3, (uint32_t)acc & 1, 1u, 0u};
            const int xop[7] = {W_MIN, W_MAX, W_MIN, W_MAX, W_OR, W_SUM, W_SUM};
            sk_allreduce_w<7>(R, xw, xop);
            unsigned long long k = sk_argmax(R, ((acc & 0xffff) << 24) | (0xFFFFFFu - (cluster.block_rank() * blockDim.x + threadIdx.x)), cluster.num_blocks() * blockDim.x, blockDim.x, who); acc += k + sk_wpay(S, who, 0) + xw[1] + xw[5];
        }
        else if (mode == 15) {  // allreduce of 6 words with plain DSMEM stores + release/acquire flag polling (no mbarrier / async proxy)
            const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
            const uint32_t CS = cluster.num_blocks(), buf = i & 1;
            uint32_t w[6] = {(uint32_t)acc, (uint32_t)acc + 1, (uint32_t)acc + 2, (uint32_t)acc + 3, (uint32_t)acc & 1, 1u};
            const int op[6] = {W_MIN, W_MAX, W_MIN, W_MAX, W_OR, W_SUM};
            for (int q = 0; q < 6; q++) w[q] = warp_w(w[q], op[q]);
            uint32_t *wp = (uint32_t *)S.wpart;
            if (lane == 0) for (int q = 0; q < 6; q++) wp[q * SK_MAX_WARPS + warp] = w[q];
            __syncthreads();
            uint32_t *flag = (uint32_t *)(S.wpart + 200);        // two counters, untouched by the partials
            if (warp == 0) {
                uint32_t c[6];
                for (int q = 0; q < 6; q++) c[q] = warp_w(lane < NW ? wp[q * SK_MAX_WARPS + lane] : w_ident(op[q]), op[q]);
                if (lane < CS) {
                    const uint32_t rbox = sk_mapa(sk_saddr(S.box + (size_t)buf * SK_NV * CS + cluster.block_rank()), lane);
                    for (int m2 = 0; m2 < 3; m2++) {
                        unsigned long long v = ((unsigned long long)c[2 * m2 + 1] << 32) | c[2 * m2];
                        asm volatile("st.shared::cluster.b64 [%0], %1;" ::"r"(rbox + 8u * m2 * CS), "l"(v) : "memory");
                    }
                    const uint32_t rflag = sk_mapa(sk_saddr(&flag[buf]), lane);
                    asm volatile("red.release.cluster.shared::cluster.add.u32 [%0], 1;" ::"r"(rflag) : "memory");
                }
            }
            const uint32_t target = ((uint32_t)(i >> 1) + 1u) * CS;
            uint32_t seen;
            do { asm volatile("ld.acquire.cluster.shared::cta.u32 %0, [%1];" : "=r"(seen) : "r"(sk_saddr(&flag[buf])) : "memory"); } while ((int32_t)(seen - target) < 0);
            const unsigned long long *bx = S.box + (size_t)buf * SK_NV * CS;
            for (int m2 = 0; m2 < 3; m2++) {
                const bool in = lane < CS;
                const unsigned long long x = in ? bx[m2 * CS + lane] : 0ull;
                w[2 * m2] = warp_w(in ? (uint32_t)x : w_ident(op[2 * m2]), op[2 * m2]);
                w[2 * m2 + 1] = warp_w(in ? (uint32_t)(x >> 32) : w_ident(op[2 * m2 + 1]), op[2 * m2 + 1]);
            }
            acc += w[1] + w[5];
        }
        else if (mode == 11) {  // CTA-level combine: per-warp slots + __syncthreads + every warp folds
            unsigned *a = (unsigned *)S.wpart + (i & 1) * 32;
            unsigned x = __reduce_max_sync(0xffffffffu, (unsigned)acc + threadIdx.x);
            if ((threadIdx.x & 31) == 0) a[threadIdx.x >> 5] = x;
            __syncthreads(); unsigned y = (threadIdx.x & 31) < NW ? a[threadIdx.x & 31] : 0u; acc += __reduce_max_sync(0xffffffffu, y);
        }
    }
    long long t1 = clock64();
    if (threadIdx.x == 0 && blockIdx.x == 0) { out[0] = (t1 - t0) / iters; out[1] = (long long)acc; }
}

int main() {
    long long *d; cudaMalloc(&d, 64);
    const char *names[16] = {"cluster.sync", "allreduce<5>", "allreduce<16>", "argmax", "__syncthreads", "threadfence+cluster.sync", "10x redux.max.u32 (dependent)", "10x warp_maxu64 (dependent)", "st.async self + mbar wait", "st.async next CTA + mbar wait", "redux+smem atomicMax+bar", "redux+slots+bar+fold", "allreduce_w<6> (32-bit words)", "allreduce_w<22> (32-bit words)", "allreduce_w<7> + arg-max", "allreduce 6 words, st.shared::cluster + flag polling"};
    for (int cs : {1, 2, 4, 8, 16}) for (int tpb : {256, 320}) for (int mode = 0; mode < 16; mode++) {
        size_t smem = sk_smem_bytes(tpb, 2, 4, 64, cs);
        cudaFuncSetAttribute(k_sync, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        cudaFuncSetAttribute(k_sync, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(cs); cfg.blockDim = dim3(tpb); cfg.dynamicSmemBytes = smem;
        cudaLaunchAttribute at[1]; at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = cs; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
        cfg.attrs = at; cfg.numAttrs = 1;
        cudaError_t e = cudaLaunchKernelEx(&cfg, k_sync, d, 2000, mode);
        cudaError_t e2 = cudaDeviceSynchronize();
        long long h[4] = {0, 0, 0, 0};
        cudaMemcpy(h, d, 32, cudaMemcpyDeviceToHost);
        printf("cs=%2d tpb=%4d %-28s %6lld cycles  acc=%lld (%s %s)\n", cs, tpb, names[mode], h[0], h[1], cudaGetErrorString(e), cudaGetErrorString(e2));
    }
    return 0;
}
