// simon_flip_word.h — the flip word of the placement kernel's steady-state all-reduce (simon_kernel.cu, "P2 + all-reduce").
//
// After P1 every thread contributes one 32-bit word (dc << NF_BITS) + nf, where nf is the number of its nodes whose feasibility
// flipped and dc the net change of its counted (feasible, not ignored) set; the words are summed modulo 2^32 over the cluster.
// The sum decodes exactly while the total flip count stays below 2^NF_BITS and the total dc fits the 32 - NF_BITS signed bits
// above it; a larger |dc| decodes modulo 2^(32 - NF_BITS).
//   - The shared-memory variants hold at most 20,480 nodes: 16 / 16 bits, both fields exact.
//   - The large-cluster variant holds up to 16 x 320 x 64 = 327,680 nodes (< 2^19): 20 bits of flip count, always exact, and
//     12 bits of dc, exact for |dc| <= 2,047.  The single-node flip fast path reads dc only when exactly one node flipped
//     (|dc| <= 1); everywhere else dc only predicts the hostname-spread sizes, which the full summary checks (sizes_ok).
// Plain C++ as well as CUDA, so that a host test can check the arithmetic with the same code.
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define SK_FLIP_HD __host__ __device__ __forceinline__
#else
#define SK_FLIP_HD inline
#endif

template <bool BIG>
struct SkFlipWord {
    static constexpr int NF_BITS = BIG ? 20 : 16;
    static constexpr uint32_t NF_MASK = (1u << NF_BITS) - 1u;
    // one thread's word: nf <= 64 node slots, |dc| <= nf
    static SK_FLIP_HD uint32_t enc(int32_t dc, uint32_t nf) { return ((uint32_t)dc << NF_BITS) + nf; }
    // the cluster sum of the words -> total flip count
    static SK_FLIP_HD uint32_t nf(uint32_t sum) { return sum & NF_MASK; }
    // the cluster sum of the words and its flip count nf(sum) -> net change of the counted set (sign-extended upper field)
    static SK_FLIP_HD int32_t dc(uint32_t sum, uint32_t nf) { return (int32_t)(sum - nf) >> NF_BITS; }
};
