// simon_moves.cuh — the per-pod record of the move kernels and the class bits it carries, shared by simon_moves.cu and the
// PodDisruptionBudget kernels (simon_pdb.cu, a translation unit of its own).
#pragma once
#include <stdint.h>

// per-pod record built by the pack kernel of every launch: everything a move needs to know about its pod in ONE 16-byte load,
// so that the class header, the static verdict record and both node records can be fetched in parallel afterwards
struct __align__(16) SmvPod {
    int32_t cls, node;      // class, current node (or < 0)
    uint32_t sig, bits;     // static signature and SmvClass::bits of the class
};
#define SMC_NOT_MOVABLE (1u << 8)
#define SMC_HAS_SCALAR (1u << 9)
#define SMC_NPORTS(b) ((((b) >> 10) & 31u) | (((b) >> 24) & 32u))   // bits 10..14 and 29: 0..63 (a class has at most SK_MAX_ENT = 32)
#define SMC_NFILT(b) (((b) >> 15) & 63u)
#define SMC_OWN_INC (1u << 21)
#define SMC_NEED(b) (((b) >> 22) & 3u)   // SIMON_MOVES_SCOPE_* bits that admit a not-movable class (GPU share, hard spread)
#define SMC_NEED_GPU (1u << 22)
#define SMC_NEED_HARD (1u << 23)
#define SMC_NEVER (1u << 24)             // pinned (DaemonSet) or Open-Local class: not movable under any scope
#define SMC_NHARD(b) (((b) >> 25) & 15u)
