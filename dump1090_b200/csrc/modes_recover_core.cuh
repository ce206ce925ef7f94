// modes_recover_core.cuh — the arithmetic of the recovery pass (modes_recover.cu); the definition is
// in include/modes_b200.h (modes_recovered).
//
// Per bit i < 112 of the candidate's window: the hard bit a_i > c_i, and the selection key
// (w_i << 7) | i with w_i = |a_i - c_i| < 2^16, so that the smallest keys are the smallest (w_i, i).
// The 2^10 subsets of the ten selected positions are searched in 32 parts, one per value of the high
// five subset bits (one warp lane each on the device); each part walks the low five bits in Gray-code
// order, one syndrome XOR per step.  Solutions of the least weight are counted across the parts.
//
// Like modes_signal_core.cuh the file needs nothing from CUDA but a few integer intrinsics, so the
// test suite also compiles it for the host (tests/host_shim/recover_core_host.cpp) and checks it
// against a numpy restatement of the definition.  That build is test infrastructure.
#pragma once
#include <cstdint>
#include "modes_b200.h"

#if defined(__CUDACC__)
#define MODES_RECOVER_FN __host__ __device__ __forceinline__
#else
#define MODES_RECOVER_FN static inline
#endif
#if defined(__CUDA_ARCH__)
#define MODES_RECOVER_UNROLL _Pragma("unroll")
#else
#define MODES_RECOVER_UNROLL
#endif

namespace modes {
namespace recover {

constexpr int kBits = MODES_RECOVER_BITS;             // the positions searched
constexpr int kLowBits = 5;                           // subset bits walked by one part
constexpr uint32_t kNoKey = 0xFFFFFFFFu;              // a position that is never selected
constexpr uint32_t kNoSolution = 0xFFu;               // weight of a part without solution
static_assert(kBits == 2 * kLowBits, "one part per lane: 32 values of the high subset bits");

MODES_RECOVER_FN uint32_t popc(uint32_t x) {
#if defined(__CUDA_ARCH__)
    return __popc(x);
#else
    return (uint32_t)__builtin_popcount(x);
#endif
}

// Selection key of bit i (a = first, c = second magnitude of its pair); bits 0..4 (the DF) and bits
// beyond 111 are never selected.
MODES_RECOVER_FN uint32_t bit_key(uint32_t a, uint32_t c, uint32_t i) {
    const uint32_t w = a > c ? a - c : c - a;
    return (i >= 5 && i < 112) ? (w << 7) | i : kNoKey;
}

// The least weight of a solution among the subsets whose high five bits are `hi`, how many
// solutions have that weight, and (when there is one) its subset: bit k = position k of the ten.
struct Part { uint32_t minw, count, mask; };

// ctz of the Gray-code step (1..31), constant when the walk is unrolled
MODES_RECOVER_FN int step_bit(uint32_t step) {
    int k = 0;
    while (!((step >> k) & 1u)) k++;
    return k;
}

MODES_RECOVER_FN Part search_part(uint32_t hi, const uint32_t syn[kBits], uint32_t s0) {
    uint32_t s = s0;                                  // s0 ^ the syndrome of the subset: 0 when it solves the frame
MODES_RECOVER_UNROLL
    for (int k = 0; k < kLowBits; k++) s ^= ((hi >> k) & 1u) ? syn[kLowBits + k] : 0u;
    const uint32_t wh = popc(hi);
    Part p{kNoSolution, 0u, 0u};
    uint32_t g = 0;
MODES_RECOVER_UNROLL
    for (uint32_t step = 0; step < (1u << kLowBits); step++) {
        if (step) {
            const int k = step_bit(step);
            g ^= 1u << k;
            s ^= syn[k];
        }
        const uint32_t w = wh + popc(g);
        const bool hit = s == 0;
        const bool better = hit && w < p.minw;
        p.count = better ? 1u : p.count + ((hit && w == p.minw) ? 1u : 0u);
        p.mask = better ? (hi << kLowBits) | g : p.mask;
        p.minw = better ? w : p.minw;
    }
    return p;
}

// Status from the least weight over all parts and the number of solutions of that weight.
MODES_RECOVER_FN uint32_t status_of(uint32_t minw, uint32_t count) {
    return minw == kNoSolution ? (uint32_t)MODES_RECOVER_NOT_FOUND
                               : (count == 1 ? (uint32_t)MODES_RECOVER_FOUND : (uint32_t)MODES_RECOVER_AMBIGUOUS);
}

// Record words: frame = the four 32-bit words of frame bits 0..127 (bit 32r + l at bit 31 - l of
// word r, i.e. big-endian bytes), written as the record's 20 little-endian bytes.
MODES_RECOVER_FN uint32_t bswap32(uint32_t x) {
    return (x >> 24) | ((x >> 8) & 0xff00u) | ((x << 8) & 0xff0000u) | (x << 24);
}

MODES_RECOVER_FN void record_words(const uint32_t frame[4], uint32_t status, uint32_t nflips, uint32_t signal,
                                   uint32_t out[5]) {
    out[0] = bswap32(frame[0]);
    out[1] = bswap32(frame[1]);
    out[2] = bswap32(frame[2]);
    out[3] = (bswap32(frame[3]) & 0xffffu) | (status << 16) | (nflips << 24);
    out[4] = signal & 0xffffu;
}

}  // namespace recover
}  // namespace modes
