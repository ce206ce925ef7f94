// modes_signal_core.cuh — the arithmetic of the signal-level pass (modes_signal.cu).
//
// The signal level of a decoded frame of b bits (56 or 112) at reference-buffer position j is
//     S      = sum_{i < b} max(m[j+16+2i], m[j+17+2i])^2            (dump1090.c:1670-1671 sample pairs)
//     signal = floor(sqrt(floor(S / b)))                             (the RMS pulse magnitude)
// over the reference's magnitudes m = round(360 * sqrt((I-127)^2 + (Q-127)^2)) (dump1090.c:359-364),
// always the uncorrected ones.  m <= 65167, so a square fits in 32 bits, S in 39 and the signal in 16.
//
// Like modes_scan_core.cuh the file needs nothing from CUDA but a few integer intrinsics, so the test
// suite also compiles it for the host (tests/host_shim/signal_core_host.cpp) and checks it against a
// plain restatement of the definition.  That build is test infrastructure.
#pragma once
#include <cmath>
#include <cstdint>

#if defined(__CUDACC__)
#define MODES_SIGNAL_FN __host__ __device__ __forceinline__
#else
#define MODES_SIGNAL_FN static inline
#endif

namespace modes {
namespace signal {

// |byte - 127| of the four bytes of a word (I0 Q0 I1 Q1: two samples).
MODES_SIGNAL_FN uint32_t absdiff127x4(uint32_t w) {
#if defined(__CUDA_ARCH__)
    return __vabsdiffu4(w, 0x7f7f7f7fu);
#else
    uint32_t r = 0;
    for (int k = 0; k < 4; k++) {
        const int b = (int)((w >> (8 * k)) & 0xff) - 127;
        r |= (uint32_t)(b < 0 ? -b : b) << (8 * k);
    }
    return r;
#endif
}

// Sum of the products of the four byte pairs of a and b.
MODES_SIGNAL_FN uint32_t dot4(uint32_t a, uint32_t b) {
#if defined(__CUDA_ARCH__)
    return __dp4a(a, b, 0u);
#else
    uint32_t c = 0;
    for (int k = 0; k < 4; k++) c += ((a >> (8 * k)) & 0xff) * ((b >> (8 * k)) & 0xff);
    return c;
#endif
}

// The magnitudes of a bit's two samples: pair = the two samples as one word (first sample in the low
// half), lutn = magnitude keyed by I*I + Q*Q (modes_tables.cpp).
MODES_SIGNAL_FN void pair_mags(uint32_t pair, const uint16_t *lutn, uint32_t &first, uint32_t &second) {
    const uint32_t a = absdiff127x4(pair);
#if defined(__CUDA_ARCH__)
    first = __ldg(lutn + dot4(a & 0x0000ffffu, a)); second = __ldg(lutn + dot4(a & 0xffff0000u, a));
#else
    first = lutn[dot4(a & 0x0000ffffu, a)]; second = lutn[dot4(a & 0xffff0000u, a)];
#endif
}

// Squared pulse of one bit (the larger of its two magnitudes, squared).
MODES_SIGNAL_FN uint32_t pulse_sq(uint32_t pair, const uint16_t *lutn) {
    uint32_t lo, hi;
    pair_mags(pair, lutn, lo, hi);
    const uint32_t p = lo > hi ? lo : hi;
    return p * p;
}

// floor(sqrt(x)) for any 32-bit x: a single-precision estimate is within one of the root
// (x rounds to 24 significant bits, the root to 24 more), so one step each way corrects it.
MODES_SIGNAL_FN uint32_t isqrt32(uint32_t x) {
#if defined(__CUDA_ARCH__)
    uint32_t r = (uint32_t)sqrtf((float)x);
#else
    uint32_t r = (uint32_t)std::sqrt((float)x);
#endif
    if (r > 65535u) r = 65535u;
    if ((uint64_t)r * r > x) r--;
    else if ((uint64_t)(r + 1) * (r + 1) <= x) r++;
    return r;
}

// The signal of a frame of `bits` bits (56 or 112) from its sum of squared pulses.  The mean of the
// squares is at most the largest square, so it fits in 32 bits.
MODES_SIGNAL_FN uint16_t signal_of(uint64_t sum_sq, uint32_t bits) {
    return (uint16_t)isqrt32((uint32_t)(bits == 112 ? sum_sq / 112u : sum_sq / 56u));
}

}  // namespace signal
}  // namespace modes

#if defined(__CUDACC__)
// ---- the window loads the signal and recovery passes share (device only)
#include "modes_internal.h"

namespace modes {
namespace signal {

__device__ __forceinline__ uint32_t raw_sample16(const BatchView &in, uint32_t v) {
    const uint8_t *p = (v < (uint32_t)kHaloSamples) ? in.halo + 2 * v : in.body + 2 * (v - kHaloSamples);
    return *reinterpret_cast<const uint16_t *>(p);
}

// The sample pairs of bits 32r + lane < nb of the frame whose first pair starts at virtual index s;
// bits beyond nb read as no signal (magnitude 0).
__device__ __forceinline__ void load_pairs(const BatchView &in, uint32_t s, uint32_t nb, int lane, uint32_t pair[4]) {
    if (s >= (uint32_t)kHaloSamples) {
        const uint32_t f = s - kHaloSamples;                              // body sample of the first pair
        const uint32_t *wp = reinterpret_cast<const uint32_t *>(in.body) + (f >> 1);
#pragma unroll
        for (int r = 0; r < 4; r++) {
            const uint32_t b = 32 * r + lane;
            pair[r] = 0x7f7f7f7fu;
            if (b < nb) pair[r] = (f & 1u) ? __byte_perm(wp[b], wp[b + 1], 0x5432) : wp[b];
        }
    } else {
        // the window starts in the carry block (first positions of a batch): sample by sample
#pragma unroll
        for (int r = 0; r < 4; r++) {
            const uint32_t b = 32 * r + lane;
            pair[r] = 0x7f7f7f7fu;
            if (b < nb) pair[r] = raw_sample16(in, s + 2 * b) | (raw_sample16(in, s + 2 * b + 1) << 16);
        }
    }
}

}  // namespace signal
}  // namespace modes
#endif
