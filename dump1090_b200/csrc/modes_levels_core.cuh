// modes_levels_core.cuh — the arithmetic of the level pass (modes_levels.cu).
//
// Per reference buffer the pass sums, over the buffer's own 131072 samples,
//     sum_mag   = sum m          sum_power = sum m^2          peak = max m
//     clipped   = samples whose I or Q byte is 0 or 255 (the ADC's rails)
// with m = round(360 * sqrt((I-127)^2 + (Q-127)^2)), the reference's magnitude (dump1090.c:359-364,
// :1454-1469).  m <= 65167, so m^2 fits in 32 bits; the sums are 64-bit integers and do not depend on
// the order they are added in.
//
// A word is four stream bytes I0 Q0 I1 Q1: two samples.  |byte - 127| of the four bytes (SIMD),
// then n = I^2 + Q^2 of each sample as a byte dot product, then m = lutn[n] (modes_tables.cpp).
// Clipping is tested cheaply first: a byte with |b - 127| >= 127 is 0, 254 or 255, and only words
// holding one are counted exactly.
//
// Like modes_signal_core.cuh the file needs nothing from CUDA but a few integer intrinsics, so the
// test suite also compiles it for the host (tests/host_shim/levels_core_host.cpp) and checks it
// against a plain restatement of the definition.  That build is test infrastructure.
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define MODES_LEVELS_FN __host__ __device__ __forceinline__
#else
#define MODES_LEVELS_FN static inline
#endif

namespace modes {
namespace levels {

// One thread's partial sums.  sum_mag fits in 32 bits for up to 65 909 samples (2^32 / 65167).
struct Acc {
    uint32_t sum_mag;
    uint32_t peak;
    uint32_t clipped;
    uint64_t sum_power;
};

MODES_LEVELS_FN void acc_clear(Acc &a) { a.sum_mag = 0; a.peak = 0; a.clipped = 0; a.sum_power = 0; }

// |byte - 127| of the four bytes of a word.
MODES_LEVELS_FN uint32_t absdiff127x4(uint32_t w) {
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
MODES_LEVELS_FN uint32_t dot4(uint32_t a, uint32_t b) {
#if defined(__CUDA_ARCH__)
    return __dp4a(a, b, 0u);
#else
    uint32_t c = 0;
    for (int k = 0; k < 4; k++) c += ((a >> (8 * k)) & 0xff) * ((b >> (8 * k)) & 0xff);
    return c;
#endif
}

MODES_LEVELS_FN void add_sample(Acc &a, uint32_t m) {
    a.sum_mag += m;
    a.sum_power += (uint64_t)m * m;
    a.peak = m > a.peak ? m : a.peak;
}

// The two samples of word w.  Returns a non-zero mask when a byte may be clipped (0, 254 or 255):
// the caller then counts the word with clipped_in().  |b - 127| <= 128, so adding 1 per byte never
// carries into the next byte, and bit 7 of a byte is set exactly when |b - 127| >= 127.
MODES_LEVELS_FN uint32_t add_word(Acc &a, uint32_t w, const uint16_t *lut) {
    const uint32_t d = absdiff127x4(w);
    add_sample(a, lut[dot4(d & 0x0000ffffu, d)]);
    add_sample(a, lut[dot4(d & 0xffff0000u, d)]);
    return (d + 0x01010101u) & 0x80808080u;
}

// Samples of word w with an I or Q byte at a rail (0 or 255): 0, 1 or 2.
MODES_LEVELS_FN uint32_t clipped_in(uint32_t w) {
    uint32_t n = 0;
    for (int s = 0; s < 2; s++) {
        const uint32_t i = (w >> (16 * s)) & 0xff, q = (w >> (16 * s + 8)) & 0xff;
        n += (i == 0 || i == 255 || q == 0 || q == 255) ? 1u : 0u;
    }
    return n;
}

// Four words (one 16-byte load): eight samples.
MODES_LEVELS_FN void add_quad(Acc &a, uint32_t x, uint32_t y, uint32_t z, uint32_t w, const uint16_t *lut) {
    const uint32_t maybe = add_word(a, x, lut) | add_word(a, y, lut) | add_word(a, z, lut) | add_word(a, w, lut);
    if (maybe) a.clipped += clipped_in(x) + clipped_in(y) + clipped_in(z) + clipped_in(w);
}

}  // namespace levels
}  // namespace modes
