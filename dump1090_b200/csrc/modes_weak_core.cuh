// modes_weak_core.cuh — the arithmetic of the weak-preamble scan (modes_weak.cu); the definition is
// in include/modes_b200.h (modes_set_weak_preambles).
//
// A position's window is the magnitudes m[j .. j+25] (m = lutn[I^2 + Q^2], the reference's magnitude,
// dump1090.c:359-364).  Conditions 1 and 2 (pulse shape and pulse/quiet contrast) are the cheap part
// and reject almost every position; conditions 3 (hard DF 17/18) and 4 (the reference's test fails)
// are only evaluated for the survivors.  All arithmetic is on integers: 7 * 4 * 65167 and
// 8 * 7 * 65167 fit in 32 bits.
//
// Like modes_levels_core.cuh the file needs nothing from CUDA but a few integer intrinsics, so the
// test suite also compiles it for the host (tests/host_shim/weak_core_host.cpp) and checks it against
// a numpy restatement of the definition.  That build is test infrastructure.
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define MODES_WEAK_FN __host__ __device__ __forceinline__
#else
#define MODES_WEAK_FN static inline
#endif

namespace modes {
namespace weak {

constexpr int kWindow = 26;                          // samples m[j .. j+25] one position reads

// |byte - 127| of the four bytes of a word (I0 Q0 I1 Q1: two samples).
MODES_WEAK_FN uint32_t absdiff127x4(uint32_t w) {
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

MODES_WEAK_FN uint32_t dot4(uint32_t a, uint32_t b) {
#if defined(__CUDA_ARCH__)
    return __dp4a(a, b, 0u);
#else
    uint32_t c = 0;
    for (int k = 0; k < 4; k++) c += ((a >> (8 * k)) & 0xff) * ((b >> (8 * k)) & 0xff);
    return c;
#endif
}

// The magnitudes of the two samples of word w, packed: first sample in the low half.
MODES_WEAK_FN uint32_t word_mags(uint32_t w, const uint16_t *lut) {
    const uint32_t d = absdiff127x4(w);
    return (uint32_t)lut[dot4(d & 0x0000ffffu, d)] | ((uint32_t)lut[dot4(d & 0xffff0000u, d)] << 16);
}

// Conditions 1 and 2 for the window starting at m[o].
template <class M>
MODES_WEAK_FN bool shape_and_contrast(const M &m, int o) {
    const uint32_t m0 = m[o], m1 = m[o + 1], m2 = m[o + 2], m7 = m[o + 7], m8 = m[o + 8], m9 = m[o + 9];
    const uint32_t quiet = (uint32_t)m[o + 4] + m[o + 5] + m[o + 6] + m[o + 11] + m[o + 12] + m[o + 13] + m[o + 14];
    return (m0 > m1) & (m2 > m1) & (m7 > m8) & (m9 > m8) & (7u * (m0 + m2 + m7 + m9) > 8u * quiet);
}

// Condition 3: the hard DF, b_i = m[16+2i] > m[17+2i], is 17 or 18.
template <class M>
MODES_WEAK_FN bool df_17_18(const M &m, int o) {
    uint32_t df = 0;
    for (int i = 0; i < 5; i++) df = (df << 1) | ((uint32_t)m[o + 16 + 2 * i] > (uint32_t)m[o + 17 + 2 * i] ? 1u : 0u);
    return df == 17 || df == 18;
}

// The reference's preamble test, dump1090.c:1602-1650: the ten comparisons and the "high" tests.
template <class M>
MODES_WEAK_FN bool reference_preamble(const M &m, int o) {
    const uint32_t m0 = m[o], m1 = m[o + 1], m2 = m[o + 2], m3 = m[o + 3], m4 = m[o + 4], m5 = m[o + 5], m6 = m[o + 6];
    const uint32_t m7 = m[o + 7], m8 = m[o + 8], m9 = m[o + 9];
    if (!(m0 > m1 && m1 < m2 && m2 > m3 && m3 < m0 && m4 < m0 && m5 < m0 && m6 < m0 && m7 > m8 && m8 < m9 && m9 > m6))
        return false;
    const uint32_t high = (m0 + m2 + m7 + m9) / 6;
    return m4 < high && m5 < high && (uint32_t)m[o + 11] < high && (uint32_t)m[o + 12] < high && (uint32_t)m[o + 13] < high &&
           (uint32_t)m[o + 14] < high;
}

// Conditions 3 and 4, for a window that passed conditions 1 and 2.
template <class M>
MODES_WEAK_FN bool weak_rest(const M &m, int o) {
    return df_17_18(m, o) && !reference_preamble(m, o);
}

template <class M>
MODES_WEAK_FN bool weak_preamble(const M &m, int o) {
    return shape_and_contrast(m, o) && weak_rest(m, o);
}

}  // namespace weak
}  // namespace modes
