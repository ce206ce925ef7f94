// modes_arrival_core.cuh — the arithmetic of the arrival-time measurement (modes_set_arrival,
// definition in include/modes_b200.h), run by the signal pass's kernel (modes_signal.cu).
//
// Window samples are numbered relative to the attempt's position j.  The frame's bits are held as
// four words, word r bit l = frame bit 32r + l (bits >= b cleared).  Bit i owns the samples 16+2i
// (first) and 17+2i (second); with e[16+2i] = bit i, e[17+2i] = !bit i, e[15] = 0 and e[16+2b] = 0,
// the classes of a bit's samples depend on bit i-1, bit i and bit i+1 only:
//     first  sample: (!bit i-1, bit i, !bit i)   main  when bit i and (i == 0 or bit i-1)
//                                                 early when !bit i and (i == 0 or bit i-1)
//     second sample: (bit i, !bit i, bit i+1)     late  when bit i and !bit i+1 (bit b reads 0)
//                                                 main  when !bit i and !bit i+1
// so the four class masks of 32 bits are word operations.  The samples outside the bit pairs are
// the preamble's 1..15 (fixed classes, except 15: early when bit 0 is 1, quiet otherwise) and 16+2b
// (late when bit b-1 is 0, quiet otherwise).
//
// Like modes_signal_core.cuh the file needs nothing from CUDA but a few integer intrinsics, so the test
// suite also compiles it for the host (tests/host_shim/arrival_core_host.cpp) and checks it against a
// plain restatement of the definition.  That build is test infrastructure.
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define MODES_ARRIVAL_FN __host__ __device__ __forceinline__
#else
#define MODES_ARRIVAL_FN static inline
#endif

namespace modes {
namespace arrival {

enum { kMain = 0, kLate = 1, kEarly = 2, kQuiet = 3, kUnused = 4 };

MODES_ARRIVAL_FN uint32_t brev32(uint32_t x) {
#if defined(__CUDA_ARCH__)
    return __brev(x);
#else
    uint32_t r = 0;
    for (int k = 0; k < 32; k++) r |= ((x >> k) & 1u) << (31 - k);
    return r;
#endif
}

MODES_ARRIVAL_FN uint32_t popc32(uint32_t x) {
#if defined(__CUDA_ARCH__)
    return (uint32_t)__popc(x);
#else
    return (uint32_t)__builtin_popcount(x);
#endif
}

// The frame bits of msg bytes 0..15 held as four little-endian words (as in modes_frame_eval), with
// the bits from b on cleared.
MODES_ARRIVAL_FN void bit_words(const uint32_t msg_w[4], uint32_t b, uint32_t B[4]) {
    for (int r = 0; r < 4; r++) {
        const uint32_t w = msg_w[r];
        const uint32_t be = (w >> 24) | ((w >> 8) & 0xff00u) | ((w << 8) & 0xff0000u) | (w << 24);   // byte 4r first
        B[r] = brev32(be);                                                                          // bit 32r + l at l
    }
    if (b == 56) { B[1] &= 0x00ffffffu; B[2] = 0; B[3] = 0; }
    else B[3] &= 0x0000ffffu;
}

// Class masks of bits 32r .. 32r+31 (bit l of each mask = bit 32r + l).
struct PairClasses { uint32_t main1, early1, main2, late2; };

MODES_ARRIVAL_FN PairClasses pair_classes(const uint32_t B[4], int r, uint32_t b) {
    const uint32_t cur = B[r];
    const uint32_t prev = (cur << 1) | (r ? B[r - 1] >> 31 : 1u);         // bit i-1; "1" before bit 0 (e[15] = 0)
    const uint32_t next = (cur >> 1) | (r < 3 ? B[r + 1] << 31 : 0u);     // bit i+1; 0 from bit b on (e[16+2b] = 0)
    const int left = (int)b - 32 * r;
    const uint32_t valid = left >= 32 ? 0xffffffffu : (left <= 0 ? 0u : (1u << left) - 1u);
    PairClasses c;
    c.main1 = cur & prev & valid;
    c.early1 = ~cur & prev & valid;
    c.late2 = cur & ~next & valid;
    c.main2 = ~cur & ~next & valid;
    return c;
}

// The class of window sample s in 1..15 (the preamble) or s == 16 + 2b; bit0 = frame bit 0, last = bit b-1.
MODES_ARRIVAL_FN uint32_t edge_class(uint32_t s, uint32_t b, uint32_t bit0, uint32_t last) {
    if (s == 16 + 2 * b) return last ? kQuiet : kLate;
    switch (s) {
    case 2: case 7: case 9: return kMain;
    case 3: case 10: return kLate;
    case 6: return kEarly;
    case 4: case 5: case 11: case 12: case 13: case 14: return kQuiet;
    case 15: return bit0 ? kEarly : kQuiet;
    default: return kUnused;                                           // 0 (outside), 1 and 8: (1,0,1)
    }
}

// The class counts: the preamble's and sample 16+2b's, plus the popcounts of the pair masks.
MODES_ARRIVAL_FN void class_counts(const uint32_t B[4], uint32_t b, uint32_t n[4]) {
    const uint32_t bit0 = B[0] & 1u, last = (B[(b - 1) >> 5] >> ((b - 1) & 31)) & 1u;
    n[kMain] = 3; n[kLate] = 2 + (last ^ 1u); n[kEarly] = 1 + bit0; n[kQuiet] = 6 + (bit0 ^ 1u) + last;
    for (int r = 0; r < 4; r++) {
        const PairClasses c = pair_classes(B, r, b);
        n[kMain] += popc32(c.main1) + popc32(c.main2);
        n[kLate] += popc32(c.late2);
        n[kEarly] += popc32(c.early1);
    }
}

// The code (0 = not measured, else offset + 8) from the class sums S and counts n (every n >= 1,
// n <= 241 and S <= 241 * 65167).  With D = n_main n_late n_early n_quiet > 0, the three terms
// scaled by D are
//     A D = (S_main n_quiet - S_quiet n_main) n_late n_early
//     L D = max(S_late n_quiet - S_quiet n_late, 0) n_main n_early
//     E D = max(S_early n_quiet - S_quiet n_early, 0) n_main n_late
// (each below 2^48), and the offset is the number of k in 1..7 with 2 |6 (L - E)| >= (2k - 1)(A + L + E),
// signed: round half away from zero, clamped to 7.
MODES_ARRIVAL_FN uint32_t code_of(const uint32_t S[4], const uint32_t n[4]) {
    const int64_t sq = S[kQuiet], nq = n[kQuiet];
    const int64_t dm = (int64_t)S[kMain] * nq - sq * n[kMain];
    int64_t dl = (int64_t)S[kLate] * nq - sq * n[kLate];
    int64_t de = (int64_t)S[kEarly] * nq - sq * n[kEarly];
    if (dl < 0) dl = 0;
    if (de < 0) de = 0;
    const int64_t a = dm * n[kLate] * n[kEarly], l = dl * n[kMain] * n[kEarly], e = de * n[kMain] * n[kLate];
    const int64_t den = a + l + e;
    if (den <= 0) return 0;
    const int64_t num = 6 * (l - e);
    const int64_t twice = 2 * (num < 0 ? -num : num);
    uint32_t q = 0;
    for (int k = 1; k <= 7; k++) q += twice >= (2 * k - 1) * den ? 1u : 0u;
    return num < 0 ? 8u - q : 8u + q;
}

}  // namespace arrival
}  // namespace modes
