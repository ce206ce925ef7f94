// modes_scan_core.cuh — the arithmetic of the preamble scan (K1), one lane's share of one row.
//
// Replaces, for 32 consecutive positions at a time, computeMagnitudeVector (dump1090.c:1454-1469)
// and the ten comparisons of detectModeS (dump1090.c:1602-1611).  scan2_kernel (modes_scan2.cu)
// wraps it with the loads, the cross-lane lookahead and the per-tile survivor stage.
//
// Like modes_eval_serial.cuh the file needs nothing from CUDA but a few integer intrinsics, so the
// test suite also compiles it for the host (tests/host_shim/scan_core_host.cpp) and checks the
// masks against a plain restatement of the ten comparisons.  That build is test infrastructure.
//
// Exactness.  The reference compares magnitudes m = round(360*sqrt(n)), n = i*i + q*q with
// i,q in [0,128]; m is strictly increasing over the reachable n, so the comparisons are decided
// on n.  n is held as 15-bit fields, two per register (n = 32768 clamps to 32767, which no other
// sample reaches: 32767 = 3 mod 4 is not a sum of two squares).
//
// Pipe balance.  An sm_90 scheduler issues one instruction per cycle, but the integer ALU pipe
// and the FMA pipe each take a warp instruction every second cycle: the loop only runs at the
// issue rate if its instructions split evenly between the two.  The packed comparison
// "L + 0x7fff - R has bit 15 set <=> L > R" is therefore written as a multiply-add with operands
// the compiler cannot see through ((L + 0x7fff) - R = R * 0xffffffff + LK, one IMAD), the biased
// copies LK = L + 0x7fff are IMADs as well, and the pass flags are gathered by byte dot products
// (IDP4A, FMA pipe) instead of shifts and masks.
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define MODES_SCAN_FN __device__ __forceinline__
#else
#define MODES_SCAN_FN static inline
#endif

namespace modes {
namespace scan2 {

constexpr uint32_t kK15 = 0x7fff7fffu;
constexpr int kLaneWords = 16;          // 32 samples = 16 packed words per lane and row
constexpr int kLookWords = 5;           // words of the next lane a lane's last positions reach into

#if defined(__CUDA_ARCH__)
MODES_SCAN_FN uint32_t absdiff127x4(uint32_t w) { return __vabsdiffu4(w, 0x7f7f7f7fu); }
MODES_SCAN_FN uint32_t dot4(uint32_t a, uint32_t b, uint32_t c) { return __dp4a(a, b, c); }
MODES_SCAN_FN uint32_t min2(uint32_t a, uint32_t b) { return __vminu2(a, b); }
MODES_SCAN_FN uint32_t max2(uint32_t a, uint32_t b) { return __vmaxu2(a, b); }
MODES_SCAN_FN uint32_t max2x3(uint32_t a, uint32_t b, uint32_t c) { return __vimax3_u16x2(a, b, c); }
MODES_SCAN_FN uint32_t odd_pair(uint32_t lo, uint32_t hi) { return __byte_perm(lo, hi, 0x5432); }
// a * b + c as one multiply-add (b comes from a kernel parameter: the compiler cannot fold it into an add)
MODES_SCAN_FN uint32_t mad(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t d;
    asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}
#else
MODES_SCAN_FN uint32_t absdiff127x4(uint32_t w) {
    uint32_t r = 0;
    for (int k = 0; k < 4; k++) {
        int b = (int)((w >> (8 * k)) & 0xff) - 127;
        r |= (uint32_t)(b < 0 ? -b : b) << (8 * k);
    }
    return r;
}
MODES_SCAN_FN uint32_t dot4(uint32_t a, uint32_t b, uint32_t c) {
    for (int k = 0; k < 4; k++) c += ((a >> (8 * k)) & 0xff) * ((b >> (8 * k)) & 0xff);
    return c;
}
MODES_SCAN_FN uint32_t min2(uint32_t a, uint32_t b) {
    const uint32_t al = a & 0xffffu, bl = b & 0xffffu, ah = a >> 16, bh = b >> 16;
    return (al < bl ? al : bl) | ((ah < bh ? ah : bh) << 16);
}
MODES_SCAN_FN uint32_t max2(uint32_t a, uint32_t b) {
    const uint32_t al = a & 0xffffu, bl = b & 0xffffu, ah = a >> 16, bh = b >> 16;
    return (al > bl ? al : bl) | ((ah > bh ? ah : bh) << 16);
}
MODES_SCAN_FN uint32_t max2x3(uint32_t a, uint32_t b, uint32_t c) { return max2(max2(a, b), c); }
MODES_SCAN_FN uint32_t odd_pair(uint32_t lo, uint32_t hi) { return (lo >> 16) | (hi << 16); }
MODES_SCAN_FN uint32_t mad(uint32_t a, uint32_t b, uint32_t c) { return a * b + c; }
#endif

// Two I/Q pairs (I0,Q0,I1,Q1) -> their squared magnitudes as 15-bit fields, first sample low.
//   nt = n0 + n1,  n1 * 65535 + nt = n0 + (n1 << 16)
MODES_SCAN_FN uint32_t npack(uint32_t raw) {
    const uint32_t a = absdiff127x4(raw);
    const uint32_t nt = dot4(a, a, 0u);
    const uint32_t n1 = dot4(a, a & 0xffff0000u, 0u);
    return min2(n1 * 65535u + nt, kK15);
}

// Weights that put the pass flags of pair q (bit 15 = even position, bit 31 = odd position of a
// masked comparison word) at bits 2q, 2q+1 of a byte scaled by 128.
MODES_SCAN_FN constexpr uint32_t flag_weights(int q) { return (1u << (8 + 2 * q)) | (1u << (24 + 2 * q + 1)); }

// The ten comparisons of dump1090.c:1602-1611 for the 32 positions whose first samples are the
// halves of P[0..15]; P[16..20] are the next five words of the stream.  Bit p of the result:
// position p passes.  With m_d = sample p+d the comparisons are
//     min(m0,m2) > max(m1,m3)      m0 > max(m4,m5,m6)      m9 > max(m6,m8)      m7 > m8
// `one` = 1 and `minus_one` = 0xffffffff must be values the compiler cannot see (kernel parameters).
MODES_SCAN_FN uint32_t row_mask(const uint32_t P[kLaneWords + kLookWords], uint32_t one, uint32_t minus_one) {
    uint32_t S[20], PK[17], SK[20];
#pragma unroll
    for (int k = 0; k < 20; k++) S[k] = odd_pair(P[k], P[k + 1]);          // samples (2k+1, 2k+2)
#pragma unroll
    for (int k = 0; k < 17; k++) PK[k] = mad(P[k], one, kK15);
#pragma unroll
    for (int k = 3; k < 20; k++) SK[k] = mad(S[k], one, kK15);
    uint32_t acc[4] = {0u, 0u, 0u, 0u};
#pragma unroll
    for (int u = 0; u < 16; u++) {
        const uint32_t AK = min2(PK[u], PK[u + 1]);                        // min(m0, m2) + K
        const uint32_t B = max2(S[u], S[u + 1]);                           // max(m1, m3)
        const uint32_t W = max2x3(P[u + 2], S[u + 2], P[u + 3]);           // max(m4, m5, m6)
        const uint32_t E = max2(P[u + 3], P[u + 4]);                       // max(m6, m8)
        // L + K - R per 16-bit half: bit 15 set <=> L > R; no borrow or carry between the halves
        const uint32_t D1 = mad(B, minus_one, AK);
        const uint32_t D2 = mad(W, minus_one, PK[u]);
        const uint32_t D3 = mad(E, minus_one, SK[u + 4]);                  // m9 - max(m6, m8)
        const uint32_t D4 = mad(P[u + 4], minus_one, SK[u + 3]);           // m7 - m8
        const uint32_t T = (D1 & D2 & D3) & (D4 & 0x80008000u);
        acc[u >> 2] = dot4(T, flag_weights(u & 3), acc[u >> 2]);
    }
    return (acc[0] >> 7) | (acc[1] << 1) | (acc[2] << 9) | (acc[3] << 17);
}


// ---- two rows per register --------------------------------------------------------------------
// The same arithmetic with the two 16-bit halves of a register holding the same sample of two
// DIFFERENT rows (row A low, row B high) instead of two neighbouring samples of one row: every
// operand of a position is then a whole register (no odd-aligned copies to build: one PRMT and one
// bias less per position pair), and the per-step overhead is paid once for 64 positions.
constexpr int kPairLook = 9;             // registers of the next lane a lane's last positions reach into

// One 32-bit word of each row (two I/Q pairs each) -> X0 = (nA0, nB0), X1 = (nA1, nB1).
// `c65536` = 65536 as a value the compiler cannot see (keeps the packing on the FMA pipe).
MODES_SCAN_FN void npack2(uint32_t rawA, uint32_t rawB, uint32_t c65536, uint32_t minus_one, uint32_t &X0, uint32_t &X1) {
    const uint32_t aA = absdiff127x4(rawA), aB = absdiff127x4(rawB);
    const uint32_t nA0 = dot4(aA, aA & 0xffffu, 0u), nB0 = dot4(aB, aB & 0xffffu, 0u);
    const uint32_t ntA = dot4(aA, aA, 0u), ntB = dot4(aB, aB, 0u);
    const uint32_t x0 = mad(nB0, c65536, nA0);
    const uint32_t nt = mad(ntB, c65536, ntA);
    const uint32_t x1 = mad(x0, minus_one, nt);                          // (nA1, nB1) = totals - first samples
    X0 = min2(x0, kK15); X1 = min2(x1, kK15);
}

// Weights that put the flags of position k (bit 15 = row A, bit 31 = row B of a masked comparison
// word) at bits q and 4+q (q = k & 3) of a byte scaled by 128.
MODES_SCAN_FN constexpr uint32_t pair_weights(int q) { return (1u << (8 + q)) | (1u << (24 + 4 + q)); }

// Positions K0 .. K1-1 of the comparison; accumulates the flags into acc[k / 4].
template <int K0, int K1>
MODES_SCAN_FN void rows2_compare(const uint32_t X[32 + kPairLook], uint32_t one, uint32_t minus_one, uint32_t acc[8]) {
    uint32_t XK[32 + kPairLook];
#pragma unroll
    for (int k = K0; k < K1 + kPairLook; k++) XK[k] = mad(X[k], one, kK15);
#pragma unroll
    for (int k = K0; k < K1; k++) {
        const uint32_t AK = min2(XK[k], XK[k + 2]);                        // min(m0, m2) + K
        const uint32_t B = max2(X[k + 1], X[k + 3]);                       // max(m1, m3)
        const uint32_t W = max2x3(X[k + 4], X[k + 5], X[k + 6]);           // max(m4, m5, m6)
        const uint32_t E = max2(X[k + 6], X[k + 8]);                       // max(m6, m8)
        const uint32_t D1 = mad(B, minus_one, AK);
        const uint32_t D2 = mad(W, minus_one, XK[k]);
        const uint32_t D3 = mad(E, minus_one, XK[k + 9]);                  // m9 - max(m6, m8)
        const uint32_t D4 = mad(X[k + 8], minus_one, XK[k + 7]);           // m7 - m8
        const uint32_t T = (D1 & D2 & D3) & (D4 & 0x80008000u);
        acc[k >> 2] = dot4(T, pair_weights(k & 3), acc[k >> 2]);
    }
}

// The accumulated flags -> outA / outB: bit p = position p of row A / row B passes.
MODES_SCAN_FN void rows2_finish(const uint32_t acc[8], uint32_t &outA, uint32_t &outB) {
    // byte b of m_j = (row B flags of positions 16j+4b..+3) << 4 | (row A flags of the same positions)
    const uint32_t m0 = (acc[0] >> 7) | (acc[1] << 1) | (acc[2] << 9) | (acc[3] << 17);
    const uint32_t m1 = (acc[4] >> 7) | (acc[5] << 1) | (acc[6] << 9) | (acc[7] << 17);
    // nibbles -> two 32-bit masks
    uint32_t a0 = m0 & 0x0f0f0f0fu, a1 = m1 & 0x0f0f0f0fu, b0 = (m0 >> 4) & 0x0f0f0f0fu, b1 = (m1 >> 4) & 0x0f0f0f0fu;
    a0 = (a0 | (a0 >> 4)) & 0x00ff00ffu; a1 = (a1 | (a1 >> 4)) & 0x00ff00ffu;
    b0 = (b0 | (b0 >> 4)) & 0x00ff00ffu; b1 = (b1 | (b1 >> 4)) & 0x00ff00ffu;
    a0 = (a0 | (a0 >> 8)) & 0xffffu; a1 = (a1 | (a1 >> 8)) & 0xffffu;
    b0 = (b0 | (b0 >> 8)) & 0xffffu; b1 = (b1 | (b1 >> 8)) & 0xffffu;
    outA = a0 | (a1 << 16);
    outB = b0 | (b1 << 16);
}

// The ten comparisons for positions 0..31 of both rows; X[0..31] = the lane's samples, X[32..40] =
// the next nine.
MODES_SCAN_FN void rows2_mask(const uint32_t X[32 + kPairLook], uint32_t one, uint32_t minus_one, uint32_t &outA, uint32_t &outB) {
    uint32_t acc[8] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
    rows2_compare<0, 32>(X, one, minus_one, acc);
    rows2_finish(acc, outA, outB);
}

}  // namespace scan2
}  // namespace modes
