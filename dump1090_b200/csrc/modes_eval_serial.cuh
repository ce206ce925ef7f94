// modes_eval_serial.cuh — evaluation of ONE preamble candidate by ONE thread.
//
// This is the body of detectModeS after the preamble test (dump1090.c:1653-1735: bit slicing, delta
// gate, the phase-corrected retry of :1498-1558) and the order-independent half of
// decodeModesMessage (:1099-1128: CRC syndrome, single/two-bit repair), written as straight
// sequential code over the candidate's 241-sample window, in two formulations: namespace `fused`
// (at the end of the file: both attempts in ONE walk; eval_fused_kernel, modes_eval_fused.cu, the
// default) and `evaluate` (two passes; eval_serial_kernel, modes_kernels.cu).  Both run with lane =
// candidate, the 32 windows of a warp staged in shared memory.
//
// The file has no CUDA dependencies besides a few integer intrinsics, so the test suite also
// compiles it for the host (tests/host_shim/) and checks the logic against the oracle without a
// GPU.  That build is test infrastructure; the product library contains only the device code.
#pragma once
#include <cstdint>
#include "modes_b200.h"

#if defined(__CUDACC__)
#define MODES_SERIAL_FN __device__ __forceinline__
#else
#define MODES_SERIAL_FN static inline
#endif

namespace modes {
namespace serial {

// ---- the intrinsics ----------------------------------------------------------------------
#if defined(__CUDA_ARCH__)
MODES_SERIAL_FN uint32_t absdiff127x4(uint32_t w) { return __vabsdiffu4(w, 0x7f7f7f7fu); }
MODES_SERIAL_FN uint32_t dot4(uint32_t a, uint32_t b) { return __dp4a(a, b, 0u); }
MODES_SERIAL_FN uint32_t bitrev(uint32_t x) { return __brev(x); }
// (hi:lo) >> s for s in {16, 32}
MODES_SERIAL_FN uint32_t funnel(uint32_t lo, uint32_t hi, uint32_t s) { return __funnelshift_rc(lo, hi, s); }
MODES_SERIAL_FN uint32_t bswap(uint32_t x) { return __byte_perm(x, 0u, 0x0123u); }
MODES_SERIAL_FN uint32_t absdiff_add(uint32_t a, uint32_t b, uint32_t c) { return __usad(a, b, c); }   // |a-b| + c
MODES_SERIAL_FN uint32_t perm(uint32_t x, uint32_t sel) { return __byte_perm(x, 0u, sel); }             // bytes of x picked by sel's nibbles
MODES_SERIAL_FN uint32_t opaque(uint32_t x) { asm volatile("" : "+r"(x)); return x; }                    // keep a value in its register
#else
MODES_SERIAL_FN uint32_t bswap(uint32_t x) { return (x >> 24) | ((x >> 8) & 0xff00u) | ((x << 8) & 0xff0000u) | (x << 24); }
MODES_SERIAL_FN uint32_t absdiff_add(uint32_t a, uint32_t b, uint32_t c) { return (a > b ? a - b : b - a) + c; }
MODES_SERIAL_FN uint32_t perm(uint32_t x, uint32_t sel) {
    uint32_t r = 0;
    for (int k = 0; k < 4; k++) {
        const uint32_t n = (sel >> (4 * k)) & 7u;
        r |= (n < 4 ? (x >> (8 * n)) & 0xffu : 0u) << (8 * k);
    }
    return r;
}
MODES_SERIAL_FN uint32_t opaque(uint32_t x) { return x; }
MODES_SERIAL_FN uint32_t absdiff127x4(uint32_t w) {
    uint32_t r = 0;
    for (int k = 0; k < 4; k++) {
        int b = (int)((w >> (8 * k)) & 0xff) - 127;
        r |= (uint32_t)(b < 0 ? -b : b) << (8 * k);
    }
    return r;
}
MODES_SERIAL_FN uint32_t dot4(uint32_t a, uint32_t b) {
    uint32_t r = 0;
    for (int k = 0; k < 4; k++) r += ((a >> (8 * k)) & 0xff) * ((b >> (8 * k)) & 0xff);
    return r;
}
MODES_SERIAL_FN uint32_t bitrev(uint32_t x) {
    uint32_t r = 0;
    for (int k = 0; k < 32; k++) r |= ((x >> k) & 1u) << (31 - k);
    return r;
}
MODES_SERIAL_FN uint32_t funnel(uint32_t lo, uint32_t hi, uint32_t s) {
    return s >= 32 ? hi : (uint32_t)((((uint64_t)hi << 32) | lo) >> s);
}
#endif

// ---- window layout ----------------------------------------------------------------------------
// A candidate at virtual position v owns the samples m[-1..239] = virtual samples v-1 .. v+239.
// They are staged as kWindowWords aligned 32-bit words (two samples each); `odd` says whether
// m[-1] is the high half of word 0.  Window sample w (w = 0 is m[-1]) is halfword w + odd.
// Bit b of the frame is the sample pair (m[16+2b], m[17+2b]) = window samples 17+2b, 18+2b, i.e.
// halfwords of words 8+b and 9+b.  After the first pass word 8+b holds the pair's magnitudes
// (first | second << 16) instead; words 0..7 keep the raw preamble samples.
constexpr int kWindowWords = 121;

// Rows of the (|I-127|, |Q-127|) magnitude table are 136 entries (68 words) apart: consecutive rows
// start 4 banks apart in shared memory, so the small amplitudes that most half-bit samples have
// (|I-127|, |Q-127| < 8) spread over all 32 banks instead of piling onto two or three.
constexpr int kIqLutStride = 136;
constexpr int kIqLutEntries = 129 * kIqLutStride;

struct Tables {
    const uint16_t *lut_iq;      // [129 rows of kIqLutStride] magnitude by (|I-127|, |Q-127|): round(sqrt(i*i+q*q)*360), dump1090.c:362
    const uint32_t *bit_syn;     // [112]   syndrome of one flipped bit
    const uint32_t *nib_syn;     // [28*16] syndrome of nibble value x at frame nibble i: XOR of bit_syn over its set bits
    const uint32_t *fix_hash;    // [256]   inverse of bit_syn over positions 5..111
    const uint32_t *pair_hash;   // [1 << kPairHashBits] syndrome of two flipped bits p < q -> p (global memory on the device)
};
constexpr int kPairHashBits = 14, kPairHashMaxProbe = 16;

// First flipped bit p of the two-bit pattern with syndrome s, or -1.
MODES_SERIAL_FN int pair_first(const uint32_t *pair_hash, uint32_t s) {
    const uint32_t h = (s * 0x9E3779B1u) >> (32 - kPairHashBits);
    for (int i = 0; i < kPairHashMaxProbe; i++) {
        const uint32_t e = pair_hash[(h + i) & ((1u << kPairHashBits) - 1u)];
        if (e == 0xFFFFFFFFu) return -1;
        if ((e >> 7) == s) return (int)(e & 0x7f);
    }
    return -1;
}

// Index into lut_iq of the sample held in the low (kLutLow) or high (kLutHigh) half of a word of
// |byte - 127| values: kIqLutStride * |I-127| + |Q-127| as one byte dot product.
constexpr uint32_t kLutLow = (uint32_t)kIqLutStride | 0x100u, kLutHigh = kLutLow << 16;

// What one attempt (uncorrected, or phase corrected) yields: the six 32-bit words of a
// modes_frame_eval (include/modes_b200.h) are made from it by eval_words().
struct Verdict {
    uint32_t F[4];               // frame bits, bit b of the frame at bit b (LSB first); after repair
    uint32_t msgtype, flags, errorbit, nfixed, crc;
};

// Entry (pos, value) of Tables::nib_syn from the bit syndromes: bit 3-k of the nibble is frame bit 4*pos+k.
MODES_SERIAL_FN uint32_t nibble_syndrome(const uint32_t *bit_syn, int pos, uint32_t value) {
    uint32_t x = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) x ^= ((value >> (3 - k)) & 1u) ? bit_syn[4 * pos + k] : 0u;
    return x;
}

MODES_SERIAL_FN uint32_t fix_hash_of(uint32_t s) { return (s * 0x9E3779B1u) >> 24; }

// Position (5..111) whose single-bit syndrome is s, or -1.
MODES_SERIAL_FN int syndrome_pos(const uint32_t *fix_hash, uint32_t s) {
    uint32_t h = fix_hash_of(s);
    for (int i = 0; i < 256; i++) {
        uint32_t e = fix_hash[(h + i) & 255u];
        if (e == 0xFFFFFFFFu) return -1;
        if ((e >> 8) == s) return (int)(e & 0xff);
    }
    return -1;
}

MODES_SERIAL_FN void flip_bit(uint32_t F[4], int b) {
    // no dynamic register indexing: four predicated XORs
    const uint32_t m = 1u << (b & 31);
    const int w = b >> 5;
    F[0] ^= (w == 0) ? m : 0u; F[1] ^= (w == 1) ? m : 0u;
    F[2] ^= (w == 2) ? m : 0u; F[3] ^= (w == 3) ? m : 0u;
}

// Frame nibble i (0..27) of F: bit 4i is its most significant bit.
MODES_SERIAL_FN uint32_t frame_nibble(const uint32_t W[4], int i) {      // W = bit-reversed F words
    const uint32_t w = (i < 8) ? W[0] : (i < 16) ? W[1] : (i < 24) ? W[2] : W[3];
    return (w >> (28 - 4 * (i & 7))) & 0xfu;
}

// CRC syndrome of the first msgbits of F, then the repairs of dump1090.c:1114-1126 (:733-742
// checksum, :854-894 fixes).  F is modified by a repair.
MODES_SERIAL_FN void crc_and_fix(uint32_t F[4], int msgbits, uint32_t msgtype, int fix_errors, int aggressive,
                                 const Tables &tab, uint32_t &crc, uint32_t &errorbit, uint32_t &nfixed) {
    const int off = 112 - msgbits;                      // a short frame uses the last 56 table positions
    const uint32_t W[4] = {bitrev(F[0]), bitrev(F[1]), bitrev(F[2]), bitrev(F[3])};
    uint32_t S = 0;
    const uint32_t *first14 = tab.nib_syn + (off >> 2) * 16;       // a short frame uses table nibbles 14..27
#pragma unroll
    for (int i = 0; i < 14; i++) S ^= first14[i * 16 + frame_nibble(W, i)];
    if (msgbits == 112) {                               // one branch, not one per nibble
#pragma unroll
        for (int i = 14; i < 28; i++) S ^= tab.nib_syn[i * 16 + frame_nibble(W, i)];
    }
    errorbit = 0xFF; nfixed = 0;
    if (S != 0 && fix_errors && (msgtype == 11 || msgtype == 17 || msgtype == 18)) {
        const int pmin = off > 5 ? off : 5;             // table positions 5..111 (dump1090.c:806)
        const int hit = syndrome_pos(tab.fix_hash, S);
        if (hit >= pmin) {
            flip_bit(F, hit - off);
            errorbit = (uint32_t)(hit - off); nfixed = 1; S = 0;
        } else if (aggressive) {
            // two flipped bits p < q (all 5671 patterns have distinct syndromes): p from the pair
            // table, q as the position whose syndrome is S ^ syn[p]; both must lie in the frame
            const int p = pair_first(tab.pair_hash, S);
            if (p >= pmin) {
                const int q = syndrome_pos(tab.fix_hash, S ^ tab.bit_syn[p]);
                flip_bit(F, p - off); flip_bit(F, q - off);
                errorbit = (uint32_t)(p - off); nfixed = 2; S = 0;
            }
        }
    }
    crc = S;
}

// One attempt after slicing: message type, delta gate (dump1090.c:1713-1726), CRC and repair.
MODES_SERIAL_FN void judge_sliced(const uint32_t Fs[4], uint32_t tri, uint32_t sum56, uint32_t sum112, int fix_errors,
                                  int aggressive, const Tables &tab, Verdict &R) {
    R.F[0] = Fs[0]; R.F[1] = Fs[1]; R.F[2] = Fs[2]; R.F[3] = Fs[3];
    R.msgtype = bitrev(Fs[0]) >> 27;
    const int msgbits = (R.msgtype >= 16 && R.msgtype <= 21) ? 112 : 56;       // dump1090.c:746-753
    const uint32_t delta = (msgbits == 112) ? sum112 / 56u : sum56 / 28u;       // :1713-1718
    R.flags = tri ? MODES_EVAL_ERRORS : 0;
    R.crc = 0; R.errorbit = 0xFF; R.nfixed = 0;
    if (delta >= 2550u) {                                                       // :1723
        R.flags |= MODES_EVAL_GATE_OK;
        if (!tri || aggressive) {                                               // :1731 (errors is 0 or 1)
            R.flags |= MODES_EVAL_DECODED;
            crc_and_fix(R.F, msgbits, R.msgtype, fix_errors, aggressive, tab, R.crc, R.errorbit, R.nfixed);
        }
    }
}

MODES_SERIAL_FN bool unconditionally_good(const Verdict &R) {
    return (R.flags & MODES_EVAL_DECODED) && R.crc == 0 && (R.msgtype == 11 || R.msgtype == 17 || R.msgtype == 18);
}

// The six 32-bit words of a modes_frame_eval as laid out in memory.
MODES_SERIAL_FN void eval_words(const Verdict &R, uint32_t w[6]) {
    const uint32_t W0 = bitrev(R.F[0]), W1 = bitrev(R.F[1]), W2 = bitrev(R.F[2]), W3 = bitrev(R.F[3]) & 0xffff0000u;
    w[0] = bswap(W0); w[1] = bswap(W1); w[2] = bswap(W2);              // big-endian words -> bytes in memory order
    w[3] = (W3 >> 24) | ((W3 >> 8) & 0xff00u) | ((R.msgtype & 0xffu) << 16) | ((R.flags & 0xffu) << 24);
    w[4] = (R.errorbit & 0xffu) | ((R.nfixed & 0xffu) << 8);
    w[5] = R.crc & 0xffffffu;
}

MODES_SERIAL_FN uint32_t scale_sample(uint32_t v, uint32_t s) {               // dump1090.c:1473-1476
    const uint32_t r = (v * s) >> 14;
    return r > 65535u ? 65535u : r;
}

// "bits[0] == 2" (dump1090.c:1681): the first pair is a tie.  The 2 is copied into every
// following indefinite bit (:1675); packed with << (7 - k%8) (:1696-1706) a 2 at bit k sets bit
// k-1 unless k starts a byte, and leaves bit k clear.  `pairs` holds the magnitude pairs.
MODES_SERIAL_FN void spread_tie(const uint32_t *pairs, uint32_t F[4]) {
    for (int k = 1; k < 112; k++) {
        const uint32_t m = pairs[k];
        int d = (int)(m & 0xffffu) - (int)(m >> 16);
        d = d < 0 ? -d : d;
        if (d >= 256) break;                             // definite: the run ends
        if (k & 7) { const int b = k - 1; const uint32_t bit = 1u << (b & 31); const int w = b >> 5;
                     F[0] |= (w == 0) ? bit : 0u; F[1] |= (w == 1) ? bit : 0u; F[2] |= (w == 2) ? bit : 0u; F[3] |= (w == 3) ? bit : 0u; }
    }
}

// OR sixteen frame bits (bits 16k .. 16k+15) into F without dynamic register indexing.
MODES_SERIAL_FN void put16(uint32_t F[4], int k, uint32_t f16) {
    const uint32_t v = f16 << ((k & 1) * 16);
    const int w = k >> 1;
    F[0] |= (w == 0) ? v : 0u; F[1] |= (w == 1) ? v : 0u;
    F[2] |= (w == 2) ? v : 0u; F[3] |= (w == 3) ? v : 0u;
}

// The three per-bit loops below handle the 112 bits as 7 blocks of 16 (the block body is
// unrolled, the block loop is not: ~50 instructions per block keeps the kernel small).

// First pass, block k: raw samples -> magnitude pairs (stored back into the window) -> sliced
// bits (dump1090.c:1667-1690); accumulates the delta sums (:1692-1693).
MODES_SERIAL_FN uint32_t first_pass_block(uint32_t *win, int k, uint32_t shift, const uint16_t *lut_iq, uint32_t &wa,
                                          uint32_t &prev, uint32_t &dsum, uint32_t &d56) {
    uint32_t f = 0;
    uint32_t *p = win + 8 + 16 * k;
#pragma unroll
    for (int i = 0; i < 16; i++) {
        const uint32_t wb = p[i + 1];
        const uint32_t a = absdiff127x4(funnel(wa, wb, shift));
        wa = wb;
        const int lo = (int)lut_iq[dot4(a, kLutLow)];
        const int hi = (int)lut_iq[dot4(a, kLutHigh)];
        p[i] = (uint32_t)lo | ((uint32_t)hi << 16);
        int d = lo - hi; d = d < 0 ? -d : d;
        dsum += (uint32_t)d;
        if (i == 7 && k == 3) d56 = dsum;                                      // bits 0..55 (:1716)
        bool definite = d >= 256;
        if (i == 0) definite = definite || k == 0;                             // bit 0 is always taken (:1675)
        prev = definite ? (uint32_t)(lo > hi) : prev;
        f |= prev << i;
    }
    return f;
}

// Phase correction (dump1090.c:1498-1558) and slicing of the corrected samples, one block of 16
// bits walking from *p in direction `step` (+1 forwards along the frame, -1 backwards): the
// half-bit sample next to the previous decision is rescaled by f_one or f_zero according to that
// decision, then the corrected pair is classified like the first pass (:1675): `d16` collects the
// definite bits, `o16` the definite ones, both in walk order.  `end0` / `end15` say that the
// first / last bit of the block is bit 0 of the frame (always definite; a tie there is the
// tri-state of :1681).
MODES_SERIAL_FN void correct_slice_block(const uint32_t *p, int step, bool fwd, bool end0, bool end15, uint32_t f_one,
                                         uint32_t f_zero, uint32_t &prev_e, uint32_t &d16, uint32_t &o16, uint32_t &tie0) {
    d16 = 0; o16 = 0;
#pragma unroll
    for (int i = 0; i < 16; i++) {
        const uint32_t m = p[i * step];
        const uint32_t lo = m & 0xffffu, hi = m >> 16;
        const uint32_t xs = scale_sample(fwd ? lo : hi, prev_e ? f_one : f_zero);
        const int nlo = (int)(fwd ? xs : lo), nhi = (int)(fwd ? hi : xs);
        prev_e = (uint32_t)(nlo > nhi);
        int d = nlo - nhi; d = d < 0 ? -d : d;
        bool definite = d >= 256;
        if (i == 0 && end0) { definite = true; tie0 = (uint32_t)(nlo == nhi); }
        if (i == 15 && end15) { definite = true; tie0 = (uint32_t)(nlo == nhi); }
        d16 |= (uint32_t)definite << i;
        o16 |= (uint32_t)(definite && nlo > nhi) << i;
    }
}

// Leaner code for the same first-pass block (|lo - hi| as one VABSDIFF; 18.7 instead of 24.6
// instructions per bit).  First pass, block k: raw samples -> magnitude pairs (stored back into the window) -> sliced
// bits (dump1090.c:1667-1690); accumulates the delta sums (:1692-1693).
MODES_SERIAL_FN uint32_t first_pass_block_lean(uint32_t *win, int k, uint32_t shift, const uint16_t *lut_iq, uint32_t &wa,
                                          uint32_t &prev, uint32_t &dsum, uint32_t &d56) {
    uint32_t f = 0;
    uint32_t *p = win + 8 + 16 * k;
#pragma unroll
    for (int i = 0; i < 16; i++) {
        const uint32_t wb = p[i + 1];
        const uint32_t a = absdiff127x4(funnel(wa, wb, shift));
        wa = wb;
        const uint32_t lo = lut_iq[dot4(a, kLutLow)];
        const uint32_t hi = lut_iq[dot4(a, kLutHigh)];
        p[i] = lo | (hi << 16);
        const uint32_t d = absdiff_add(lo, hi, 0u);
        dsum += d;
        if (i == 7 && k == 3) d56 = dsum;                                      // bits 0..55 (:1716)
        bool definite = d >= 256u;
        if (i == 0) definite = definite || k == 0;                             // bit 0 is always taken (:1675)
        prev = definite ? (uint32_t)(lo > hi) : prev;
        f |= prev << i;
    }
    return f;
}

// Leaner code for the same block (20.3 instead of 24.8 instructions per bit).
// Phase correction (dump1090.c:1498-1558) and slicing of the corrected samples, one block of 16
// bits walking from *p in direction `step` (+1 forwards along the frame, -1 backwards): the
// half-bit sample next to the previous decision is rescaled by f_one or f_zero according to that
// decision, then the corrected pair is classified like the first pass (:1675): `d16` collects the
// definite bits, `o16` the definite ones, both in walk order.  `end0` / `end15` say that the
// first / last bit of the block is bit 0 of the frame (always definite; a tie there is the
// tri-state of :1681).
//
// Written on integer masks rather than bools (all-ones = true): with sixteen unrolled steps the
// compiler otherwise shuttles the conditions between predicates and registers (7 SEL per bit).
//   sel_x / sel_y  byte selectors that extract the rescaled / the other half of a pair, zero-extended
//   dir            0 forwards, ~0 backwards;   f_pick = f_one ^ f_zero
//   not_e          ~0 unless the previous decision was "one"
MODES_SERIAL_FN void correct_slice_block_lean(const uint32_t *p, int step, uint32_t sel_x, uint32_t sel_y, uint32_t dir,
                                         bool end0, bool end15, uint32_t f_one, uint32_t f_pick, uint32_t &not_e,
                                         uint32_t &d16, uint32_t &o16, uint32_t &tie0) {
    uint32_t nd = 0, no = 0;                               // complements of d16 / o16, built by OR
#pragma unroll
    for (int i = 0; i < 16; i++) {
        const uint32_t m = p[i * step];
        const uint32_t x = perm(m, sel_x), y = perm(m, sel_y);
        const uint32_t xs = scale_sample(x, f_one ^ (not_e & f_pick));          // previous one: f_one, else f_zero
        const int32_t s = (int32_t)(xs - y);
        // "one" = first corrected sample > second: forwards s > 0, backwards s < 0.
        // u = forwards s-1, backwards ~s: one <=> u >= 0
        const int32_t u = (int32_t)(((uint32_t)s ^ dir) + ~dir);
        not_e = (uint32_t)(u >> 31);
        uint32_t not_def = (uint32_t)((int32_t)(absdiff_add(xs, y, 0u) - 256u) >> 31);   // ~0 when |delta| < 256
        if (i == 0 && end0) { not_def = 0; tie0 = (uint32_t)(s == 0); }
        if (i == 15 && end15) { not_def = 0; tie0 = (uint32_t)(s == 0); }
        nd |= not_def & (1u << i);
        no |= (not_def | not_e) & (1u << i);
    }
    d16 = ~nd & 0xffffu;
    o16 = ~no & 0xffffu;
}

// Bits with D=1 are definite and take their value from O; bits with D=0 copy the nearest
// definite bit below (:1675).  That is the carry into each bit of (O|~D) + O.  Bit 0 must be in D.
MODES_SERIAL_FN void fill_copies(const uint32_t D[4], const uint32_t O[4], uint32_t F[4]) {
    const uint64_t d0 = D[0] | ((uint64_t)D[1] << 32), d1 = D[2] | ((uint64_t)D[3] << 32);
    const uint64_t o0 = O[0] | ((uint64_t)O[1] << 32), o1 = O[2] | ((uint64_t)O[3] << 32);
    const uint64_t a0 = o0 | ~d0, a1 = o1 | ~d1;
    const uint64_t s0 = a0 + o0;
    const uint64_t s1 = a1 + o1 + (s0 < a0 ? 1ull : 0ull);
    const uint64_t ci0 = s0 ^ a0 ^ o0, ci1 = s1 ^ a1 ^ o1;                   // carry INTO each bit
    const uint64_t f0 = (ci0 >> 1) | (ci1 << 63), f1 = (ci1 >> 1) & 0x0000ffffffffffffull;
    F[0] = (uint32_t)f0; F[1] = (uint32_t)(f0 >> 32); F[2] = (uint32_t)f1; F[3] = (uint32_t)(f1 >> 32);
}

// spread_tie on the definite mask instead of the pairs: the run of indefinite bits after bit 0.
MODES_SERIAL_FN void spread_tie_mask(const uint32_t D[4], uint32_t F[4]) {
    const uint64_t t0 = ~(D[0] | ((uint64_t)D[1] << 32)) | 1ull, t1 = ~(D[2] | ((uint64_t)D[3] << 32));
    const uint64_t u0 = t0 + 1ull, u1 = t1 + (u0 == 0 ? 1ull : 0ull);
    const uint64_t run0 = t0 & ~u0, run1 = (u0 == 0) ? (t1 & ~u1) : 0ull;       // bits 0..r
    const uint64_t e0 = ((run0 >> 1) | (run1 << 63)) & 0x7f7f7f7f7f7f7f7full;
    const uint64_t e1 = (run1 >> 1) & 0x00007f7f7f7f7f7full;
    F[0] |= (uint32_t)e0; F[1] |= (uint32_t)(e0 >> 32); F[2] |= (uint32_t)e1; F[3] |= (uint32_t)(e1 >> 32);
}

MODES_SERIAL_FN uint32_t window_sample(const uint32_t *win, uint32_t odd, int w) {
    const uint32_t h = (uint32_t)w + odd;
    const uint32_t word = win[h >> 1];
    return (h & 1u) ? (word >> 16) : (word & 0xffffu);
}

MODES_SERIAL_FN uint32_t magnitude_of(const uint16_t *lut_iq, uint32_t iq) {
    return lut_iq[dot4(absdiff127x4(iq | 0x7f7f0000u), kLutLow)];
}

// Evaluate one candidate.  win: its kWindowWords staged words (modified); odd: see above;
// at_buffer_start: j == 0, where the reference retries without correcting (dump1090.c:1660);
// rec: the 12 words of pass[0] and pass[1] of its modes_candidate.
template <bool kLean>
MODES_SERIAL_FN void evaluate(uint32_t *win, uint32_t odd, bool at_buffer_start, int fix_errors, int aggressive,
                              const Tables &tab, uint32_t rec[12]) {
    const uint32_t shift = odd ? 32u : 16u;
    uint32_t F[4] = {0u, 0u, 0u, 0u};
    uint32_t prev = 0, dsum = 0, d56 = 0;
    uint32_t wa = win[8];
#pragma unroll 1
    for (int k = 0; k < 7; k++) {
        if constexpr (kLean) put16(F, k, first_pass_block_lean(win, k, shift, tab.lut_iq, wa, prev, dsum, d56));
        else put16(F, k, first_pass_block(win, k, shift, tab.lut_iq, wa, prev, dsum, d56));
    }
    const uint32_t d112 = dsum;
    uint32_t *pairs = win + 8;
    const uint32_t tri1 = (pairs[0] & 0xffffu) == (pairs[0] >> 16);
    if (tri1) spread_tie(pairs, F);

    Verdict P1, P2;
    judge_sliced(F, tri1, d56, d112, fix_errors, aggressive, tab, P1);
    P2.F[0] = P2.F[1] = P2.F[2] = P2.F[3] = 0;
    P2.msgtype = 0; P2.flags = 0; P2.errorbit = 0; P2.nfixed = 0; P2.crc = 0;

    if ((P1.flags & MODES_EVAL_GATE_OK) && !unconditionally_good(P1)) {
        P1.flags |= MODES_EVAL_P2_VALID;
        if (at_buffer_start) {
            P2 = P1;
            P2.flags &= ~(uint32_t)MODES_EVAL_P2_VALID;
        } else {
            // applyPhaseCorrection, dump1090.c:1498-1558
            const uint32_t m_1 = magnitude_of(tab.lut_iq, window_sample(win, odd, 0));
            const uint32_t m0 = magnitude_of(tab.lut_iq, window_sample(win, odd, 1));
            const uint32_t m2 = magnitude_of(tab.lut_iq, window_sample(win, odd, 3));
            const uint32_t m3 = magnitude_of(tab.lut_iq, window_sample(win, odd, 4));
            const uint32_t m6 = magnitude_of(tab.lut_iq, window_sample(win, odd, 7));
            const uint32_t m7 = magnitude_of(tab.lut_iq, window_sample(win, odd, 8));
            const uint32_t m9 = magnitude_of(tab.lut_iq, window_sample(win, odd, 10));
            const uint32_t m10 = magnitude_of(tab.lut_iq, window_sample(win, odd, 11));
            const uint32_t on_time = m0 + m2 + m7 + m9;
            const uint32_t early = (m_1 + m6) * 2u, late = (m3 + m10) * 2u;
            // early > late: walk backwards, the second half-bit samples are rescaled;
            // otherwise forwards, the first half-bit samples are.
            const bool fwd = !(early > late);
            const uint32_t lead = fwd ? late : early;
            const uint32_t q = 16384u * lead / (lead + on_time);
            const uint32_t up = (16384u + q) & 0xffffu, down = (16384u - q) & 0xffffu;
            // forwards a previous 1 scales up, backwards a following 1 scales down; the first
            // bit handled always scales up
            const uint32_t f_one = fwd ? up : down, f_zero = fwd ? down : up;
            uint32_t Dm[4] = {0u, 0u, 0u, 0u}, Om[4] = {0u, 0u, 0u, 0u}, tri2 = 0;
            if constexpr (kLean) {
                const int step = fwd ? 1 : -1;
                // forwards the first half-bit sample (low half of a pair) is rescaled, backwards the second
                const uint32_t sel_x = fwd ? 0x4410u : 0x4432u, sel_y = fwd ? 0x4432u : 0x4410u;
                const uint32_t dir = fwd ? 0u : ~0u;
                const uint32_t g_one = opaque(f_one), g_pick = opaque(f_one ^ f_zero);
                uint32_t not_e = fwd ? 0u : ~0u;               // the first bit handled always scales up
                const uint32_t *cp = fwd ? pairs : pairs + 111;
    #pragma unroll 1
                for (int k = 0; k < 7; k++, cp += 16 * step) {
                    uint32_t d16, o16;
                    correct_slice_block_lean(cp, step, sel_x, sel_y, dir, fwd && k == 0, !fwd && k == 6, g_one, g_pick, not_e, d16, o16, tri2);
                    if (!fwd) { d16 = bitrev(d16) >> 16; o16 = bitrev(o16) >> 16; }      // walk order -> frame order
                    put16(Dm, fwd ? k : 6 - k, d16);
                    put16(Om, fwd ? k : 6 - k, o16);
                }
            } else {
                uint32_t prev_e = fwd ? 1u : 0u;
                const int step = fwd ? 1 : -1;
                const uint32_t *cp = fwd ? pairs : pairs + 111;
    #pragma unroll 1
                for (int k = 0; k < 7; k++, cp += 16 * step) {
                    uint32_t d16, o16;
                    correct_slice_block(cp, step, fwd, fwd && k == 0, !fwd && k == 6, f_one, f_zero, prev_e, d16, o16, tri2);
                    if (!fwd) { d16 = bitrev(d16) >> 16; o16 = bitrev(o16) >> 16; }      // walk order -> frame order
                    put16(Dm, fwd ? k : 6 - k, d16);
                    put16(Om, fwd ? k : 6 - k, o16);
                }
            }
            uint32_t G[4];
            fill_copies(Dm, Om, G);
            if (tri2) spread_tie_mask(Dm, G);
            if (G[0] == F[0] && G[1] == F[1] && G[2] == F[2] && G[3] == F[3] && tri2 == tri1) {
                P2 = P1;                                 // same bits, same (uncorrected) delta sums: same verdict
                P2.flags &= ~(uint32_t)MODES_EVAL_P2_VALID;
            } else {
                judge_sliced(G, tri2, d56, d112, fix_errors, aggressive, tab, P2);
            }
        }
    }
    eval_words(P1, rec);
    eval_words(P2, rec + 6);
}


// ================================================================================================
// Fused single sweep (eval_fused_kernel, modes_eval_fused.cu).
//
// The first attempt and the phase-corrected retry read the same 112 sample pairs; what differs is
// a handful of integer operations per pair.  Which way the retry walks (dump1090.c:1517 / :1537)
// and its two scale factors depend only on eight preamble samples, so they are known BEFORE any
// bit is looked at.  One walk in the retry's direction therefore serves both attempts: per pair
// the two magnitudes are looked up once, the first attempt's "definite" and "greater" flags and
// the retry's "definite" and "one" flags are shifted into four mask words (the sign bit of a
// difference goes into the mask with one funnel shift), and the only serial dependency left is
// the retry's previous decision.  The copy rule of :1675 ("an indefinite bit repeats the bit
// before it") is applied afterwards on the masks (fill_copies), for both attempts and in either
// walk direction.  Nothing is written back to the window.
//
// The window is handed over in WALK ORDER: the kernel stages a backwards-walked candidate's words
// reversed, so every lane reads ascending slots and only a per-lane byte selector tells the four
// cases (direction x odd alignment) apart.
namespace fused {

#if defined(__CUDA_ARCH__)
MODES_SERIAL_FN uint32_t perm2(uint32_t a, uint32_t b, uint32_t sel) { return __byte_perm(a, b, sel); }
MODES_SERIAL_FN uint32_t push_sign(uint32_t acc, uint32_t v) { return __funnelshift_l(v, acc, 1); }   // acc << 1 | sign(v)
// The (|I-127|, |Q-127|) magnitude table in shared memory, by its 32-bit shared address: the
// entry's byte address base + 2 * (136 i + q) is two chained byte dot products (FMA pipe; the
// walk is bound by the integer ALU pipe, where "index * 2 + base" would otherwise go).
// a * b + c as one multiply-add on the FMA pipe (b is a register the compiler cannot see through)
MODES_SERIAL_FN uint32_t mad(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t d;
    asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}
struct Lut { uint32_t base; };
MODES_SERIAL_FN uint32_t lut_at(Lut l, uint32_t a, uint32_t weights) {
    const uint32_t addr = __dp4a(a, weights, __dp4a(a, weights, l.base));
    uint16_t v;
    asm("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(addr));
    return v;
}
#else
MODES_SERIAL_FN uint32_t perm2(uint32_t a, uint32_t b, uint32_t sel) {
    const uint64_t ab = ((uint64_t)b << 32) | a;
    uint32_t r = 0;
    for (int k = 0; k < 4; k++) r |= (uint32_t)((ab >> (8 * ((sel >> (4 * k)) & 7u))) & 0xffu) << (8 * k);
    return r;
}
MODES_SERIAL_FN uint32_t push_sign(uint32_t acc, uint32_t v) { return (acc << 1) | (v >> 31); }
MODES_SERIAL_FN uint32_t mad(uint32_t a, uint32_t b, uint32_t c) { return a * b + c; }
struct Lut { const uint16_t *base; };
MODES_SERIAL_FN uint32_t lut_at(Lut l, uint32_t a, uint32_t weights) { return l.base[dot4(a, weights)]; }
#endif

// A candidate's walk: slots[0] is the word the first pair starts in; step t (t = 0..111) reads
// slots[t + 1].  Forwards, slots[u] = window word 8 + u; backwards, slots[u] = window word 120 - u.
constexpr int kSlots = 113;
constexpr int kBlockBits = 28, kBlocks = 4;             // 112 bits = 4 blocks of 28 (one mask word each)

struct Lane {
    uint32_t sel;                // byte selector: (previous slot, this slot) -> (near sample | far sample << 16), raw I/Q
    uint32_t sgn, k;             // forwards 1, -16384; backwards -1, -1: the retry decides "one" <=> sgn * T + k >= 0
    uint32_t f_one, f_zero;      // scale factor after a decided one / zero
    uint32_t fwd;                // 1 forwards
    uint32_t c_one, c_m1, c_m16k;   // 1, -1, -16384 in registers: multipliers that keep additions on the FMA pipe
};

// applyPhaseCorrection's preamble measurements (dump1090.c:1498-1517): walk direction and scale
// factors from window samples m[-1], m[0], m[2], m[3], m[6], m[7], m[9], m[10].  `pre` = the first
// seven words of the window (forward order), `odd` as in the window layout above.
// `c_one`, `c_m1`, `c_m16k` = 1, -1, -16384 as values the compiler cannot see (kernel parameters).
MODES_SERIAL_FN void phase_setup(const uint32_t *pre, uint32_t odd, const uint16_t *lut_iq, uint32_t c_one, uint32_t c_m1,
                                 uint32_t c_m16k, Lane &L) {
    const uint32_t m_1 = magnitude_of(lut_iq, window_sample(pre, odd, 0));
    const uint32_t m0 = magnitude_of(lut_iq, window_sample(pre, odd, 1));
    const uint32_t m2 = magnitude_of(lut_iq, window_sample(pre, odd, 3));
    const uint32_t m3 = magnitude_of(lut_iq, window_sample(pre, odd, 4));
    const uint32_t m6 = magnitude_of(lut_iq, window_sample(pre, odd, 7));
    const uint32_t m7 = magnitude_of(lut_iq, window_sample(pre, odd, 8));
    const uint32_t m9 = magnitude_of(lut_iq, window_sample(pre, odd, 10));
    const uint32_t m10 = magnitude_of(lut_iq, window_sample(pre, odd, 11));
    const uint32_t on_time = m0 + m2 + m7 + m9;
    const uint32_t early = (m_1 + m6) * 2u, late = (m3 + m10) * 2u;
    const bool fwd = !(early > late);                    // early > late: walk backwards (:1517)
    const uint32_t lead = fwd ? late : early;
    const uint32_t den = lead + on_time;
    const uint32_t q = den ? 16384u * lead / den : 0u;   // den > 0 for every real candidate (m0 > m1 >= 0)
    const uint32_t up = (16384u + q) & 0xffffu, down = (16384u - q) & 0xffffu;
    // forwards a previous 1 scales the next first half-bit up, backwards a following 1 scales the
    // previous second half-bit down
    // (opaque: the walk should multiply by these registers, not re-derive them from `fwd` and `q`
    // with selects and negations inside its loop)
    L.f_one = opaque(fwd ? up : down); L.f_zero = opaque(fwd ? down : up);
    L.fwd = fwd ? 1u : 0u;
    L.sgn = opaque(fwd ? 1u : 0xffffffffu);
    L.k = opaque(fwd ? (uint32_t)-16384 : 0xffffffffu);
    L.c_one = c_one; L.c_m1 = c_m1; L.c_m16k = c_m16k;
    // near = the half-bit sample next to the previous decision (the one the retry rescales)
    //   forwards : near = first sample of the pair, far = second
    //   backwards: near = second sample, far = first
    L.sel = fwd ? (odd ? 0x7654u : 0x5432u) : (odd ? 0x1032u : 0x7610u);
}

struct Sweep {
    uint32_t wo;                 // previous slot
    uint32_t one;                // the retry's previous decision
    uint32_t dsum;               // sum of |first - second| over the pairs walked so far (:1714-1717)
};

// 28 pairs.  First attempt: g1 = near > far, nd1 = |near - far| < 256 (an indefinite bit, :1675);
// retry: gp2 / lp2 = the rescaled near sample exceeds far / far exceeds it by 256 or more.  Step t
// ends up at bit 27 - t of each word.  c1 = near - far uncorrected and c2 = the retry's decision
// value U of the block's first pair (`_first`) and last pair (`_last`): frame bit 0 is one of them.
//
// The retry in the scaled domain.  scaleSample (:1473) gives near' = min(floor(P / 2^14), 65535),
// P = near * factor < 2^31.  Magnitudes are below 65535 - 256, so with T = P - far * 2^14:
//     near' >  far        <=>  T >= 2^14          far  >  near'       <=>  T < 0
//     near' -  far >= 256 <=>  T >= 2^22          far  -  near' >= 256 <=>  T < -255 * 2^14
//     near' == far        <=>  0 <= T < 2^14
// (the clamp never matters: every threshold on the right is below 65535).  The decision "one"
// (forwards near' > far, backwards far > near') is U = sgn * T + k >= 0 with (sgn, k) = (1, -2^14)
// or (-1, -1); a tie is -2^14 <= U < 0 either way.  No shift, no clamp, and the serial chain from
// one decision to the next is multiply-add, multiply-add, multiply-add, compare, select.
//
// Pipes.  An sm_90 scheduler's integer ALU pipe and FMA pipe each take a warp instruction every
// second cycle; the walk is ALU-heavy by nature (funnel shifts, byte permutes, absolute
// differences), so every addition that can be a multiply-add with a register multiplier is one:
// per pair 10 ALU + 10 FMA + 3 load instructions.
MODES_SERIAL_FN void sweep_block(const uint32_t *slot, const Lane &L, Lut lut, Sweep &S, uint32_t &g1, uint32_t &nd1,
                                 uint32_t &gp2, uint32_t &lp2, uint32_t &c1_first, uint32_t &c2_first, uint32_t &c1_last,
                                 uint32_t &c2_last) {
    uint32_t a_g1 = 0, a_nd1 = 0, a_gp2 = 0, a_lp2 = 0;
#pragma unroll
    for (int t = 0; t < kBlockBits; t++) {
        const uint32_t wn = slot[t + 1];
        const uint32_t a = absdiff127x4(perm2(S.wo, wn, L.sel));
        S.wo = wn;
        const uint32_t X = lut_at(lut, a, kLutLow);       // near
        const uint32_t Y = lut_at(lut, a, kLutHigh);      // far
        // first attempt (:1667-1690)
        S.dsum = absdiff_add(X, Y, S.dsum);
        const uint32_t c1 = mad(Y, L.c_m1, X);            // near - far
        a_g1 = push_sign(a_g1, mad(X, L.c_m1, Y));        // far - near < 0
        a_nd1 = push_sign(a_nd1, absdiff_add(X, Y, 0xffffff00u));          // |near - far| - 256 < 0
        // retry (:1498-1558, then the same slicing): the near sample is rescaled by the factor the
        // previous decision selects
        const uint32_t P = X * (S.one ? L.f_one : L.f_zero);
        const uint32_t T = mad(Y, L.c_m16k, P);
        const uint32_t U = mad(T, L.sgn, L.k);
        S.one = (uint32_t)((int32_t)U >= 0);
        a_gp2 = push_sign(a_gp2, mad(T, L.c_m1, 0x3fffffu));               // T >= 2^22
        a_lp2 = push_sign(a_lp2, mad(T, L.c_one, 255u * 16384u));          // T < -255 * 2^14
        if (t == 0) { c1_first = c1; c2_first = U; }
        if (t == kBlockBits - 1) { c1_last = c1; c2_last = U; }
    }
    g1 = a_g1; nd1 = a_nd1; gp2 = a_gp2; lp2 = a_lp2;
}

// Four block words (step t of block k at bit 27 - t of w[k]) -> the 112-bit mask in frame order.
MODES_SERIAL_FN void frame_order(const uint32_t w[kBlocks], uint32_t fwd, uint32_t M[4]) {
    uint32_t g[kBlocks];
#pragma unroll
    for (int j = 0; j < kBlocks; j++) g[j] = fwd ? (bitrev(w[j]) >> 4) : w[kBlocks - 1 - j];
    M[0] = g[0] | (g[1] << 28);
    M[1] = (g[1] >> 4) | (g[2] << 24);
    M[2] = (g[2] >> 8) | (g[3] << 20);
    M[3] = g[3] >> 12;
}

// The walk's state between blocks: the eval_fused_kernel variant that stages half a window at a
// time runs blocks 0-1, restages, then runs blocks 2-3.
struct Walk {
    Sweep S;
    uint32_t G1[kBlocks], ND1[kBlocks], GP2[kBlocks], LP2[kBlocks];
    uint32_t c1f, c2f, c1l, c2l, dhalf;
};

MODES_SERIAL_FN void walk_begin(Walk &W, const Lane &L, uint32_t slot0) {
    W.S.wo = slot0;
    W.S.one = L.fwd;                                     // the first pair handled always scales up (:1523, :1544): forwards f_one, backwards f_zero
    W.S.dsum = 0;
#pragma unroll
    for (int j = 0; j < kBlocks; j++) W.G1[j] = W.ND1[j] = W.GP2[j] = W.LP2[j] = 0u;
    W.c1f = W.c2f = W.c1l = W.c2l = W.dhalf = 0u;
}

// Blocks k0 .. k1-1; `slots` is indexed as the whole walk (slots[28k + t + 1] is read).
MODES_SERIAL_FN void walk_blocks(Walk &W, const Lane &L, const uint32_t *slots, int k0, int k1, Lut lut) {
#pragma unroll 1
    for (int k = k0; k < k1; k++) {
        uint32_t g1, nd1, gp2, lp2, a, b, c, d;
        sweep_block(slots + kBlockBits * k, L, lut, W.S, g1, nd1, gp2, lp2, a, b, c, d);
        // no dynamic register indexing
#pragma unroll
        for (int j = 0; j < kBlocks; j++) {
            W.G1[j] = k == j ? g1 : W.G1[j]; W.ND1[j] = k == j ? nd1 : W.ND1[j];
            W.GP2[j] = k == j ? gp2 : W.GP2[j]; W.LP2[j] = k == j ? lp2 : W.LP2[j];
        }
        if (k == 0) { W.c1f = a; W.c2f = b; }
        if (k == 1) W.dhalf = W.S.dsum;                  // the first 56 pairs of the walk
        W.c1l = c; W.c2l = d;
    }
}

// Masks -> both attempts' verdicts; rec: the 12 words of pass[0] and pass[1] of the modes_candidate.
MODES_SERIAL_FN void walk_finish(const Walk &W, const Lane &L, bool at_buffer_start, int fix_errors, int aggressive,
                                 const Tables &tab, uint32_t rec[12]) {
    const uint32_t d112 = W.S.dsum;
    const uint32_t d56 = L.fwd ? W.dhalf : d112 - W.dhalf;   // bits 0..55 (:1716)
    // frame bit 0 is the walk's first pair forwards, its last pair backwards
    const int32_t c1 = (int32_t)(L.fwd ? W.c1f : W.c1l), c2 = (int32_t)(L.fwd ? W.c2f : W.c2l);
    const uint32_t tri1 = c1 == 0;                       // first pair is a tie: bits[0] == 2 (:1681)
    const uint32_t tri2 = c2 < 0 && c2 >= -16384;        // see sweep_block
    const uint32_t one0 = L.fwd ? (uint32_t)(c1 > 0) : (uint32_t)(c1 < 0);   // first > second (backwards near = second)
    const uint32_t one0_retry = (uint32_t)(c2 >= 0);

    uint32_t Gp[4], Lp[4], D[4], O[4], F[4];
    frame_order(W.G1, L.fwd, Gp);
    frame_order(W.ND1, L.fwd, Lp);
    // definite = the halves differ by 256 or more; bit 0 is always taken (:1675).  Backwards near/far
    // = second/first: on a definite pair first > second <=> !(near > far).
    const uint32_t flip = L.fwd ? 0u : 0xffffffffu;
    D[0] = ~Lp[0] | 1u; D[1] = ~Lp[1]; D[2] = ~Lp[2]; D[3] = ~Lp[3] & 0x0000ffffu;
#pragma unroll
    for (int j = 0; j < 4; j++) O[j] = D[j] & (Gp[j] ^ flip);                // first > second
    O[0] = (O[0] & ~1u) | one0;
    fill_copies(D, O, F);
    if (tri1) spread_tie_mask(D, F);

    Verdict P1, P2;
    judge_sliced(F, tri1, d56, d112, fix_errors, aggressive, tab, P1);
    P2.F[0] = P2.F[1] = P2.F[2] = P2.F[3] = 0;
    P2.msgtype = 0; P2.flags = 0; P2.errorbit = 0; P2.nfixed = 0; P2.crc = 0;
    if ((P1.flags & MODES_EVAL_GATE_OK) && !unconditionally_good(P1)) {
        P1.flags |= MODES_EVAL_P2_VALID;
        if (at_buffer_start) {                           // j == 0: retried without correction (:1660)
            P2 = P1;
            P2.flags &= ~(uint32_t)MODES_EVAL_P2_VALID;
        } else {
            uint32_t G[4];
            frame_order(W.GP2, L.fwd, Gp);
            frame_order(W.LP2, L.fwd, Lp);
            D[0] = Gp[0] | Lp[0] | 1u; D[1] = Gp[1] | Lp[1]; D[2] = Gp[2] | Lp[2]; D[3] = Gp[3] | Lp[3];
#pragma unroll
            for (int j = 0; j < 4; j++) O[j] = L.fwd ? Gp[j] : Lp[j];
            O[0] = (O[0] & ~1u) | one0_retry;
            fill_copies(D, O, G);
            if (tri2) spread_tie_mask(D, G);
            if (G[0] == F[0] && G[1] == F[1] && G[2] == F[2] && G[3] == F[3] && tri2 == tri1) {
                P2 = P1;                                 // same bits, same (uncorrected) delta sums: same verdict
                P2.flags &= ~(uint32_t)MODES_EVAL_P2_VALID;
            } else {
                judge_sliced(G, tri2, d56, d112, fix_errors, aggressive, tab, P2);
            }
        }
    }
    eval_words(P1, rec);
    eval_words(P2, rec + 6);
}

// Evaluate one candidate.  slots: its kSlots words in walk order (not modified); L: phase_setup's
// result for it; rec: the 12 words of pass[0] and pass[1] of its modes_candidate.
MODES_SERIAL_FN void evaluate(const uint32_t *slots, const Lane &L, bool at_buffer_start, int fix_errors, int aggressive,
                              const Tables &tab, Lut lut, uint32_t rec[12]) {
    Walk W;
    walk_begin(W, L, slots[0]);
    walk_blocks(W, L, slots, 0, kBlocks, lut);
    walk_finish(W, L, at_buffer_start, fix_errors, aggressive, tab, rec);
}

}  // namespace fused

}  // namespace serial
}  // namespace modes
