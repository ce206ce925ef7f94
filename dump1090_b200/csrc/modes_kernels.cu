// modes_kernels.cu — sm_90a kernels of the Mode S demodulator.
//
//   (K1, the fused magnitude + preamble scan, lives in modes_scan2.cu.)
//   eval_kernel   (K2)  one warp per candidate: bit slicing (dump1090.c:1668-1706),
//                       delta gate (:1713-1726), phase-corrected retry (:1498-1558),
//                       CRC syndrome (:703-742) and syndrome-table repair
//                       (:795-894), both passes, as pure functions of the samples.
//   magnitude_kernel    computeMagnitudeVector alone, materialising u16 (tests only).
//   eval_frames_kernel  CRC + repair on raw frame bytes (hex door, :2472-2502).
//
// Integer-only; no tensor cores (there is no dense contraction on this path).
//
// Exactness notes.
//  * The reference compares magnitudes m = round(360*sqrt(n)), n = i*i+q*q with
//    i,q in [0,128].  m is strictly increasing over the reachable values of n
//    (consecutive integers n <= 32400 differ by >= 1.0 in 360*sqrt(n); the only
//    reachable values above are 32513 and 32768), so every magnitude-vs-magnitude
//    comparison of dump1090.c:1602-1611 is decided exactly on n.  Only the
//    "high" tests (:1624-1642) and the frame evaluation need m itself, read from
//    a table keyed by n that the host builds with the reference's formula.
//  * "copy the previous bit" slicing (dump1090.c:1675) and the decision chain
//    inside applyPhaseCorrection are both "last definite value wins" scans; on
//    ballot words they are the carry chain of one 128-bit addition (fill128).
#include <cstdint>
#include <cstdlib>
#include <cuda_runtime.h>
#include "modes_internal.h"
#include "modes_eval_serial.cuh"

namespace modes {

// ------------------------------------------------------------------ helpers

// One sample of the virtual array -> squared magnitude.
__device__ __forceinline__ uint32_t sample_n(const BatchView &in, uint64_t v) {
    const uint8_t *p = (v < (uint64_t)kHaloSamples) ? in.halo + 2 * v : in.body + 2 * (v - kHaloSamples);
    uint32_t w = *reinterpret_cast<const uint16_t *>(p);
    uint32_t a = __vabsdiffu4(w | 0x7f7f0000u, 0x7f7f7f7fu);
    return __dp4a(a, a, 0u);
}

// ------------------------------------------------------- K2: frame evaluation

struct U128 { uint64_t lo, hi; };

// Bits with D=1 are "definite" and take their value from O; bits with D=0 copy
// the nearest definite bit below.  That is the carry-out of (O|~D) + O.
__device__ __forceinline__ U128 fill128(U128 D, U128 O) {
    uint64_t a0 = O.lo | ~D.lo, a1 = O.hi | ~D.hi;
    uint64_t s0 = a0 + O.lo;
    uint64_t c = s0 < a0 ? 1ull : 0ull;
    uint64_t s1 = a1 + O.hi + c;
    uint64_t ci0 = s0 ^ a0 ^ O.lo, ci1 = s1 ^ a1 ^ O.hi;     // carry INTO each bit
    U128 f;
    f.lo = (ci0 >> 1) | (ci1 << 63);
    f.hi = ci1 >> 1;                                          // top bit unused (bits >= 112 are padding)
    return f;
}

__device__ __forceinline__ U128 ballot128(bool p0, bool p1, bool p2, bool p3) {
    uint32_t w0 = __ballot_sync(0xffffffffu, p0), w1 = __ballot_sync(0xffffffffu, p1);
    uint32_t w2 = __ballot_sync(0xffffffffu, p2), w3 = __ballot_sync(0xffffffffu, p3);
    U128 r; r.lo = w0 | ((uint64_t)w1 << 32); r.hi = w2 | ((uint64_t)w3 << 32);
    return r;
}

__device__ __forceinline__ uint32_t bit_of(U128 x, int b) {
    return (uint32_t)(((b < 64) ? (x.lo >> b) : (x.hi >> (b - 64))) & 1ull);
}

// Reverse the 112 valid bits (bit b <-> bit 111-b).
__device__ __forceinline__ U128 rev112(U128 x) {
    uint64_t rl = __brevll(x.hi), rh = __brevll(x.lo);       // 128-bit reversal: bit b -> 127-b
    U128 r; r.lo = (rl >> 16) | (rh << 48); r.hi = rh >> 16;  // then down by 16
    return r;
}

__device__ __forceinline__ int scale_sample(int v, int s) {   // dump1090.c:1473-1476
    uint32_t r = ((uint32_t)v * (uint32_t)s) >> 14;
    return r > 65535u ? 65535 : (int)r;
}

struct PassResult {
    uint32_t W[4];          // frame bytes as big-endian words (W[3]: top 16 bits)
    uint32_t msgtype, flags, errorbit, nfixed, crc;
};

__device__ __forceinline__ uint32_t fix_hash_of(uint32_t s) { return (s * 0x9E3779B1u) >> 24; }

// Position whose single-bit syndrome is s, or -1.
__device__ __forceinline__ int syndrome_pos(const uint32_t *s_hash, uint32_t s) {
    uint32_t h = fix_hash_of(s);
    for (int i = 0; i < kFixHashSlots; i++) {
        uint32_t e = s_hash[(h + i) & (kFixHashSlots - 1)];
        if (e == 0xFFFFFFFFu) return -1;
        if ((e >> 8) == s) return (int)(e & 0xff);
    }
    return -1;
}

// CRC syndrome + repair on frame bits F (bit b of the frame at bit b of F).
// dump1090.c:1099-1128 with :733-742 and :854-894.  Warp-uniform result.
__device__ __forceinline__ void crc_and_fix(U128 &F, int msgbits, uint32_t msgtype, int fix_errors, int aggressive,
                                            const uint32_t *s_syn, const uint32_t *s_hash, int lane,
                                            uint32_t &crc, uint32_t &errorbit, uint32_t &nfixed) {
    const int off = 112 - msgbits;
    uint32_t acc = 0;
    const uint32_t fw[4] = {(uint32_t)F.lo, (uint32_t)(F.lo >> 32), (uint32_t)F.hi, (uint32_t)(F.hi >> 32)};
#pragma unroll
    for (int r = 0; r < 4; r++) {
        const int b = 32 * r + lane;                     // bit b of the frame = bit `lane` of word r
        if (b < msgbits && ((fw[r] >> lane) & 1u)) acc ^= s_syn[b + off];
    }
    uint32_t S = __reduce_xor_sync(0xffffffffu, acc);
    errorbit = 0xFF; nfixed = 0;
    if (S != 0 && fix_errors && (msgtype == 11 || msgtype == 17 || msgtype == 18)) {
        const int pmin = off > 5 ? off : 5;                  // table covers frame positions 5..111
        // single-bit patterns
        int hit = -1;
#pragma unroll
        for (int r = 0; r < 4; r++) {
            int p = 32 * r + lane;
            uint32_t m = __ballot_sync(0xffffffffu, p >= pmin && p < 112 && s_syn[p] == S);
            if (m && hit < 0) hit = 32 * r + (__ffs(m) - 1);
        }
        if (hit >= 0) {
            int fb = hit - off;
            if (fb < 64) F.lo ^= 1ull << fb; else F.hi ^= 1ull << (fb - 64);
            errorbit = fb; nfixed = 1; S = 0;
        } else if (aggressive) {
            // two-bit patterns p<q: S ^ syn[p] must be the syndrome of some q
            int hp = -1, hq = -1;
#pragma unroll
            for (int r = 0; r < 4; r++) {
                int p = 32 * r + lane, q = -1;
                if (p >= pmin && p < 112) {
                    q = syndrome_pos(s_hash, S ^ s_syn[p]);
                    if (q <= p || q < pmin) q = -1;
                }
                uint32_t m = __ballot_sync(0xffffffffu, q >= 0);
                if (m && hp < 0) {
                    int src = __ffs(m) - 1;
                    hp = 32 * r + src;
                    hq = __shfl_sync(0xffffffffu, q, src);
                }
            }
            if (hp >= 0) {
                int f0 = hp - off, f1 = hq - off;
                if (f0 < 64) F.lo ^= 1ull << f0; else F.hi ^= 1ull << (f0 - 64);
                if (f1 < 64) F.lo ^= 1ull << f1; else F.hi ^= 1ull << (f1 - 64);
                errorbit = f0; nfixed = 2; S = 0;
            }
        }
    }
    crc = S;
}

__device__ __forceinline__ void frame_words(U128 F, uint32_t W[4]) {
    W[0] = __brev((uint32_t)F.lo); W[1] = __brev((uint32_t)(F.lo >> 32));
    W[2] = __brev((uint32_t)F.hi); W[3] = __brev((uint32_t)(F.hi >> 32)) & 0xffff0000u;
}

// Slice 112 bits from (lo, hi) half-bit magnitudes held 4 rounds per lane
// (round r, lane l <-> bit 32r+l), then gate, CRC, repair.
// `sliced` carries the frame bits as sliced (before any repair) and the tri-state flag; when
// `prev`/`prev_sliced` describe an earlier attempt that sliced the very same bits (the phase
// correction often changes no decision), its gate / CRC / repair results are reused.
struct Sliced { U128 F; uint32_t tri; };

__device__ __forceinline__ void evaluate_pass(const int lo[4], const int hi[4], uint32_t sum56, uint32_t sum112,
                                              int fix_errors, int aggressive, const uint32_t *s_syn,
                                              const uint32_t *s_hash, int lane, PassResult &R, Sliced &sliced,
                                              const PassResult *prev = nullptr, const Sliced *prev_sliced = nullptr) {
    bool def[4], one[4];
#pragma unroll
    for (int r = 0; r < 4; r++) {
        int b = 32 * r + lane;
        int d = lo[r] - hi[r]; d = d < 0 ? -d : d;
        bool valid = b < 112;
        def[r] = valid && (b == 0 || d >= 256);              // dump1090.c:1675
        one[r] = def[r] && lo[r] > hi[r];
    }
    U128 D = ballot128(def[0], def[1], def[2], def[3]);
    U128 O = ballot128(one[0], one[1], one[2], one[3]);
    uint32_t tri = __ballot_sync(0xffffffffu, lane == 0 && lo[0] == hi[0]) & 1u;   // bits[0] = 2, :1681
    U128 F = fill128(D, O);
    if (tri) {
        // The 2 propagates through the copy bits after bit 0; packed with <<(7-k%8)
        // each 2 at bit k sets bit k-1 unless k is the first bit of a byte (:1696-1706).
        U128 T; T.lo = ~D.lo | 1ull; T.hi = ~D.hi;
        uint64_t t0 = T.lo + 1ull, t1 = T.hi + (t0 == 0 ? 1ull : 0ull);
        U128 run; run.lo = T.lo & ~t0; run.hi = (t0 == 0) ? (T.hi & ~t1) : 0ull;
        uint64_t e0 = (run.lo >> 1) | (run.hi << 63), e1 = run.hi >> 1;
        F.lo |= e0 & 0x7f7f7f7f7f7f7f7full;
        F.hi |= e1 & 0x7f7f7f7f7f7f7f7full;
    }
    F.hi &= 0x0000ffffffffffffull;
    sliced.F = F; sliced.tri = tri;
    if (prev && prev_sliced->F.lo == F.lo && prev_sliced->F.hi == F.hi && prev_sliced->tri == tri) {
        R = *prev;                                       // same bits, same (uncorrected) delta sums: same verdict
        R.flags &= ~(uint32_t)MODES_EVAL_P2_VALID;
        return;
    }
    uint32_t W0 = __brev((uint32_t)F.lo);
    R.msgtype = W0 >> 27;
    const int msgbits = (R.msgtype >= 16 && R.msgtype <= 21) ? 112 : 56;      // dump1090.c:746-753
    uint32_t delta = (msgbits == 112) ? sum112 / 56u : sum56 / 28u;            // :1713-1718
    R.flags = tri ? MODES_EVAL_ERRORS : 0;
    R.crc = 0; R.errorbit = 0xFF; R.nfixed = 0;
    if (delta >= 2550u) {                                                      // :1723
        R.flags |= MODES_EVAL_GATE_OK;
        if (!tri || aggressive) {                                              // :1731 (errors is 0 or 1)
            R.flags |= MODES_EVAL_DECODED;
            crc_and_fix(F, msgbits, R.msgtype, fix_errors, aggressive, s_syn, s_hash, lane, R.crc, R.errorbit, R.nfixed);
        }
    }
    frame_words(F, R.W);
}

__device__ __forceinline__ bool unconditionally_good(const PassResult &R) {
    return (R.flags & MODES_EVAL_DECODED) && R.crc == 0 && (R.msgtype == 11 || R.msgtype == 17 || R.msgtype == 18);
}

// The six 32-bit words of a modes_frame_eval as laid out in memory.
__device__ __forceinline__ void eval_words(const PassResult &R, uint32_t w[6]) {
    w[0] = __byte_perm(R.W[0], 0, 0x0123);
    w[1] = __byte_perm(R.W[1], 0, 0x0123);
    w[2] = __byte_perm(R.W[2], 0, 0x0123);
    w[3] = (R.W[3] >> 24) | ((R.W[3] >> 8) & 0xff00u) | ((R.msgtype & 0xffu) << 16) | ((R.flags & 0xffu) << 24);
    w[4] = (R.errorbit & 0xffu) | ((R.nfixed & 0xffu) << 8);
    w[5] = R.crc & 0xffffffu;
}

constexpr int kEvalThreads = 256;

// Raw 32-bit words of one candidate's window m[-1..239] as held by one lane: window sample w
// (w = 0 is m[-1]) is halfword w + odd of the aligned word array starting at body sample
// (v-241) & ~1; bit b = 32r+lane needs words 8+b and 9+b, the preamble lanes word (lane+odd)/2.
struct RawWindow { uint32_t v, pw, wa[4], wb[4]; };

__device__ __forceinline__ void load_window(const BatchView &in, uint32_t v, int lane, RawWindow &w) {
    w.v = v;
    if (v <= (uint32_t)kHaloSamples) return;             // carry-block window: loaded on demand
    const uint32_t first = v - 1 - kHaloSamples;         // body sample index of m[-1]
    const uint32_t *wp = reinterpret_cast<const uint32_t *>(in.body) + (first >> 1);
    w.pw = (lane < 17) ? __ldg(wp + ((lane + (first & 1u)) >> 1)) : 0u;
#pragma unroll
    for (int r = 0; r < 4; r++) {
        const int b = 32 * r + lane;
        w.wa[r] = 0; w.wb[r] = 0;
        if (b < 112) { w.wa[r] = __ldg(wp + 8 + b); w.wb[r] = __ldg(wp + 9 + b); }
    }
}

constexpr uint32_t kEvalChunk = 8;

__global__ void __launch_bounds__(kEvalThreads)
eval_kernel(BatchView in, DeviceTables tab, const uint32_t *__restrict__ cand_v, uint32_t *counters,
            uint32_t cand_capacity, modes_candidate *records, int fix_errors, int aggressive) {
    __shared__ uint32_t s_syn[112];
    __shared__ uint32_t s_hash[kFixHashSlots];
    __shared__ __align__(8) uint32_t s_rec[16 * (kEvalThreads / 32)];
    for (int i = threadIdx.x; i < 112; i += blockDim.x) s_syn[i] = tab.bit_syn[i];
    for (int i = threadIdx.x; i < kFixHashSlots; i += blockDim.x) s_hash[i] = tab.fix_hash[i];
    __syncthreads();

    const int lane = threadIdx.x & 31;
    const uint32_t warps_per_block = kEvalThreads / 32;
    uint32_t n_cand = counters[0];
    if (n_cand > cand_capacity) n_cand = cand_capacity;

    // Candidates are handed out in chunks of kEvalChunk from a global counter (counters[3]), the
    // next chunk requested while the current one is evaluated: evaluation cost varies by candidate
    // (second pass or not, fix or not), so a static split leaves warps idle at the tail.
    // Software pipeline across the chunk sequence: the raw words of the next candidate are
    // requested before this one is evaluated, so the HBM round trip (cand_v -> I/Q words)
    // overlaps a full evaluation; positions are fetched two candidates ahead.
    const uint32_t total_warps = gridDim.x * warps_per_block;
    uint32_t ci = (blockIdx.x * warps_per_block + (threadIdx.x >> 5)) * kEvalChunk;   // chunk bases are multiples of kEvalChunk
    uint32_t pending = 0;                                 // lane 0: chunk requested ahead
    if (lane == 0) pending = total_warps + atomicAdd(&counters[3], 1u);
    RawWindow cur;
    uint32_t v1 = 0;                                      // position of the candidate after ci
    if (ci < n_cand) load_window(in, cand_v[ci], lane, cur);
    if (ci + 1 < n_cand) v1 = cand_v[ci + 1];
    while (ci < n_cand) {
        const uint32_t pos = ci & (kEvalChunk - 1);
        uint32_t next_base = 0;                           // needed for the last two of a chunk only
        if (pos >= kEvalChunk - 2) next_base = __shfl_sync(0xffffffffu, pending, 0) * kEvalChunk;
        const uint32_t i1 = pos + 1 < kEvalChunk ? ci + 1 : next_base + (pos + 1 - kEvalChunk);
        const uint32_t i2 = pos + 2 < kEvalChunk ? ci + 2 : next_base + (pos + 2 - kEvalChunk);
        RawWindow nxt;
        nxt.v = 0;
        if (i1 < n_cand) load_window(in, v1, lane, nxt);
        uint32_t v2 = 0;
        if (i2 < n_cand) v2 = cand_v[i2];

        const uint32_t v = cur.v;
        const uint64_t t = (uint64_t)v - 2;

        // magnitudes: 17 preamble samples m[-1..15] (lane p holds m[p-1]) and 112 (low, high) pairs
        int pm = 0;
        int lo[4], hi[4];
        if (v > (uint32_t)kHaloSamples) {
            const uint32_t odd = (v - 1 - kHaloSamples) & 1u;
            if (lane < 17) {
                const uint32_t h = lane + odd;
                const uint32_t a = __vabsdiffu4(((h & 1u) ? (cur.pw >> 16) : (cur.pw & 0xffffu)) | 0x7f7f0000u, 0x7f7f7f7fu);
                pm = __ldg(tab.lutn + __dp4a(a, a, 0u));
            }
#pragma unroll
            for (int r = 0; r < 4; r++) {
                lo[r] = 0; hi[r] = 0;
                if (32 * r + lane < 112) {
                    // low = window sample 17+2b, high = 18+2b
                    const uint32_t pair = odd ? cur.wb[r] : __byte_perm(cur.wa[r], cur.wb[r], 0x5432);
                    const uint32_t a = __vabsdiffu4(pair, 0x7f7f7f7fu);
                    lo[r] = __ldg(tab.lutn + __dp4a(a & 0x0000ffffu, a, 0u));
                    hi[r] = __ldg(tab.lutn + __dp4a(a & 0xffff0000u, a, 0u));
                }
            }
        } else {
            // window reaches into the carry block (first 240 positions of a batch)
            if (lane < 17) pm = __ldg(tab.lutn + sample_n(in, (uint64_t)v - 1 + lane));
#pragma unroll
            for (int r = 0; r < 4; r++) {
                const int b = 32 * r + lane;
                lo[r] = 0; hi[r] = 0;
                if (b < 112) {
                    const uint64_t sidx = (uint64_t)v + 16 + 2 * b;
                    lo[r] = __ldg(tab.lutn + sample_n(in, sidx));
                    hi[r] = __ldg(tab.lutn + sample_n(in, sidx + 1));
                }
            }
        }
        // sums for the delta gate, on the uncorrected samples (dump1090.c:1692-1693, :1713-1718)
        uint32_t d56 = 0, d112 = 0;
#pragma unroll
        for (int r = 0; r < 4; r++) {
            int d = lo[r] - hi[r]; d = d < 0 ? -d : d;
            d112 += d;
            if (32 * r + lane < 56) d56 += d;
        }
        d56 = __reduce_add_sync(0xffffffffu, d56);
        d112 = __reduce_add_sync(0xffffffffu, d112);

        PassResult P1, P2;
        Sliced S1, S2;
        evaluate_pass(lo, hi, d56, d112, fix_errors, aggressive, s_syn, s_hash, lane, P1, S1);
        P2.W[0] = P2.W[1] = P2.W[2] = P2.W[3] = 0;
        P2.msgtype = 0; P2.flags = 0; P2.errorbit = 0; P2.nfixed = 0; P2.crc = 0;

        if ((P1.flags & MODES_EVAL_GATE_OK) && !unconditionally_good(P1)) {
            P1.flags |= MODES_EVAL_P2_VALID;
            if ((((uint32_t)t) & (kBufSamples - 1)) == 0) {
                P2 = P1;                                     // j == 0: retry without correction (:1660)
                P2.flags &= ~MODES_EVAL_P2_VALID;
            } else {
                // applyPhaseCorrection, dump1090.c:1498-1558
                int m_1 = __shfl_sync(0xffffffffu, pm, 0), m0 = __shfl_sync(0xffffffffu, pm, 1);
                int m2 = __shfl_sync(0xffffffffu, pm, 3),  m3 = __shfl_sync(0xffffffffu, pm, 4);
                int m6 = __shfl_sync(0xffffffffu, pm, 7),  m7 = __shfl_sync(0xffffffffu, pm, 8);
                int m9 = __shfl_sync(0xffffffffu, pm, 10), m10 = __shfl_sync(0xffffffffu, pm, 11);
                uint32_t on_time = m0 + m2 + m7 + m9;
                uint32_t early = (uint32_t)(m_1 + m6) * 2u, late = (uint32_t)(m3 + m10) * 2u;
                int clo[4], chi[4];
                if (early > late) {
                    // walk backwards: only the second half-bit samples are rescaled
                    uint32_t q = 16384u * early / (early + on_time);
                    int up = (int)((16384u + q) & 0xffffu), down = (int)((16384u - q) & 0xffffu);
                    int hu[4], hd[4];
                    bool def[4], one[4];
#pragma unroll
                    for (int r = 0; r < 4; r++) {
                        int b = 32 * r + lane;
                        hu[r] = scale_sample(hi[r], up); hd[r] = scale_sample(hi[r], down);
                        bool g0 = lo[r] > hu[r], g1 = lo[r] > hd[r];        // decision if the bit above was 0 / 1
                        def[r] = b < 112 && (b == 111 || g0 == g1);
                        one[r] = def[r] && g0;
                    }
                    U128 D = rev112(ballot128(def[0], def[1], def[2], def[3]));
                    U128 O = rev112(ballot128(one[0], one[1], one[2], one[3]));
                    D.hi |= 0xffff000000000000ull;                          // padding: definite zeros
                    U128 E = fill128(D, O);                                 // E bit (111-b) = decision at bit b
#pragma unroll
                    for (int r = 0; r < 4; r++) {
                        int b = 32 * r + lane;
                        clo[r] = lo[r];
                        chi[r] = hi[r];
                        if (b == 111) chi[r] = hu[r];
                        else if (b < 111) chi[r] = bit_of(E, 110 - b) ? hd[r] : hu[r];
                    }
                } else {
                    // walk forwards: only the first half-bit samples are rescaled
                    uint32_t q = 16384u * late / (late + on_time);
                    int up = (int)((16384u + q) & 0xffffu), down = (int)((16384u - q) & 0xffffu);
                    int lu[4], ld[4];
                    bool def[4], one[4];
#pragma unroll
                    for (int r = 0; r < 4; r++) {
                        int b = 32 * r + lane;
                        lu[r] = scale_sample(lo[r], up); ld[r] = scale_sample(lo[r], down);
                        bool f1 = lu[r] > hi[r], f0 = ld[r] > hi[r];        // decision if the bit below was 1 / 0
                        def[r] = b < 112 && (b == 0 || f0 == f1);
                        one[r] = def[r] && f1;
                    }
                    U128 D = ballot128(def[0], def[1], def[2], def[3]);
                    U128 O = ballot128(one[0], one[1], one[2], one[3]);
                    U128 E = fill128(D, O);                                 // E bit b = decision at bit b
#pragma unroll
                    for (int r = 0; r < 4; r++) {
                        int b = 32 * r + lane;
                        chi[r] = hi[r];
                        clo[r] = lo[r];
                        if (b == 0) clo[r] = lu[r];
                        else if (b < 112) clo[r] = bit_of(E, b - 1) ? lu[r] : ld[r];
                    }
                }
                evaluate_pass(clo, chi, d56, d112, fix_errors, aggressive, s_syn, s_hash, lane, P2, S2, &P1, &S1);
            }
        }

        // one coalesced 56-byte record: lanes 0..13 write one word each
        // every lane holds the whole (warp-uniform) record; lane 0 lines it up in shared memory and
        // lanes 0..13 store one word each: one coalesced 56-byte write
        uint32_t *stg = s_rec + 16 * (threadIdx.x >> 5);
        if (lane == 0) {
            uint32_t rec[14];
            rec[0] = (uint32_t)t; rec[1] = (uint32_t)(t >> 32);
            eval_words(P1, rec + 2);
            eval_words(P2, rec + 8);
#pragma unroll
            for (int k = 0; k < 14; k += 2) *reinterpret_cast<uint2 *>(stg + k) = make_uint2(rec[k], rec[k + 1]);
        }
        __syncwarp();
        if (lane < 14) reinterpret_cast<uint32_t *>(records + ci)[lane] = stg[lane];
        __syncwarp();
        cur = nxt;
        v1 = v2;
        if (((++ci) & (kEvalChunk - 1)) == 0) {
            ci = next_base;
            if (lane == 0 && ci < n_cand) pending = total_warps + atomicAdd(&counters[3], 1u);
        }
    }
}

// ---- K2, one thread per candidate ----------------------------------------------------------
// The evaluation itself is modes_eval_serial.cuh (sequential code over one candidate's window).
// A warp takes 32 consecutive candidates: their windows are staged in shared memory with
// coalesced loads (row stride 121 words, so that lane l walking its own row hits bank 25l+k:
// conflict free), every lane evaluates its own candidate, and the 32 records leave through the
// same shared memory as one contiguous 1792-byte store.  Chunks of 32 are handed out from a global
// counter, the next one requested before the current one is staged.
constexpr int kSerWarps = 12;                          // one CTA per SM
constexpr int kSerThreads = 32 * kSerWarps;
constexpr int kSerRow = serial::kWindowWords;          // 121 words: odd, so lane l walking its own row hits bank 25l+k
constexpr int kSerNibWords = 28 * 16;
constexpr int kSerLutWords = serial::kIqLutEntries / 2;
static_assert(serial::kIqLutStride == kLutIqStride && serial::kIqLutEntries % 8 == 0, "table geometry");
static_assert((112 + kFixHashSlots + kSerNibWords + kSerLutWords) % 2 == 0 && (32 * kSerRow) % 2 == 0, "record staging uses 8-byte stores");
constexpr int kSerTableWords = 112 + kFixHashSlots + kSerNibWords + kSerLutWords;
constexpr int kSerSmemBytes = 4 * (kSerTableWords + kSerWarps * 32 * kSerRow);

__device__ __forceinline__ uint32_t raw_sample(const BatchView &in, uint64_t v) {
    const uint8_t *p = (v < (uint64_t)kHaloSamples) ? in.halo + 2 * v : in.body + 2 * (v - kHaloSamples);
    return *reinterpret_cast<const uint16_t *>(p);
}

__device__ __forceinline__ void cp_async4(uint32_t dst_shared, const uint32_t *src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst_shared), "l"(src) : "memory");
}

// kLean selects the leaner instruction sequences of modes_eval_serial.cuh for the two per-bit loops
// (the default; MODES_EVAL_VARIANT=serial selects the other coding; same results).
template <bool kLean>
__global__ void __launch_bounds__(kSerThreads, 1)
eval_serial_kernel(BatchView in, DeviceTables tab, const uint32_t *__restrict__ cand_v, uint32_t *counters,
                   uint32_t cand_capacity, modes_candidate *records, int fix_errors, int aggressive) {
    extern __shared__ __align__(16) uint32_t s_mem[];
    uint32_t *s_syn = s_mem, *s_hash = s_syn + 112, *s_nib = s_hash + kFixHashSlots;
    uint16_t *s_lut = reinterpret_cast<uint16_t *>(s_nib + kSerNibWords);
    uint32_t *s_win = s_nib + kSerNibWords + kSerLutWords;
    for (int i = threadIdx.x; i < 112; i += kSerThreads) s_syn[i] = tab.bit_syn[i];
    for (int i = threadIdx.x; i < kFixHashSlots; i += kSerThreads) s_hash[i] = tab.fix_hash[i];
    // magnitude by (|I-127|, |Q-127|): the table the per-thread lookups hit stays in shared memory
    // (as gathers from the 64 KB n-keyed table in L1 they were the kernel's bottleneck: ~5 wavefronts each)
    for (int i = threadIdx.x; i < serial::kIqLutEntries / 8; i += kSerThreads)
        reinterpret_cast<uint4 *>(s_lut)[i] = __ldg(reinterpret_cast<const uint4 *>(tab.lut_iq) + i);
    __syncthreads();
    for (int i = threadIdx.x; i < kSerNibWords; i += kSerThreads) s_nib[i] = serial::nibble_syndrome(s_syn, i >> 4, i & 15);
    __syncthreads();

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t *wwin = s_win + warp * 32 * kSerRow;
    const uint32_t wwin_s = (uint32_t)__cvta_generic_to_shared(wwin);
    const serial::Tables T{s_lut, s_syn, s_nib, s_hash, tab.pair_hash};
    uint32_t n_cand = counters[0];
    if (n_cand > cand_capacity) n_cand = cand_capacity;
    const uint32_t n_chunks = (n_cand + 31) / 32;
    const uint32_t total_warps = gridDim.x * kSerWarps;
    const uint32_t *body32 = reinterpret_cast<const uint32_t *>(in.body);

    // Chunks of 32 candidates are handed out from a global counter, requested TWO chunks ahead: one
    // chunk ahead the candidate positions are already loaded, and while the current chunk is
    // evaluated the next chunk's windows are on their way into L2 (one prefetch per 128-byte line).
    // (The counter values are used untouched until a chunk later: arithmetic on them right away
    // would wait for the atomic's round trip.)
    uint32_t chunk = blockIdx.x * kSerWarps + warp;
    uint32_t next1 = 0, ahead_raw = 0;
    if (lane == 0) next1 = atomicAdd(&counters[3], 1u);
    next1 = total_warps + __shfl_sync(0xffffffffu, next1, 0);
    uint32_t my_v = 0;
    if (chunk < n_chunks) {
        const uint32_t n0 = n_cand - chunk * 32 < 32u ? n_cand - chunk * 32 : 32u;
        my_v = cand_v[chunk * 32 + ((uint32_t)lane < n0 ? lane : n0 - 1)];
    }
    while (chunk < n_chunks) {
        if (lane == 0) ahead_raw = atomicAdd(&counters[3], 1u);
        const uint32_t base = chunk * 32;
        const uint32_t n = n_cand - base < 32u ? n_cand - base : 32u;   // idle lanes of the last chunk duplicate its last candidate
        uint32_t v_next = 0;

        // stage the windows: row c = candidate c, words (first>>1) .. +120 of the body
        if (__all_sync(0xffffffffu, my_v > (uint32_t)kHaloSamples)) {
            // common case (no window in the carry block): asynchronous copies straight into shared
            // memory, all 32 rows in flight, one wait
#pragma unroll 8
            for (int c = 0; c < 32; c++) {
                const uint32_t v = __shfl_sync(0xffffffffu, my_v, c);
                const uint32_t *wp = body32 + ((v - 1 - kHaloSamples) >> 1) + lane;
                const uint32_t dst = wwin_s + 4u * (uint32_t)(c * kSerRow + lane);
                cp_async4(dst, wp); cp_async4(dst + 128u, wp + 32); cp_async4(dst + 256u, wp + 64);
                if (lane < serial::kWindowWords - 96) cp_async4(dst + 384u, wp + 96);
            }
            if (next1 < n_chunks) {                        // the next chunk's positions: loaded behind the copies, used a chunk later
                const uint32_t n1 = n_cand - next1 * 32 < 32u ? n_cand - next1 * 32 : 32u;
                v_next = cand_v[next1 * 32 + ((uint32_t)lane < n1 ? lane : n1 - 1)];
            }
            asm volatile("cp.async.wait_all;" ::: "memory");
        } else {
            if (next1 < n_chunks) {
                const uint32_t n1 = n_cand - next1 * 32 < 32u ? n_cand - next1 * 32 : 32u;
                v_next = cand_v[next1 * 32 + ((uint32_t)lane < n1 ? lane : n1 - 1)];
            }
            for (uint32_t c = 0; c < n; c++) {
                const uint32_t v = __shfl_sync(0xffffffffu, my_v, c);
                uint32_t *row = wwin + c * kSerRow;
                if (v > (uint32_t)kHaloSamples) {
                    const uint32_t *wp = body32 + ((v - 1 - kHaloSamples) >> 1);
                    for (int k = lane; k < serial::kWindowWords; k += 32) row[k] = __ldg(wp + k);
                } else {
                    // window reaches into the carry block (first 240 positions of a batch): sample by sample, odd = 0
                    for (int k = lane; k < serial::kWindowWords; k += 32)
                        row[k] = raw_sample(in, (uint64_t)v - 1 + 2 * k) | (raw_sample(in, (uint64_t)v + 2 * k) << 16);
                }
            }
        }
        __syncwarp();
        // the next chunk's windows -> L2 (484 bytes from a 4-byte aligned address: five 128-byte lines)
        if (v_next > (uint32_t)kHaloSamples) {
            const uint8_t *wp = in.body + 4ull * ((v_next - 1 - kHaloSamples) >> 1);
            if ((uint64_t)(wp - in.body) + 640u <= 2ull * in.n_samples) {
#pragma unroll
                for (int k = 0; k < 5; k++) asm volatile("prefetch.global.L2 [%0];" ::"l"(wp + 128 * k));
            }
        }

        uint32_t rec[14];
        if ((uint32_t)lane < n) {
            const uint64_t t = (uint64_t)my_v - 2;
            const uint32_t odd = my_v > (uint32_t)kHaloSamples ? ((my_v - 1 - kHaloSamples) & 1u) : 0u;
            rec[0] = (uint32_t)t; rec[1] = (uint32_t)(t >> 32);
            serial::evaluate<kLean>(wwin + lane * kSerRow, odd, (((uint32_t)t) & (kBufSamples - 1)) == 0, fix_errors, aggressive,
                             T, rec + 2);
        }
        __syncwarp();
        if ((uint32_t)lane < n) {
#pragma unroll
            for (int k = 0; k < 14; k += 2) *reinterpret_cast<uint2 *>(wwin + 14 * lane + k) = make_uint2(rec[k], rec[k + 1]);
        }
        __syncwarp();
        uint32_t *dst = reinterpret_cast<uint32_t *>(records + base);
        for (uint32_t i = lane; i < n * 14; i += 32) dst[i] = wwin[i];
        __syncwarp();
        chunk = next1;
        my_v = v_next;
        next1 = total_warps + __shfl_sync(0xffffffffu, ahead_raw, 0);
    }
}

// MODES_EVAL_VARIANT: default "fused" = thread per candidate, both attempts in one walk
// (modes_eval_fused.cu; measured 0.166 ms for the bench's 845 458 candidates), "fused2" = the same with
// half windows staged (0.170 ms); "lean" = thread per candidate, two passes (0.242 ms), "serial" = the same
// kernel with the first coding of the per-bit loops (0.290 ms); "warp" = the warp-per-candidate kernel
// (the first formulation, 0.56 ms).  All stay in the parity tests.  Read per launch (tests switch it
// within one process).
static int eval_variant() {
    const char *e = std::getenv("MODES_EVAL_VARIANT");
    if (!e || e[0] == 'f') return (e && e[5] == '2') ? 4 : 3;
    return e[0] == 'w' ? 1 : (e[0] == 's' ? 0 : 2);
}

template <bool kLean>
static void launch_eval_serial(const BatchView &in, const DeviceTables &tab, const ScanOutputs &scan, modes_candidate *records,
                               int fix_errors, int aggressive, int sm_count, cudaStream_t stream) {
    // the opt-in to > 48 KB of dynamic shared memory is per device
    static bool configured[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64 || !configured[dev]) {
        cudaFuncSetAttribute(eval_serial_kernel<kLean>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSerSmemBytes);
        if (dev >= 0 && dev < 64) configured[dev] = true;
    }
    eval_serial_kernel<kLean><<<sm_count, kSerThreads, kSerSmemBytes, stream>>>(in, tab, scan.cand_v, scan.counters,
                                                                                   scan.cand_capacity, records, fix_errors, aggressive);
}

void launch_eval(const BatchView &in, const DeviceTables &tab, const ScanOutputs &scan,
                 modes_candidate *records, int fix_errors, int aggressive, int sm_count,
                 cudaStream_t stream) {
    const int variant = eval_variant();
    if (variant >= 3)
        launch_eval_fused(in, tab, scan, records, fix_errors, aggressive, sm_count, variant - 2, stream);
    else if (variant == 1)
        eval_kernel<<<sm_count * 4, kEvalThreads, 0, stream>>>(in, tab, scan.cand_v, scan.counters, scan.cand_capacity,
                                                              records, fix_errors, aggressive);
    else if (variant == 2)
        launch_eval_serial<true>(in, tab, scan, records, fix_errors, aggressive, sm_count, stream);
    else
        launch_eval_serial<false>(in, tab, scan, records, fix_errors, aggressive, sm_count, stream);
}

// ------------------------------------------------------- magnitude (tests)

__global__ void __launch_bounds__(256)
magnitude_kernel(const uint8_t *__restrict__ iq, uint16_t *__restrict__ mag, uint64_t n_samples,
                 const uint16_t *__restrict__ lutn) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (; i < n_samples; i += stride) {
        uint32_t w = reinterpret_cast<const uint16_t *>(iq)[i];
        uint32_t a = __vabsdiffu4(w | 0x7f7f0000u, 0x7f7f7f7fu);
        mag[i] = __ldg(lutn + __dp4a(a, a, 0u));
    }
}

void launch_magnitude(const uint8_t *d_iq, uint16_t *d_mag, uint64_t n_samples, const uint16_t *lutn,
                      cudaStream_t stream) {
    if (!n_samples) return;
    uint64_t blocks = (n_samples + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    magnitude_kernel<<<(uint32_t)blocks, 256, 0, stream>>>(d_iq, d_mag, n_samples, lutn);
}

// ------------------------------------------------------- hex door

__global__ void __launch_bounds__(32)
eval_frames_kernel(const uint8_t *__restrict__ frames, modes_frame_eval *out, uint32_t n, DeviceTables tab,
                   int fix_errors, int aggressive) {
    __shared__ uint32_t s_syn[112];
    __shared__ uint32_t s_hash[kFixHashSlots];
    const int lane = threadIdx.x;
    for (int i = lane; i < 112; i += 32) s_syn[i] = tab.bit_syn[i];
    for (int i = lane; i < kFixHashSlots; i += 32) s_hash[i] = tab.fix_hash[i];
    __syncwarp();
    for (uint32_t f = blockIdx.x; f < n; f += gridDim.x) {
        const uint8_t *m = frames + 14 * (size_t)f;
        // frame bit b lives at bit b of F
        bool bit[4];
#pragma unroll
        for (int r = 0; r < 4; r++) {
            int b = 32 * r + lane;
            bit[r] = b < 112 && ((m[b >> 3] >> (7 - (b & 7))) & 1);
        }
        U128 F = ballot128(bit[0], bit[1], bit[2], bit[3]);
        PassResult R;
        R.msgtype = m[0] >> 3;
        const int msgbits = (R.msgtype >= 16 && R.msgtype <= 21) ? 112 : 56;
        R.flags = MODES_EVAL_GATE_OK | MODES_EVAL_DECODED;
        crc_and_fix(F, msgbits, R.msgtype, fix_errors, aggressive, s_syn, s_hash, lane, R.crc, R.errorbit, R.nfixed);
        frame_words(F, R.W);
        uint32_t rec[6], word = 0;
        eval_words(R, rec);
#pragma unroll
        for (int k = 0; k < 6; k++) word = (lane == k) ? rec[k] : word;
        if (lane < 6) reinterpret_cast<uint32_t *>(out + f)[lane] = word;
    }
}

void launch_eval_frames(const uint8_t *d_frames, modes_frame_eval *d_out, uint32_t n, const DeviceTables &tab,
                        int fix_errors, int aggressive, cudaStream_t stream) {
    if (!n) return;
    eval_frames_kernel<<<n < 1024 ? n : 1024, 32, 0, stream>>>(d_frames, d_out, n, tab, fix_errors, aggressive);
}

}  // namespace modes
