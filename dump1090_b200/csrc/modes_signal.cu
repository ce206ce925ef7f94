// modes_signal.cu — the signal-level pass (modes_set_signal), the arrival-time pass (modes_set_arrival)
// and the carrier pass (modes_set_carrier): for every decoded attempt of every candidate record, the RMS
// pulse magnitude of its frame (modes_signal_core.cuh), written into the record's pass[k].signal, its
// arrival code (modes_arrival_core.cuh), written into bits 4-7 of pass[k].flags, and its carrier record
// (modes_carrier_core.cuh), written into a separate array beside the records.
//
// It runs after frame evaluation, on the same stream and over the same virtual sample array
// (BatchView: carry block + body) while the batch is still in HBM, whichever evaluation kernel
// produced the records.  It is a separate kernel so that, with the features off, nothing about the
// default kernels changes.  One instantiation serves each combination of the three switches, so with
// several on the window is read once.
//
// Shape: a warp takes 32 consecutive records, one lane each, and reads their flags and positions
// (one load per lane); records with no decoded attempt cost nothing more.  The decoded ones are then
// measured one after the other by the whole warp: lane l holds the sample pairs of bits l, l+32,
// l+64, l+96 (one coalesced 4-byte load each, two when the window starts at an odd sample), the
// next record's pairs are requested before the current one is summed, and the warp reduces two
// sums, over the first 56 bits and over all 112, so one read of the window serves both attempts
// even when they differ in length.  For the arrival time lanes 0-15 also hold the preamble's samples
// 0-15, lane 16 sample 16+2*56 and lane 17 sample 16+2*112 (the sample after a frame's last bit);
// each attempt's bits, read from its record, give the sample classes as mask words, and the warp
// reduces four class sums per attempt.  For the carrier lanes 0 and 1 also hold the preamble pairs
// (samples 0, 2 and 7, 9); each attempt's bits pick every lane's pulse samples, the pulse of the next
// bit comes from the next lane (one shuffle per word), and the warp reduces two sums per attempt.
#include <cstdint>
#include <cuda_runtime.h>
#include "modes_internal.h"
#include "modes_signal_core.cuh"
#include "modes_arrival_core.cuh"
#include "modes_carrier_core.cuh"

namespace modes {

constexpr int kSignalThreads = 256;
constexpr int kSignalBlocksPerSm = 8;

using signal::load_pairs;

// Bits of the longest decoded attempt of a record (0 = none), from the words holding msgtype / flags.
__device__ __forceinline__ uint32_t bits_needed(uint32_t w0, uint32_t w1) {
    auto bits = [](uint32_t w) -> uint32_t {
        if (!((w >> 24) & MODES_EVAL_DECODED)) return 0;
        const uint32_t df = (w >> 16) & 0xffu;
        return (df >= 16 && df <= 21) ? 112u : 56u;                       // dump1090.c:746-753
    };
    const uint32_t a = bits(w0), b = bits(w1);
    return a > b ? a : b;
}

// The magnitude of the sample at virtual index v (one 2-byte load), as the raw sample (I, Q) word.
__device__ __forceinline__ uint32_t edge_sample(const BatchView &in, uint32_t t, int lane, uint32_t nb) {
    // lane < 16: preamble sample `lane`; 16: sample 16+2*56; 17: sample 16+2*112 (only read for 112-bit frames)
    const uint32_t s = lane < 16 ? (uint32_t)lane : (lane == 16 ? 128u : 240u);
    if (nb == 0 || lane > 17 || (lane == 17 && nb != 112)) return 0x7f7fu;
    return signal::raw_sample16(in, t + 2u + s);
}

// The arrival code of one decoded attempt of b bits whose first frame word is record word `w`:
// mf / ms = the magnitudes of the first / second sample of the lane's bit pairs, pre = the lane's
// edge sample magnitude (see edge_sample).  Every lane returns the code.
__device__ __forceinline__ uint32_t arrival_code(const uint32_t *rw, uint32_t b, const uint32_t mf[4], const uint32_t ms[4],
                                                 uint32_t pre, int lane) {
    uint32_t mw[4], B[4];
#pragma unroll
    for (int q = 0; q < 4; q++) mw[q] = rw[q];
    arrival::bit_words(mw, b, B);
    uint32_t S[4] = {0, 0, 0, 0};
#pragma unroll
    for (int r = 0; r < 4; r++) {
        const arrival::PairClasses c = arrival::pair_classes(B, r, b);
        const uint32_t bit = 1u << lane;
        S[arrival::kMain] += ((c.main1 & bit) ? mf[r] : 0u) + ((c.main2 & bit) ? ms[r] : 0u);
        S[arrival::kEarly] += (c.early1 & bit) ? mf[r] : 0u;
        S[arrival::kLate] += (c.late2 & bit) ? ms[r] : 0u;
    }
    const uint32_t bit0 = B[0] & 1u, last = (B[(b - 1) >> 5] >> ((b - 1) & 31)) & 1u;
    const uint32_t s = lane < 16 ? (uint32_t)lane : (lane == 16 ? 128u : (lane == 17 ? 240u : 0u));
    const uint32_t cls = (lane < 16 || s == 16 + 2 * b) ? arrival::edge_class(s, b, bit0, last) : (uint32_t)arrival::kUnused;
#pragma unroll
    for (int k = 0; k < 4; k++) S[k] += cls == (uint32_t)k ? pre : 0u;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
#pragma unroll
        for (int k = 0; k < 4; k++) S[k] += __shfl_xor_sync(0xffffffffu, S[k], o);
    uint32_t n[4];
    arrival::class_counts(B, b, n);
    return arrival::code_of(S, n);
}

// The preamble pair of lane 0 (samples 0 and 2) or lane 1 (samples 7 and 9) as one word, earlier sample in
// the low half; no signal on the other lanes and for a record without a decoded attempt.
__device__ __forceinline__ uint32_t carrier_preamble(const BatchView &in, uint32_t t, int lane, uint32_t nb) {
    if (nb == 0 || lane > 1) return 0x7f7f7f7fu;
    const uint32_t s = lane ? 7u : 0u;
    return signal::raw_sample16(in, t + 2u + s) | (signal::raw_sample16(in, t + 4u + s) << 16);
}

// The carrier sums (re, im) of one decoded attempt of b bits whose first frame word is record word `w`:
// pair[r] = the lane's bit pairs (see load_pairs), pre = its preamble pair (carrier_preamble).  Every lane
// returns the sums.
__device__ __forceinline__ void carrier_sums(const uint32_t *rw, uint32_t b, const uint32_t pair[4], uint32_t pre, int lane,
                                             int32_t &re, int32_t &im) {
    uint32_t mw[4], B[4], P[4];
#pragma unroll
    for (int q = 0; q < 4; q++) mw[q] = rw[q];
    arrival::bit_words(mw, b, B);
#pragma unroll
    for (int r = 0; r < 4; r++) P[r] = carrier::pulse_of(pair[r], (B[r] >> lane) & 1u);
    re = 0; im = 0;
    carrier::add_pair(pre & 0xffffu, pre >> 16, re, im);                 // 0 on lanes without a preamble pair
#pragma unroll
    for (int r = 0; r < 4; r++) {
        // the pulse of bit 32r + lane + 1: lane l reads lane l+1's, lane 31 lane 0's of the next word
        const uint32_t next = __shfl_sync(0xffffffffu, lane == 0 ? (r < 3 ? P[r + 1] : 0x7f7fu) : P[r], (lane + 1) & 31);
        if ((carrier::equal_next(B, r, b) >> lane) & 1u) carrier::add_pair(P[r], next, re, im);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        re += __shfl_xor_sync(0xffffffffu, re, o);
        im += __shfl_xor_sync(0xffffffffu, im, o);
    }
}

template <bool kSignal, bool kArrival, bool kCarrier>
__global__ void __launch_bounds__(kSignalThreads)
signal_kernel(BatchView in, const uint16_t *__restrict__ lutn, const uint32_t *counters, uint32_t cand_capacity,
              modes_candidate *records, modes_carrier *carrier) {
    const int lane = threadIdx.x & 31;
    uint32_t n = counters[0];
    if (n > cand_capacity) n = cand_capacity;
    const uint32_t n_warps = gridDim.x * (kSignalThreads / 32);
    for (uint32_t base = (blockIdx.x * kSignalThreads + threadIdx.x) / 32 * 32; base < n; base += 32 * n_warps) {
        // record words: [0] low half of t, [5] / [11] msgtype (byte 2) and flags (byte 3) of pass 0 / 1
        uint32_t t = 0, w0 = 0, w1 = 0;
        if (base + lane < n) {
            const uint32_t *rw = reinterpret_cast<const uint32_t *>(records + base + lane);
            t = rw[0]; w0 = rw[5]; w1 = rw[11];
        }
        uint32_t todo = __ballot_sync(0xffffffffu, bits_needed(w0, w1) != 0);
        if (!todo) continue;
        int c = __ffs(todo) - 1;
        todo &= todo - 1;
        uint32_t cw0 = __shfl_sync(0xffffffffu, w0, c), cw1 = __shfl_sync(0xffffffffu, w1, c);
        uint32_t cur[4], cur_pre = 0, cur_cpre = 0;
        {
            // virtual index of the candidate's m[j] is t + 2; its first bit's pair is 16 samples later
            const uint32_t ct = __shfl_sync(0xffffffffu, t, c);
            load_pairs(in, ct + 18u, bits_needed(cw0, cw1), lane, cur);
            if (kArrival) cur_pre = edge_sample(in, ct, lane, bits_needed(cw0, cw1));
            if (kCarrier) cur_cpre = carrier_preamble(in, ct, lane, bits_needed(cw0, cw1));
        }
        for (;;) {
            const bool more = todo != 0;
            int c2 = 0;
            uint32_t nw0 = 0, nw1 = 0, nxt[4], nxt_pre = 0, nxt_cpre = 0;
            if (more) {
                c2 = __ffs(todo) - 1;
                todo &= todo - 1;
                nw0 = __shfl_sync(0xffffffffu, w0, c2); nw1 = __shfl_sync(0xffffffffu, w1, c2);
                const uint32_t nt = __shfl_sync(0xffffffffu, t, c2);
                load_pairs(in, nt + 18u, bits_needed(nw0, nw1), lane, nxt);
                if (kArrival) nxt_pre = edge_sample(in, nt, lane, bits_needed(nw0, nw1));
                if (kCarrier) nxt_cpre = carrier_preamble(in, nt, lane, bits_needed(nw0, nw1));
            }
            if (kSignal) {
                uint64_t q56 = 0, q112 = 0;                               // bits < 56 / bits 56..111
#pragma unroll
                for (int r = 0; r < 4; r++) {
                    const uint64_t sq = signal::pulse_sq(cur[r], lutn);
                    if (32 * r + lane < 56) q56 += sq; else q112 += sq;
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    q56 += __shfl_xor_sync(0xffffffffu, q56, o);
                    q112 += __shfl_xor_sync(0xffffffffu, q112, o);
                }
                q112 += q56;
                if (lane == 0) {
                    uint16_t *h = reinterpret_cast<uint16_t *>(records + base + c);   // pass[k].signal = halfword 13 + 12k
#pragma unroll
                    for (int k = 0; k < 2; k++) {
                        const uint32_t nb = bits_needed(k ? cw1 : cw0, 0);
                        if (nb) h[13 + 12 * k] = signal::signal_of(nb == 112 ? q112 : q56, nb);
                    }
                }
            }
            if (kArrival) {
                uint32_t mf[4], ms[4], pre, unused;
#pragma unroll
                for (int r = 0; r < 4; r++) signal::pair_mags(cur[r], lutn, mf[r], ms[r]);
                signal::pair_mags(cur_pre | 0x7f7f0000u, lutn, pre, unused);
                const uint32_t *rw = reinterpret_cast<const uint32_t *>(records + base + c);
#pragma unroll
                for (int k = 0; k < 2; k++) {
                    const uint32_t cw = k ? cw1 : cw0, nb = bits_needed(cw, 0);
                    if (!nb) continue;                                    // warp-uniform
                    const uint32_t code = arrival_code(rw + 2 + 6 * k, nb, mf, ms, pre, lane);
                    // pass[k].flags = byte 23 + 24k; lane 0 is its only writer
                    if (lane == 0) reinterpret_cast<uint8_t *>(records + base + c)[23 + 24 * k] =
                        (uint8_t)(((cw >> 24) & 0x0fu) | (code << MODES_EVAL_ARRIVAL_SHIFT));
                }
            }
            if (kCarrier) {
                const uint32_t *rw = reinterpret_cast<const uint32_t *>(records + base + c);
                int32_t re[2] = {0, 0}, im[2] = {0, 0};
#pragma unroll
                for (int k = 0; k < 2; k++) {
                    const uint32_t nb = bits_needed(k ? cw1 : cw0, 0);
                    if (nb) carrier_sums(rw + 2 + 6 * k, nb, cur, cur_cpre, lane, re[k], im[k]);   // warp-uniform
                }
                if (lane == 0) reinterpret_cast<int4 *>(carrier)[base + c] = make_int4(re[0], re[1], im[0], im[1]);
            }
            if (!more) break;
            c = c2; cw0 = nw0; cw1 = nw1;
#pragma unroll
            for (int r = 0; r < 4; r++) cur[r] = nxt[r];
            cur_pre = nxt_pre;
            cur_cpre = nxt_cpre;
        }
    }
}

void launch_signal(const BatchView &in, const DeviceTables &tab, const ScanOutputs &scan, modes_candidate *records,
                   int sm_count, cudaStream_t stream, bool signal, bool arrival, modes_carrier *carrier) {
    const dim3 grid(sm_count * kSignalBlocksPerSm), block(kSignalThreads);
    const uint32_t cap = scan.cand_capacity;
    if (carrier) {
        if (signal && arrival)
            signal_kernel<true, true, true><<<grid, block, 0, stream>>>(in, tab.lutn, scan.counters, cap, records, carrier);
        else if (arrival)
            signal_kernel<false, true, true><<<grid, block, 0, stream>>>(in, tab.lutn, scan.counters, cap, records, carrier);
        else if (signal)
            signal_kernel<true, false, true><<<grid, block, 0, stream>>>(in, tab.lutn, scan.counters, cap, records, carrier);
        else
            signal_kernel<false, false, true><<<grid, block, 0, stream>>>(in, tab.lutn, scan.counters, cap, records, carrier);
    } else if (signal && arrival)
        signal_kernel<true, true, false><<<grid, block, 0, stream>>>(in, tab.lutn, scan.counters, cap, records, nullptr);
    else if (arrival)
        signal_kernel<false, true, false><<<grid, block, 0, stream>>>(in, tab.lutn, scan.counters, cap, records, nullptr);
    else if (signal)
        signal_kernel<true, false, false><<<grid, block, 0, stream>>>(in, tab.lutn, scan.counters, cap, records, nullptr);
}

}  // namespace modes
