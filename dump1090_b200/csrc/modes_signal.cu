// modes_signal.cu — the signal-level pass (modes_set_signal): for every decoded attempt of every
// candidate record, the RMS pulse magnitude of its frame (modes_signal_core.cuh), written into the
// record's pass[k].signal.
//
// It runs after frame evaluation, on the same stream and over the same virtual sample array
// (BatchView: carry block + body) while the batch is still in HBM, whichever evaluation kernel
// produced the records.  It is a separate kernel so that, with the feature off, nothing about the
// default kernels changes.
//
// Shape: a warp takes 32 consecutive records, one lane each, and reads their flags and positions
// (one load per lane); records with no decoded attempt cost nothing more.  The decoded ones are then
// measured one after the other by the whole warp: lane l holds the sample pairs of bits l, l+32,
// l+64, l+96 (one coalesced 4-byte load each, two when the window starts at an odd sample), the
// next record's pairs are requested before the current one is summed, and the warp reduces two
// sums, over the first 56 bits and over all 112, so one read of the window serves both attempts
// even when they differ in length.
#include <cstdint>
#include <cuda_runtime.h>
#include "modes_internal.h"
#include "modes_signal_core.cuh"

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

__global__ void __launch_bounds__(kSignalThreads)
signal_kernel(BatchView in, const uint16_t *__restrict__ lutn, const uint32_t *counters, uint32_t cand_capacity,
              modes_candidate *records) {
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
        uint32_t cur[4];
        // virtual index of the candidate's m[j] is t + 2; its first bit's pair is 16 samples later
        load_pairs(in, __shfl_sync(0xffffffffu, t, c) + 18u, bits_needed(cw0, cw1), lane, cur);
        for (;;) {
            const bool more = todo != 0;
            int c2 = 0;
            uint32_t nw0 = 0, nw1 = 0, nxt[4];
            if (more) {
                c2 = __ffs(todo) - 1;
                todo &= todo - 1;
                nw0 = __shfl_sync(0xffffffffu, w0, c2); nw1 = __shfl_sync(0xffffffffu, w1, c2);
                load_pairs(in, __shfl_sync(0xffffffffu, t, c2) + 18u, bits_needed(nw0, nw1), lane, nxt);
            }
            uint64_t q56 = 0, q112 = 0;                                   // bits < 56 / bits 56..111
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
            if (!more) break;
            c = c2; cw0 = nw0; cw1 = nw1;
#pragma unroll
            for (int r = 0; r < 4; r++) cur[r] = nxt[r];
        }
    }
}

void launch_signal(const BatchView &in, const DeviceTables &tab, const ScanOutputs &scan, modes_candidate *records,
                   int sm_count, cudaStream_t stream) {
    signal_kernel<<<sm_count * kSignalBlocksPerSm, kSignalThreads, 0, stream>>>(in, tab.lutn, scan.counters,
                                                                                scan.cand_capacity, records);
}

}  // namespace modes
