// modes_recover.cu — the recovery pass (modes_set_recovery): for every candidate record, the
// soft-decision search over its ten least confident bits (modes_recover_core.cuh), written as one
// modes_recovered record at the candidate's index.
//
// It runs after frame evaluation, on the same stream and over the same virtual sample array
// (BatchView: carry block + body) while the batch is still in HBM, and reads the candidate count on
// the device, like the signal pass.  It is a separate kernel so that, with the feature off, nothing
// about the default kernels changes (frame evaluation has no register headroom).
//
// Shape: one warp per candidate.  Lane l holds the sample pairs of bits l, l+32, l+64, l+96 (the
// signal pass's coalesced loads), slices them, and the warp assembles the hard frame with four
// ballots.  Candidates of another DF are written and left there.  For DF17/18 the warp reduces the
// syndrome, selects the ten positions with ten arg-min rounds over (w, i) keys, and searches the
// 1024 subsets: lane l takes high subset bits l and walks the low five in Gray-code order.  The
// least weight and the number of solutions of that weight are reduced across the warp; lane 0 is
// the only writer of the record, so a batch repeated after a candidate overflow writes the same bytes.
#include <cstdint>
#include <cuda_runtime.h>
#include "modes_internal.h"
#include "modes_recover_core.cuh"
#include "modes_signal_core.cuh"

namespace modes {

constexpr int kRecoverThreads = 256;

__global__ void __launch_bounds__(kRecoverThreads)
recover_kernel(BatchView in, const uint16_t *__restrict__ lutn, const uint32_t *__restrict__ bit_syn,
               const uint32_t *counters, uint32_t capacity, const modes_candidate *records, modes_recovered *out) {
    const int lane = threadIdx.x & 31;
    const uint32_t full = 0xffffffffu;
    uint32_t n = counters[0];
    if (n > capacity) n = capacity;
    const uint32_t n_warps = gridDim.x * (kRecoverThreads / 32);
    for (uint32_t c = (blockIdx.x * kRecoverThreads + threadIdx.x) / 32; c < n; c += n_warps) {
        // virtual index of the candidate's m[j] is t + 2; its first bit's pair is 16 samples later
        const uint32_t t = *reinterpret_cast<const uint32_t *>(records + c);
        uint32_t pair[4];
        signal::load_pairs(in, t + 18u, 112u, lane, pair);
        uint32_t frame[4], key[4], syn = 0;
        uint64_t sq = 0;
#pragma unroll
        for (int r = 0; r < 4; r++) {
            const uint32_t i = 32 * r + lane;
            uint32_t a, b;
            signal::pair_mags(pair[r], lutn, a, b);
            const bool one = a > b;
            frame[r] = __brev(__ballot_sync(full, one));              // bits past 111 are 0 (no signal)
            key[r] = recover::bit_key(a, b, i);
            const uint32_t p = a > b ? a : b;
            sq += (uint64_t)(p * p);
            if (one && i < 112) syn ^= __ldg(bit_syn + i);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            sq += __shfl_xor_sync(full, sq, o);
            syn ^= __shfl_xor_sync(full, syn, o);
        }
        const uint32_t signal = signal::signal_of(sq, 112);
        const uint32_t df = frame[0] >> 27;
        uint32_t status = MODES_RECOVER_INELIGIBLE, nflips = 0;
        if (df == 17 || df == 18) {                                   // warp-uniform
            uint32_t pos[recover::kBits], s[recover::kBits];
#pragma unroll
            for (int k = 0; k < recover::kBits; k++) {
                uint32_t m = min(min(key[0], key[1]), min(key[2], key[3]));
                m = __reduce_min_sync(full, m);
                pos[k] = m & 127u;
#pragma unroll
                for (int r = 0; r < 4; r++) key[r] = key[r] == m ? recover::kNoKey : key[r];
                s[k] = __ldg(bit_syn + pos[k]);
            }
            const recover::Part part = recover::search_part((uint32_t)lane, s, syn);
            const uint32_t minw = __reduce_min_sync(full, part.minw);
            const uint32_t count = __reduce_add_sync(full, part.minw == minw ? part.count : 0u);
            status = recover::status_of(minw, count);
            if (status == MODES_RECOVER_FOUND) {
                const int owner = __ffs(__ballot_sync(full, part.minw == minw && part.count)) - 1;
                const uint32_t mask = __shfl_sync(full, part.mask, owner);
#pragma unroll
                for (int k = 0; k < recover::kBits; k++)
                    if ((mask >> k) & 1u) {
#pragma unroll
                        for (int r = 0; r < 4; r++)
                            if ((pos[k] >> 5) == (uint32_t)r) frame[r] ^= 0x80000000u >> (pos[k] & 31u);
                    }
                nflips = __popc(mask);
            } else if (status == MODES_RECOVER_AMBIGUOUS) {
                nflips = minw;
            }
        }
        if (lane == 0) {
            uint32_t w[5];
            recover::record_words(frame, status, nflips, signal, w);
            uint32_t *o = reinterpret_cast<uint32_t *>(out + c);
#pragma unroll
            for (int k = 0; k < 5; k++) o[k] = w[k];
        }
    }
}

void launch_recover(const BatchView &in, const DeviceTables &tab, const ScanOutputs &scan, const modes_candidate *records,
                    uint32_t capacity, modes_recovered *out, int sm_count, cudaStream_t stream) {
    // one full wave of resident CTAs (the register count decides how many fit; every device here is sm_90a)
    static const int per_sm = [] {
        int b = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, recover_kernel, kRecoverThreads, 0) != cudaSuccess || b < 1) {
            (void)cudaGetLastError();
            b = 4;
        }
        return b;
    }();
    recover_kernel<<<sm_count * per_sm, kRecoverThreads, 0, stream>>>(in, tab.lutn, tab.bit_syn, scan.counters, capacity,
                                                                      records, out);
}

}  // namespace modes
