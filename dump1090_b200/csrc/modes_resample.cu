// modes_resample.cu — K9 (optional): 2.4 MS/s input bytes resampled to the 2 MHz bytes the scan and frame
// evaluation read (modes_set_input_rate, modes_resample_device).  The arithmetic is
// modes_resample_core.cuh; this file only moves bytes.
//
// One block makes a tile of kPeriods polyphase periods (5 output samples from 6 input samples each):
// it stages the tile's input bytes in shared memory with 16-byte loads, each thread evaluates whole
// periods (the taps are immediates, no index arithmetic by 5 or 6), and the block writes the tile's
// output with 16-byte stores.  Tiles start at a period index that is a multiple of 8 (80 output bytes),
// so with the body starting at a multiple of 8 samples every body store is aligned.
#include "modes_internal.h"
#include "modes_resample_core.cuh"

namespace modes {
namespace {

namespace R = resample;

constexpr int kThreads = 256;
constexpr int kPeriods = 1024;                                   // per tile: 5120 output samples
constexpr int kTileOutBytes = 10 * kPeriods;
constexpr int kTileInSamples = 6 * kPeriods + R::kPeriodIn;
constexpr int kInWords = (2 * kTileInSamples + 15) / 16 + 1;     // + one word of alignment slack

__global__ void __launch_bounds__(kThreads) resample_kernel(ResampleJob j, int64_t q_first) {
    __shared__ __align__(16) uint8_t s_in[kInWords * 16];
    __shared__ __align__(16) uint8_t s_out[kTileOutBytes];
    const int64_t q0 = q_first + (int64_t)blockIdx.x * kPeriods;

    // input samples 6 q0 - kLead ... of the tile; bytes outside the job's span are no signal
    const int64_t off = 2 * (6 * q0 - R::kLead - j.in_first);
    const int64_t a0 = off & ~(int64_t)15;
    const int sh = (int)(off - a0);
    const int64_t in_bytes = (int64_t)j.in_bytes;
    for (int w = threadIdx.x; w < kInWords; w += kThreads) {
        const int64_t p = a0 + 16 * (int64_t)w;
        uint4 v;
        if (p >= 0 && p + 16 <= in_bytes) {
            v = __ldg(reinterpret_cast<const uint4 *>(j.in + p));
        } else {
            uint32_t b[4];
#pragma unroll
            for (int k = 0; k < 4; k++) {
                uint32_t word = 0;
#pragma unroll
                for (int e = 0; e < 4; e++) {
                    const int64_t pe = p + 4 * k + e;
                    const uint32_t x = (pe >= 0 && pe < in_bytes) ? j.in[pe] : 127u;
                    word |= x << (8 * e);
                }
                b[k] = word;
            }
            v = make_uint4(b[0], b[1], b[2], b[3]);
        }
        *reinterpret_cast<uint4 *>(s_in + 16 * w) = v;
    }
    __syncthreads();

    for (int t = threadIdx.x; t < kPeriods; t += kThreads) {
        const uint16_t *x = reinterpret_cast<const uint16_t *>(s_in + sh + 12 * t);
        int xi[R::kPeriodIn], xq[R::kPeriodIn];
#pragma unroll
        for (int k = 0; k < R::kPeriodIn; k++) {
            const uint32_t v = x[k];
            xi[k] = (int)(v & 0xff) - 127;
            xq[k] = (int)(v >> 8) - 127;
        }
        uint32_t y[5];
        R::period(xi, xq, y);
        const int64_t n0 = 5 * (q0 + t);
        uint16_t *o = reinterpret_cast<uint16_t *>(s_out + 10 * t);
#pragma unroll
        for (int r = 0; r < 5; r++) o[r] = (uint16_t)(n0 + r >= j.out_end ? 0x7f7fu : y[r]);
    }
    __syncthreads();

    // the body: tile and body bounds are multiples of 16 bytes apart
    const int64_t tb = 2 * (5 * q0 - j.out_first);
    const int64_t body_bytes = 2 * (int64_t)j.out_samples;
    for (int w = threadIdx.x; w < kTileOutBytes / 16; w += kThreads) {
        const int64_t p = tb + 16 * (int64_t)w;
        if (p >= 0 && p + 16 <= body_bytes)
            *reinterpret_cast<uint4 *>(j.body + p) = *reinterpret_cast<const uint4 *>(s_out + 16 * w);
    }
    // the carry block: samples out_first - 238 ... out_first - 1 at halo[4 ...), no signal around them
    if (j.halo) {
        constexpr int kCarry = MODES_CARRY_BYTES / 2;
        const int64_t c0 = j.out_first - kCarry;
        const int64_t lo = c0 > 5 * q0 ? c0 : 5 * q0;
        const int64_t hi = j.out_first < 5 * q0 + 5 * kPeriods ? j.out_first : 5 * q0 + 5 * kPeriods;
        for (int64_t n = lo + threadIdx.x; n < hi; n += kThreads)
            reinterpret_cast<uint16_t *>(j.halo + kHaloBytes - MODES_CARRY_BYTES)[n - c0] =
                reinterpret_cast<const uint16_t *>(s_out)[n - 5 * q0];
        if (blockIdx.x == 0)
            for (int b = threadIdx.x; b < kHaloAlloc; b += kThreads)
                if (b < kHaloBytes - MODES_CARRY_BYTES || b >= kHaloBytes) j.halo[b] = 127;
    }
}

}  // namespace

void launch_resample(const ResampleJob &j, cudaStream_t stream) {
    const int64_t first = j.out_first - (j.halo ? MODES_CARRY_BYTES / 2 : 0);
    const int64_t q_first = R::floor_div(R::floor_div(first, 5), 8) * 8;
    const int64_t q_end = R::floor_div(j.out_first + (int64_t)j.out_samples - 1, 5) + 1;
    const int64_t blocks = (q_end - q_first + kPeriods - 1) / kPeriods;
    resample_kernel<<<(unsigned)blocks, kThreads, 0, stream>>>(j, q_first);
}

}  // namespace modes
