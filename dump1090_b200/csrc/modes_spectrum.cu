// modes_spectrum.cu — K13 (optional): the input spectrum pass (modes_set_spectrum, modes_pool_set_spectrum).
// For every reference buffer of a batch, the power spectrum of modes_spectrum_core.cuh summed over the
// buffer's frames of its own input, read where the batch already holds it in HBM: the 2 MHz batch bytes, the
// input span a batch at another rate or format was made from (before conversion, resampling, decimation and
// the offset), or a pool receiver's history and call bytes.
//
// Shape: a block of 8 warps takes kFramesPerBlock frames of one buffer (grid (frame group, buffer)); a warp
// takes one frame at a time.  It stages the frame's 512 converted bytes in shared memory with the 16-byte
// loaders K9-K12 use (the next frame's words are loaded before this frame's FFT runs), then runs the 8 stages
// in three passes over a per-warp shared-memory frame: stages 0-2 on 8 consecutive points per lane (read
// windowed and bit-reversed from the staging area), stages 3-5 and 6-7 on points 8 and 64 apart.  Each lane
// keeps its passes' twiddles in registers (the same points every frame) and the power of its 8 output bins
// in 64-bit sums; at the end the block adds its 8 warps' sums and makes one atomic add per bin into the
// buffer's record.  The records are zeroed by the caller.  Only the order of the butterflies within a stage
// differs from the definition's, which leaves every value the same.
#include "modes_internal.h"
#include "modes_input_core.cuh"
#include "modes_resample_core.cuh"
#include "modes_spectrum_core.cuh"
#include "modes_stage.cuh"

namespace modes {
namespace {

namespace SP = spectrum;

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kFramesPerBlock = 8 * kWarps;
constexpr int kStageWords = SP::kN * 2 / 16 + 1;                // a frame's bytes at any even offset in a word
constexpr int kPadded = SP::kN + SP::kN / 8;                      // point m at m + m / 8: conflict-free passes

__device__ __forceinline__ int pad(int m) { return m + (m >> 3); }
__device__ __forceinline__ int tw_c(uint32_t w) { return (int)(int16_t)(w & 0xffffu); }
__device__ __forceinline__ int tw_s(uint32_t w) { return (int)w >> 16; }
__device__ __forceinline__ void bfly(int2 &a, int2 &b, uint32_t w) { SP::butterfly(a.x, a.y, b.x, b.y, tw_c(w), tw_s(w)); }

// A span's buffer: its frames start at stream sample `first`; word(p): the 16 converted bytes at byte p of
// the span (p a multiple of 16 relative to j.in).
template <class Loader>
struct SpanReader {
    ResampleJob j;
    Loader ld;
    int64_t buffer, first;
    uint32_t frames;
    __device__ __forceinline__ int64_t byte_of(int64_t s) const { return 2 * (s - j.in_first); }
    __device__ __forceinline__ uint4 word(int64_t p) const { return ld.word(j, p); }
};

template <class Loader>
struct SpanSource {
    ResampleJob j;
    Loader ld;
    int out, in;
    int64_t first_buffer;
    __device__ __forceinline__ SpanReader<Loader> at(int k) const {
        const int64_t b = first_buffer + k;
        return SpanReader<Loader>{j, ld, b, SP::first_sample(out, in, b), SP::frames(out, in, b)};
    }
};

// A pool job's buffer: stream bytes through job_word, as resample_pool_kernel reads them.
struct PoolReader {
    PoolSpectrumJob j;
    int64_t buffer, first;
    uint32_t frames;
    __device__ __forceinline__ int64_t byte_of(int64_t s) const { return 2 * s; }
    __device__ __forceinline__ uint4 word(int64_t p) const { return job_word(j, p); }
};

struct PoolSource {
    const PoolSpectrumJob *jobs;
    __device__ __forceinline__ PoolReader at(int k) const {
        const PoolSpectrumJob j = jobs[k];
        return PoolReader{j, j.buffer, j.first, j.frames};
    }
};

template <class Source>
__global__ void __launch_bounds__(kThreads) spectrum_kernel(Source src, modes_spectrum *__restrict__ records) {
    __shared__ __align__(16) uint4 s_stage[kWarps][kStageWords];
    __shared__ __align__(16) int2 s_x[kWarps][kPadded];             // also the block's sums at the end
    __shared__ uint32_t s_tw[SP::kN / 2];
    const auto rd = src.at((int)blockIdx.y);
    const uint32_t f0 = blockIdx.x * kFramesPerBlock;
    if (f0 >= rd.frames) return;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    modes_spectrum *rec = records + blockIdx.y;
    if (blockIdx.x == 0 && threadIdx.x == 0) { rec->buffer = rd.buffer; rec->frames = rd.frames; }
    for (int k = threadIdx.x; k < SP::kN / 2; k += kThreads)
        s_tw[k] = (uint32_t)(uint16_t)shift::kCos[4 * k] | (uint32_t)(uint16_t)shift::kSin[4 * k] << 16;
    __syncthreads();

    // pass A: lane L holds points 8 L + i, i.e. samples 32 bitrev3(i) + bitrev5(L), and their windows
    const int rl = SP::bitrev8(lane) >> 3;                          // bitrev5(lane)
    int win[8];
#pragma unroll
    for (int i = 0; i < 8; i++) win[i] = SP::window(shift::kCos[4 * (32 * (SP::bitrev8(i) >> 5) + rl)]);
    const uint32_t wA1 = s_tw[64], wA2[4] = {s_tw[0], s_tw[32], s_tw[64], s_tw[96]};
    // pass B: lane L holds points lo + 8 r + 64 hi (r = 0..7), lo = L & 7, hi = L >> 3
    const int lo = lane & 7, hi = lane >> 3;
    const uint32_t wB3 = s_tw[lo << 4], wB4[2] = {s_tw[lo << 3], s_tw[(lo + 8) << 3]};
    uint32_t wB5[4];
#pragma unroll
    for (int r = 0; r < 4; r++) wB5[r] = s_tw[(lo + 8 * r) << 2];
    // pass C: lane L holds points g + 64 t (t = 0..3) of its groups g = L and L + 32
    uint32_t wC6[2], wC7[2][2];
#pragma unroll
    for (int q = 0; q < 2; q++) {
        const int g = lane + 32 * q;
        wC6[q] = s_tw[g << 1];
        wC7[q][0] = s_tw[g];
        wC7[q][1] = s_tw[g + 64];
    }
    uint64_t acc[2][4] = {};

    const uint32_t f1 = f0 + kFramesPerBlock < rd.frames ? f0 + kFramesPerBlock : rd.frames;
    uint32_t f = f0 + warp;
    uint4 nxt = make_uint4(0, 0, 0, 0), nxt2 = nxt;
    int64_t p = 0, a = 0;
    if (f < f1) {
        p = rd.byte_of(rd.first + (int64_t)SP::kN * f);
        a = p & ~(int64_t)15;
        nxt = rd.word(a + 16 * lane);
        if (lane == 0) nxt2 = rd.word(a + 16 * 32);
    }
    uint4 *stage = s_stage[warp];
    int2 *x = s_x[warp];
    for (; f < f1; f += kWarps) {
        const int sh = (int)(p - a);
        stage[lane] = nxt;
        if (lane == 0) stage[32] = nxt2;
        __syncwarp();
        if (f + kWarps < f1) {                                      // the next frame's words, behind this FFT
            p = rd.byte_of(rd.first + (int64_t)SP::kN * (f + kWarps));
            a = p & ~(int64_t)15;
            nxt = rd.word(a + 16 * lane);
            if (lane == 0) nxt2 = rd.word(a + 16 * 32);
        }
        const uint8_t *bytes = reinterpret_cast<const uint8_t *>(stage) + sh;
        {
            int2 v[8];
#pragma unroll
            for (int i = 0; i < 8; i++) {
                const uint32_t iq = *reinterpret_cast<const uint16_t *>(bytes + 2 * (32 * (SP::bitrev8(i) >> 5) + rl));
                v[i] = make_int2(SP::windowed((int)(iq & 0xff) - 127, win[i]), SP::windowed((int)(iq >> 8) - 127, win[i]));
            }
#pragma unroll
            for (int i = 0; i < 8; i += 2) bfly(v[i], v[i + 1], wA2[0]);
#pragma unroll
            for (int i = 0; i < 8; i += 4) { bfly(v[i], v[i + 2], wA2[0]); bfly(v[i + 1], v[i + 3], wA1); }
#pragma unroll
            for (int i = 0; i < 4; i++) bfly(v[i], v[i + 4], wA2[i]);
#pragma unroll
            for (int i = 0; i < 8; i++) x[pad(8 * lane + i)] = v[i];
        }
        __syncwarp();
        {
            int2 v[8];
#pragma unroll
            for (int r = 0; r < 8; r++) v[r] = x[pad(lo + 8 * r + 64 * hi)];
#pragma unroll
            for (int r = 0; r < 8; r += 2) bfly(v[r], v[r + 1], wB3);
#pragma unroll
            for (int r = 0; r < 8; r += 4) { bfly(v[r], v[r + 2], wB4[0]); bfly(v[r + 1], v[r + 3], wB4[1]); }
#pragma unroll
            for (int r = 0; r < 4; r++) bfly(v[r], v[r + 4], wB5[r]);
#pragma unroll
            for (int r = 0; r < 8; r++) x[pad(lo + 8 * r + 64 * hi)] = v[r];
        }
        __syncwarp();
#pragma unroll
        for (int q = 0; q < 2; q++) {
            const int g = lane + 32 * q;
            int2 v[4];
#pragma unroll
            for (int t = 0; t < 4; t++) v[t] = x[pad(g + 64 * t)];
            bfly(v[0], v[1], wC6[q]);
            bfly(v[2], v[3], wC6[q]);
            bfly(v[0], v[2], wC7[q][0]);
            bfly(v[1], v[3], wC7[q][1]);
#pragma unroll
            for (int t = 0; t < 4; t++) acc[q][t] += SP::power(v[t].x, v[t].y);
        }
        __syncwarp();
    }

    // the block's sums: warp w's bins at red[w][m], then one atomic add per bin
    __syncthreads();
    uint64_t *red = reinterpret_cast<uint64_t *>(&s_x[0][0]);
    static_assert(sizeof(s_x) >= sizeof(uint64_t) * kWarps * SP::kN, "room for the block's sums");
#pragma unroll
    for (int q = 0; q < 2; q++)
#pragma unroll
        for (int t = 0; t < 4; t++) red[warp * SP::kN + lane + 32 * q + 64 * t] = acc[q][t];
    __syncthreads();
    uint64_t sum = 0;
#pragma unroll
    for (int w = 0; w < kWarps; w++) sum += red[w * SP::kN + threadIdx.x];
    if (sum) atomicAdd(reinterpret_cast<unsigned long long *>(&rec->power[SP::bin_of(threadIdx.x)]), (unsigned long long)sum);
}

static_assert(kThreads == SP::kN, "one thread per bin in the block's sums");

}  // namespace

void launch_spectrum(const ResampleJob &j, int shift, int out, int in, int64_t first_buffer, uint32_t n_buffers,
                     modes_spectrum *records, cudaStream_t stream) {
    if (!n_buffers) return;
    const dim3 grid((SP::max_frames(out, in) + kFramesPerBlock - 1) / kFramesPerBlock, n_buffers);
    if (shift < 0) spectrum_kernel<<<grid, kThreads, 0, stream>>>(SpanSource<Uc8Input>{j, Uc8Input{}, out, in, first_buffer}, records);
    else spectrum_kernel<<<grid, kThreads, 0, stream>>>(SpanSource<Sc16Input>{j, Sc16Input{shift}, out, in, first_buffer}, records);
}

void launch_spectrum_pool(const PoolSpectrumJob *d_jobs, uint32_t n_jobs, uint32_t max_frames, modes_spectrum *records,
                          cudaStream_t stream) {
    if (!n_jobs) return;
    const dim3 grid((max_frames + kFramesPerBlock - 1) / kFramesPerBlock, n_jobs);
    spectrum_kernel<<<grid, kThreads, 0, stream>>>(PoolSource{d_jobs}, records);
}

}  // namespace modes
