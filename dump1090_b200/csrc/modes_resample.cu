// modes_resample.cu — K9 (optional): 2.4 MS/s input bytes resampled to the 2 MHz bytes the scan and frame
// evaluation read (modes_set_input_rate, modes_resample_device).  The arithmetic is
// modes_resample_core.cuh; this file only moves bytes.
//
// One block makes a tile of kPeriods polyphase periods (5 output samples from 6 input samples each):
// it stages the tile's input bytes in shared memory with 16-byte loads, each thread evaluates whole
// periods (the taps are immediates, no index arithmetic by 5 or 6), and the block writes the tile's
// output with 16-byte stores.  Tiles start at a period index that is a multiple of 8 (80 output bytes),
// so with the body starting at a multiple of 8 samples every body store is aligned.
//
// 16-bit input (modes_set_input_format, arithmetic in modes_input_core.cuh) is converted, then resampled:
// at 2.4 MS/s K9's staging loader converts each int16 sample to its UC8 pair as it fills s_in, so the
// filter sees exactly the bytes it would see on the converted stream; at 2 MHz K10 (convert_kernel)
// converts the batch's span straight into its body and carry block.  UC8 keeps its own loader, chosen
// at compile time.  The receiver pool's 16-bit receivers have K10's pool form (convert_pool_kernel): one
// launch converts every 16-bit buffer of a call, ahead of the pool's resampling launches.  A device-fed pool
// call (modes_pool_submit_device) moves its 2 MHz receivers' buffers and carries with gather_pool_kernel.
//
// K11 (decimate_kernel): 4, 6, 8 and 10 MS/s input decimated by M = 2..5, in K10's groups of 8 output
// samples, from either staging loader.  K12 (its Shift form): the same with each input sample first
// rotated by the capture's offset from 1090 MHz (modes_set_input_offset).
#include "modes_internal.h"
#include "modes_input_core.cuh"
#include "modes_resample_core.cuh"
#include "modes_stage.cuh"

namespace modes {
namespace {

namespace R = resample;

constexpr int kThreads = 256;
constexpr int kPeriods = 1024;                                   // per tile: 5120 output samples
constexpr int kTileOutBytes = 10 * kPeriods;
constexpr int kTileInSamples = 6 * kPeriods + R::kPeriodIn;
constexpr int kInWords = (2 * kTileInSamples + 15) / 16 + 1;     // + one word of alignment slack

// The tile's periods q0 ... q0 + kPeriods - 1 from its input samples 6 q0 - kLead ... at x (staged in shared
// memory) into s_out; output samples at or past out_end are no signal.
__device__ __forceinline__ void tile_periods(const uint8_t *x_in, uint8_t *s_out, int64_t q0, int64_t out_end) {
    for (int t = threadIdx.x; t < kPeriods; t += kThreads) {
        const uint16_t *x = reinterpret_cast<const uint16_t *>(x_in + 12 * t);
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
        for (int r = 0; r < 5; r++) o[r] = (uint16_t)(n0 + r >= out_end ? 0x7f7fu : y[r]);
    }
}

template <class Input>
__device__ __forceinline__ void resample_tile(const ResampleJob &j, int64_t q_first, const Input &input) {
    __shared__ __align__(16) uint8_t s_in[kInWords * 16];
    __shared__ __align__(16) uint8_t s_out[kTileOutBytes];
    const int64_t q0 = q_first + (int64_t)blockIdx.x * kPeriods;

    // input samples 6 q0 - kLead ... of the tile
    const int64_t off = 2 * (6 * q0 - R::kLead - j.in_first);
    const int64_t a0 = off & ~(int64_t)15;
    const int sh = (int)(off - a0);
    for (int w = threadIdx.x; w < kInWords; w += kThreads)
        *reinterpret_cast<uint4 *>(s_in + 16 * w) = input.word(j, a0 + 16 * (int64_t)w);
    __syncthreads();

    tile_periods(s_in + sh, s_out, q0, j.out_end);
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

__global__ void __launch_bounds__(kThreads) resample_kernel(ResampleJob j, int64_t q_first) {
    resample_tile(j, q_first, Uc8Input{});
}

__global__ void __launch_bounds__(kThreads) resample_sc16_kernel(ResampleJob j, int64_t q_first, int shift) {
    resample_tile(j, q_first, Sc16Input{shift});
}

// K10: 2 MHz int16 input.  Output sample n is input sample n converted, so a thread converts a group of 8
// samples (32 input bytes, two 16-byte loads) into one 16-byte store.  The groups start at g_first
// (8 g_first = out_first, or out_first - 240 with the carry block) and cover the carry block's 240
// samples (the first 2 no signal) and the body; block 0 also writes the block's trailing no-signal bytes.
__global__ void __launch_bounds__(kThreads) convert_kernel(ResampleJob j, int64_t g_first, int64_t n_groups, int shift) {
    if (j.halo && blockIdx.x == 0 && threadIdx.x < (kHaloAlloc - kHaloBytes) / 16)
        reinterpret_cast<uint4 *>(j.halo + kHaloBytes)[threadIdx.x] = make_uint4(0x7f7f7f7fu, 0x7f7f7f7fu, 0x7f7f7f7fu, 0x7f7f7f7fu);
    const int64_t g = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (g >= n_groups) return;
    const int64_t n0 = 8 * (g_first + g);
    uint4 v = Sc16Input{shift}.word(j, 2 * (n0 - j.in_first));
    const int64_t c0 = j.out_first - MODES_CARRY_BYTES / 2;
    if (n0 + 8 > j.out_end || n0 < c0) {
        uint16_t *x = reinterpret_cast<uint16_t *>(&v);
#pragma unroll
        for (int k = 0; k < 8; k++)
            if (n0 + k >= j.out_end || n0 + k < c0) x[k] = 0x7f7fu;
    }
    uint8_t *dst = n0 >= j.out_first ? j.body + 2 * (n0 - j.out_first) : j.halo + 2 * (n0 - (j.out_first - kHaloSamples));
    *reinterpret_cast<uint4 *>(dst) = v;
}

// K11: 4, 6, 8 and 10 MS/s input decimated by M (modes_resample_core.cuh).  The groups are convert_kernel's:
// a thread makes 8 output samples, one 16-byte store into the body or the carry block.  Its group_in(M)
// input samples are consecutive, so it loads the 16-byte words of the (converted) stream that hold them with
// the staging loaders, straight into registers, and aligns them there: the window starts sh bytes into its
// first word, and sh is the same for every group of a launch (groups are 16 M bytes apart).  The taps are
// immediates; neighbouring groups share at most two words, which L1 serves.
//
// K12 (Shift): the same kernel for a capture tuned off 1090 MHz (modes_set_input_offset).  Each sample of the
// window is rotated once, by the phase of its absolute stream index (so batches, shards and GPUs agree with
// nothing carried between them), and the filter runs on the rotated values (shift::shift_group).  The 1024
// rotations sit in shared memory, one word (C, S) each, written by each block from the header's C and S: a
// warp's phases differ from thread to thread unless 8 M step is a multiple of 2^32, which __constant__ would
// serialise.  One word per phase keeps a warp's gather to one wavefront when its phases fall in distinct
// banks; 16-byte entries that also held (-S, C) and both constants cost 1.5-2x K11's time at such offsets on
// an H100, and the same table read with __ldg from global memory no less (DESIGN §3 K12).  Shift = false is
// K11 as it was: step is not read.
template <int M, class Input, bool Shift>
__global__ void __launch_bounds__(kThreads) decimate_kernel(ResampleJob j, int64_t g_first, int64_t n_groups, Input input,
                                                            uint32_t step) {
    namespace D = decimate;
    if (j.halo && blockIdx.x == 0 && threadIdx.x < (kHaloAlloc - kHaloBytes) / 16)
        reinterpret_cast<uint4 *>(j.halo + kHaloBytes)[threadIdx.x] = make_uint4(0x7f7f7f7fu, 0x7f7f7f7fu, 0x7f7f7f7fu, 0x7f7f7f7fu);
    __shared__ uint32_t s_rot[Shift ? shift::kPhases : 1];
    if constexpr (Shift) {
#pragma unroll
        for (int k = threadIdx.x; k < shift::kPhases; k += kThreads) s_rot[k] = shift::rotation(shift::kCos[k], shift::kSin[k]);
        __syncthreads();
    }
    const int64_t g = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (g >= n_groups) return;
    const int64_t n0 = 8 * (g_first + g);
    const int64_t p = 2 * (M * n0 - D::extent(M) - j.in_first);     // the window's first byte
    const int64_t a = p & ~(int64_t)15;
    const int sh = (int)(p - a);
    constexpr int kWords = (2 * D::group_in(M) + 14 + 15) / 16;       // 16-byte words holding the window at any sh
    uint32_t w[4 * kWords + 4];
#pragma unroll
    for (int k = 0; k < kWords; k++) {
        const uint4 v = input.word(j, a + 16 * k);
        w[4 * k] = v.x; w[4 * k + 1] = v.y; w[4 * k + 2] = v.z; w[4 * k + 3] = v.w;
    }
#pragma unroll
    for (int k = 4 * kWords; k < 4 * kWords + 4; k++) w[k] = 0;
    // w[i] = window bytes 4i .. 4i + 3: shift down by sh (even, block-uniform) in three selects
#pragma unroll
    for (int i = 0; i < 4 * kWords + 2; i++) w[i] = (sh & 8) ? w[i + 2] : w[i];
#pragma unroll
    for (int i = 0; i < 4 * kWords + 3; i++) w[i] = (sh & 4) ? w[i + 1] : w[i];
#pragma unroll
    for (int i = 0; i < 4 * kWords + 3; i++) w[i] = (sh & 2) ? __funnelshift_r(w[i], w[i + 1], 16) : w[i];
    uint4 v;
    if constexpr (Shift)
        shift::shift_group<M>(w, s_rot, (uint32_t)(M * n0 - D::extent(M)) * step, step, reinterpret_cast<uint32_t *>(&v));
    else
        D::group<M>(w, reinterpret_cast<uint32_t *>(&v));
    const int64_t c0 = j.out_first - MODES_CARRY_BYTES / 2;
    if (n0 + 8 > j.out_end || n0 < c0) {
        uint16_t *x = reinterpret_cast<uint16_t *>(&v);
#pragma unroll
        for (int k = 0; k < 8; k++)
            if (n0 + k >= j.out_end || n0 + k < c0) x[k] = 0x7f7fu;
    }
    uint8_t *dst = n0 >= j.out_first ? j.body + 2 * (n0 - j.out_first) : j.halo + 2 * (n0 - (j.out_first - kHaloSamples));
    *reinterpret_cast<uint4 *>(dst) = v;
}

// ---- the receiver pool (modes_pool.cpp): one launch for the batch's jobs, grid (tile, job)

constexpr int kCarrySamples = MODES_CARRY_BYTES / 2;
constexpr int64_t kPoolOut = (int64_t)kBufSamples + kCarrySamples;           // samples a job writes
// Tiles of a job: its periods [q_first, q_end), q_first rounded down to a multiple of 8, for any out_first.
constexpr int kPoolTiles = (int)((kPoolOut / 5 + 2 + 8 + kPeriods - 1) / kPeriods);
constexpr int kBufWords = MODES_BUFFER_BYTES / 16;

__global__ void __launch_bounds__(kThreads) resample_pool_kernel(const PoolResampleJob *jobs) {
    __shared__ __align__(16) uint8_t s_in[kInWords * 16];
    __shared__ __align__(16) uint8_t s_out[kTileOutBytes];
    const PoolResampleJob j = jobs[blockIdx.y];
    if (j.out_first < 0) {
        // a 2 MHz receiver: its buffer moves from the staging area to its pair's data buffer as it is
        constexpr int kPer = (kBufWords + kPoolTiles - 1) / kPoolTiles;
        const int w1 = (int)blockIdx.x * kPer + kPer < kBufWords ? (int)blockIdx.x * kPer + kPer : kBufWords;
        for (int w = (int)blockIdx.x * kPer + threadIdx.x; w < w1; w += kThreads)
            reinterpret_cast<uint4 *>(j.data)[w] = __ldg(reinterpret_cast<const uint4 *>(j.stage) + w);
        return;
    }
    const int64_t c0 = j.out_first - kCarrySamples;
    const int64_t q0 = R::floor_div(R::floor_div(c0, 5), 8) * 8 + (int64_t)blockIdx.x * kPeriods;
    if (5 * q0 >= j.out_first + (int64_t)kBufSamples) return;

    // input samples 6 q0 - kLead ... of the tile, stream bytes from a0 (hist0 and call0 are multiples of 16)
    const int64_t s0 = 2 * (6 * q0 - R::kLead);
    const int64_t a0 = s0 & ~(int64_t)15;
    for (int w = threadIdx.x; w < kInWords; w += kThreads)
        *reinterpret_cast<uint4 *>(s_in + 16 * w) = job_word(j, a0 + 16 * (int64_t)w);
    __syncthreads();
    tile_periods(s_in + (int)(s0 - a0), s_out, q0, INT64_MAX);
    __syncthreads();

    // the data buffer: tile and buffer bounds are multiples of 16 bytes apart
    const int64_t tb = 2 * (5 * q0 - j.out_first);
    for (int w = threadIdx.x; w < kTileOutBytes / 16; w += kThreads) {
        const int64_t p = tb + 16 * (int64_t)w;
        if (p >= 0 && p + 16 <= (int64_t)MODES_BUFFER_BYTES)
            *reinterpret_cast<uint4 *>(j.data + p) = *reinterpret_cast<const uint4 *>(s_out + 16 * w);
    }
    // the carry: samples out_first - 238 ... out_first - 1 into the tail of the pair's pad buffer, and
    // nothing else of it (its other bytes stay no signal)
    const int64_t lo = c0 > 5 * q0 ? c0 : 5 * q0;
    const int64_t hi = j.out_first < 5 * q0 + 5 * kPeriods ? j.out_first : 5 * q0 + 5 * kPeriods;
    for (int64_t n = lo + threadIdx.x; n < hi; n += kThreads)
        reinterpret_cast<uint16_t *>(j.pad_tail)[n - c0] = reinterpret_cast<const uint16_t *>(s_out)[n - 5 * q0];
}

constexpr int kHistWordsPerThread = 4;
constexpr int64_t kHistBlockBytes = 16 * kHistWordsPerThread * kThreads;

__global__ void __launch_bounds__(kThreads) history_pool_kernel(const PoolHistoryJob *jobs) {
    const PoolHistoryJob j = jobs[blockIdx.y];
    const int64_t end = j.call0 + MODES_BUFFER_BYTES;
#pragma unroll
    for (int k = 0; k < kHistWordsPerThread; k++) {
        const int64_t p = j.keep + (int64_t)blockIdx.x * kHistBlockBytes + 16 * (int64_t)(k * kThreads + threadIdx.x);
        if (p < end) *reinterpret_cast<uint4 *>(j.out + (p - j.keep)) = job_word(j, p);
    }
}

// K10's pool form: job blockIdx.y's buffer, 8 samples a thread (two 16-byte loads, one 16-byte store) as
// convert_kernel's whole groups; a pool buffer is always whole, so there is no span edge and no carry block.
constexpr int kConvertGroups = MODES_BUFFER_SAMPLES / 8;
constexpr int kConvertBlocks = kConvertGroups / kThreads;
static_assert(kConvertBlocks * kThreads == kConvertGroups, "whole blocks of groups");

__global__ void __launch_bounds__(kThreads) convert_pool_kernel(const PoolConvertJob *jobs) {
    const PoolConvertJob j = jobs[blockIdx.y];
    const int g = (int)blockIdx.x * kThreads + threadIdx.x;
    const uint4 lo = __ldg(reinterpret_cast<const uint4 *>(j.in) + 2 * g);
    const uint4 hi = __ldg(reinterpret_cast<const uint4 *>(j.in) + 2 * g + 1);
    uint4 o;
    o.x = input::convert_pair(lo.x, j.shift) | input::convert_pair(lo.y, j.shift) << 16;
    o.y = input::convert_pair(lo.z, j.shift) | input::convert_pair(lo.w, j.shift) << 16;
    o.z = input::convert_pair(hi.x, j.shift) | input::convert_pair(hi.y, j.shift) << 16;
    o.w = input::convert_pair(hi.z, j.shift) | input::convert_pair(hi.w, j.shift) << 16;
    reinterpret_cast<uint4 *>(j.out)[g] = o;
}

// Device-fed 2 MHz receivers: job blockIdx.y's buffer moves from the caller's memory to its pair in
// kGatherBlocks blocks of 16-byte copies, kGatherWords per thread; block 0 also moves the two carries,
// one 4-byte word per thread (476 bytes: 119 words).
constexpr int kGatherWords = 4;
constexpr int kGatherBlocks = kBufWords / (kGatherWords * kThreads);
static_assert(kGatherBlocks * kGatherWords * kThreads == kBufWords, "whole blocks of words");
constexpr int kCarryWords = MODES_CARRY_BYTES / 4;
static_assert(kCarryWords * 4 == MODES_CARRY_BYTES && kCarryWords <= kThreads, "one carry word per thread");

__global__ void __launch_bounds__(kThreads) gather_pool_kernel(const PoolGatherJob *jobs) {
    const PoolGatherJob j = jobs[blockIdx.y];
    if (j.in) {
        const uint4 *in = reinterpret_cast<const uint4 *>(j.in);
        uint4 *out = reinterpret_cast<uint4 *>(j.data);
        const int w0 = (int)blockIdx.x * kGatherWords * kThreads + threadIdx.x;
        uint4 v[kGatherWords];
#pragma unroll
        for (int k = 0; k < kGatherWords; k++) v[k] = __ldg(in + w0 + k * kThreads);
#pragma unroll
        for (int k = 0; k < kGatherWords; k++) out[w0 + k * kThreads] = v[k];
    }
    if (blockIdx.x != 0 || threadIdx.x >= kCarryWords) return;
    const int t = threadIdx.x;
    const uint32_t *tail = reinterpret_cast<const uint32_t *>((j.in ? j.in : j.data) + MODES_BUFFER_BYTES - MODES_CARRY_BYTES);
    const uint32_t c = j.carry_in ? __ldg(reinterpret_cast<const uint32_t *>(j.carry_in) + t) : 0x7f7f7f7fu;
    reinterpret_cast<uint32_t *>(j.pad_tail)[t] = c;
    reinterpret_cast<uint32_t *>(j.carry_out)[t] = j.in ? __ldg(tail + t) : tail[t];
}

}  // namespace

void launch_gather_pool(const PoolGatherJob *d_jobs, uint32_t n_jobs, cudaStream_t stream) {
    if (n_jobs) gather_pool_kernel<<<dim3(kGatherBlocks, n_jobs), kThreads, 0, stream>>>(d_jobs);
}

void launch_convert_pool(const PoolConvertJob *d_jobs, uint32_t n_jobs, cudaStream_t stream) {
    if (n_jobs) convert_pool_kernel<<<dim3(kConvertBlocks, n_jobs), kThreads, 0, stream>>>(d_jobs);
}

void launch_resample_pool(const PoolResampleJob *d_jobs, uint32_t n_jobs, cudaStream_t stream) {
    if (n_jobs) resample_pool_kernel<<<dim3(kPoolTiles, n_jobs), kThreads, 0, stream>>>(d_jobs);
}

void launch_history_pool(const PoolHistoryJob *d_jobs, uint32_t n_jobs, uint64_t max_bytes, cudaStream_t stream) {
    const unsigned blocks = (unsigned)((max_bytes + kHistBlockBytes - 1) / kHistBlockBytes);
    if (n_jobs && blocks) history_pool_kernel<<<dim3(blocks, n_jobs), kThreads, 0, stream>>>(d_jobs);
}

// K9's tiles for a job: the first period (a multiple of 8) and the number of tiles.
void resample_grid(const ResampleJob &j, int64_t *q_first, unsigned *blocks) {
    const int64_t first = j.out_first - (j.halo ? MODES_CARRY_BYTES / 2 : 0);
    *q_first = R::floor_div(R::floor_div(first, 5), 8) * 8;
    const int64_t q_end = R::floor_div(j.out_first + (int64_t)j.out_samples - 1, 5) + 1;
    *blocks = (unsigned)((q_end - *q_first + kPeriods - 1) / kPeriods);
}

void launch_resample(const ResampleJob &j, cudaStream_t stream) {
    int64_t q_first;
    unsigned blocks;
    resample_grid(j, &q_first, &blocks);
    resample_kernel<<<blocks, kThreads, 0, stream>>>(j, q_first);
}

void launch_resample_sc16(const ResampleJob &j, int shift, cudaStream_t stream) {
    int64_t q_first;
    unsigned blocks;
    resample_grid(j, &q_first, &blocks);
    resample_sc16_kernel<<<blocks, kThreads, 0, stream>>>(j, q_first, shift);
}

void launch_convert_sc16(const ResampleJob &j, int shift, cudaStream_t stream) {
    const int64_t first = j.out_first - (j.halo ? kHaloSamples : 0);
    const int64_t groups = (j.out_first + (int64_t)j.out_samples - first) / 8;
    const int64_t blocks = (groups + kThreads - 1) / kThreads;
    convert_kernel<<<(unsigned)blocks, kThreads, 0, stream>>>(j, first / 8, groups, shift);
}

namespace {
template <int M, bool Shift>
void launch_decimate_m(const ResampleJob &j, int64_t g_first, int64_t groups, int shift, uint32_t step, cudaStream_t stream) {
    const unsigned blocks = (unsigned)((groups + kThreads - 1) / kThreads);
    if (shift < 0) decimate_kernel<M, Uc8Input, Shift><<<blocks, kThreads, 0, stream>>>(j, g_first, groups, Uc8Input{}, step);
    else decimate_kernel<M, Sc16Input, Shift><<<blocks, kThreads, 0, stream>>>(j, g_first, groups, Sc16Input{shift}, step);
}

template <int M>
void launch_decimate_m(const ResampleJob &j, int64_t g_first, int64_t groups, int shift, uint32_t step, cudaStream_t stream) {
    if (step) launch_decimate_m<M, true>(j, g_first, groups, shift, step, stream);
    else launch_decimate_m<M, false>(j, g_first, groups, shift, 0, stream);
}
}  // namespace

void launch_decimate(const ResampleJob &j, int m, int shift, uint32_t step, cudaStream_t stream) {
    const int64_t first = j.out_first - (j.halo ? kHaloSamples : 0);
    const int64_t groups = (j.out_first + (int64_t)j.out_samples - first) / 8;
    switch (m) {
    case 2: launch_decimate_m<2>(j, first / 8, groups, shift, step, stream); break;
    case 3: launch_decimate_m<3>(j, first / 8, groups, shift, step, stream); break;
    case 4: launch_decimate_m<4>(j, first / 8, groups, shift, step, stream); break;
    case 5: launch_decimate_m<5>(j, first / 8, groups, shift, step, stream); break;
    }
}

}  // namespace modes
