// modes_weak.cu — the weak-preamble scan (modes_set_weak_preambles, modes_weak_device): every
// position of a batch tested against the weak-preamble definition of include/modes_b200.h
// (arithmetic in modes_weak_core.cuh), the passing positions written as one list in stream order.
//
// One pass over the batch while it is in HBM, on the same virtual sample array as the scan
// (BatchView: carry block + body).  It is a separate kernel so that, with the feature off, nothing
// about the default kernels changes.
//
// Shape, modelled on the level pass: the magnitude table (lutn, 64 KB) is staged in shared memory
// once per CTA.  The CTAs (one wave) take tiles of 4096 positions in turn (tile b + k * gridDim.x);
// a CTA reads the tile's samples plus 28 more with 16-byte loads (issued one tile ahead, into registers)
// and turns them into magnitudes in shared memory (a layout skewed by one word in nine, so that the
// per-thread windows below are read without bank conflicts).  Only the buffers first_buffer +
// i * buffer_step are scanned (the receiver pool skips its pad buffers); tile k of the scan is tile
// k % 32 of the k / 32-th of them.  Thread i owns positions 16i .. 16i+15 of the tile: it tests conditions 1 and 2 on a
// 30-sample window held in registers, and conditions 3 and 4 on the few survivors from shared memory.
//
// Stream order without a sort: a tile's passing positions are counted (a block-wide scan) and written,
// in order, to a block of a scratch list reserved with one atomic; the tile records where its block
// is and how long.  weak_order_kernel (one CTA) turns the tiles' counts into their offsets in the
// output list (an exclusive scan over the tiles in stream order), and weak_gather_kernel (a thread
// per tile) copies every tile's block there.  So the output list is identical from run to run, also
// when the batch is repeated, although the scratch list's layout is not.  The count (the atomic's
// total) is exact; positions past the capacity are not written.  A scratch list that overflowed is
// reported through the count, and then nothing at all is written to the output list (the caller
// repeats the batch with a larger scratch list).
#include <cstdint>
#include <cuda_runtime.h>
#include "modes_internal.h"
#include "modes_weak_core.cuh"

namespace modes {
namespace {

constexpr int kWeakThreads = 256;
constexpr int kWeakWarps = kWeakThreads / 32;
constexpr int kWeakPer = 16;                                    // positions per thread and tile
static_assert(kWeakTileSamples == kWeakThreads * kWeakPer, "tile geometry");
static_assert(kBufSamples % kWeakTileSamples == 0, "tiles never straddle a buffer");
// a position's m[j] is virtual sample t + 2; the tile reads virtual samples [t0, t0 + 4096 + 28)
constexpr int kWeakChunks = (kWeakTileSamples + 2 + weak::kWindow + 7) / 8;    // 8-sample (16-byte) chunks: 516
constexpr int kWeakWords = 4 * kWeakChunks;                     // magnitude words (two samples each)
constexpr int kWeakSmemWords = kWeakWords + kWeakWords / 8 + 1;
constexpr int kWeakWinWords = 15;                               // a thread's window: samples 16i+2 .. 16i+31
constexpr int kWeakLutBytes = (kNLutEntries * 2 + 15) / 16 * 16;
constexpr int kOrderThreads = 1024;

__device__ __forceinline__ int skew(int w) { return w + (w >> 3); }

// The window of conditions 1 and 2: magnitudes of 30 consecutive samples, two per register.
struct RegWindow {
    const uint32_t *w;
    __device__ __forceinline__ uint32_t operator[](int x) const { return (w[x >> 1] >> (16 * (x & 1))) & 0xffffu; }
};

// Samples from the shared tile (conditions 3 and 4 of a survivor): x is relative to sample `base`.
struct SmemWindow {
    const uint32_t *words;
    int base;
    __device__ __forceinline__ uint32_t operator[](int x) const {
        const int s = base + x;
        return (words[skew(s >> 1)] >> (16 * (s & 1))) & 0xffffu;
    }
};

// Chunk c of the virtual sample array; chunks past the end read as no signal.
__device__ __forceinline__ uint4 load_chunk(const BatchView &in, uint64_t c, uint64_t n_vchunks) {
    if (c >= n_vchunks) return make_uint4(0x7f7f7f7fu, 0x7f7f7f7fu, 0x7f7f7f7fu, 0x7f7f7f7fu);
    const uint4 *p = (c < kHaloSamples / 8) ? reinterpret_cast<const uint4 *>(in.halo) + c
                                            : reinterpret_cast<const uint4 *>(in.body) + (c - kHaloSamples / 8);
    return __ldcs(p);
}

__global__ void __launch_bounds__(kWeakThreads)
weak_scan_kernel(BatchView in, const uint16_t *__restrict__ lutn, uint32_t n_tiles, uint32_t first_buffer, uint32_t buffer_step,
                 uint32_t *tile_src, uint32_t *tile_count, uint32_t *counters, uint32_t *scratch, uint32_t scratch_cap) {
    extern __shared__ uint4 s_raw[];
    const uint16_t *s_lut = reinterpret_cast<const uint16_t *>(s_raw);
    __shared__ uint32_t s_words[kWeakSmemWords];
    __shared__ uint32_t s_warp[kWeakWarps];
    __shared__ uint32_t s_base;
    constexpr int kLoads = (kWeakChunks + kWeakThreads - 1) / kWeakThreads;    // chunks per thread and tile: 3
    for (int i = threadIdx.x; i < (kNLutEntries - 1) / 8; i += kWeakThreads) s_raw[i] = __ldg(reinterpret_cast<const uint4 *>(lutn) + i);
    if (threadIdx.x == 0) reinterpret_cast<uint16_t *>(s_raw)[kNLutEntries - 1] = lutn[kNLutEntries - 1];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint64_t n_vchunks = (in.n_samples + kHaloSamples) / 8;
    const uint32_t full = 0xffffffffu;
    constexpr uint32_t kTilesPerBuffer = kBufSamples / kWeakTileSamples;
    // the batch tile of scan tile k
    auto batch_tile = [&](uint32_t k) { return (first_buffer + (k / kTilesPerBuffer) * buffer_step) * kTilesPerBuffer + k % kTilesPerBuffer; };
    // the samples of a tile: virtual samples [t0, t0 + 8 * kWeakChunks), t0 = the tile's first position;
    // the next tile's loads are issued before the current tile is tested, so that they are in flight
    // during its tests
    uint4 pre[kLoads];
    auto load_tile = [&](uint32_t tile) {
        const uint64_t c0 = (uint64_t)batch_tile(tile) * (kWeakTileSamples / 8);
#pragma unroll
        for (int k = 0; k < kLoads; k++) {
            const int c = tid + k * kWeakThreads;
            if (tile < n_tiles && c < kWeakChunks) pre[k] = load_chunk(in, c0 + c, n_vchunks);
        }
    };
    // A tile's block of the scratch list is reserved with one atomic, whose result is used only in the
    // next round, after the next tile's magnitudes are staged: the atomic is off the critical path.  The
    // tile's positions wait in registers (its mask, first position and offset inside the tile).
    uint32_t prev_tile = UINT32_MAX, prev_total = 0, prev_base = 0;        // prev_base: thread 0 only
    uint32_t prev_keep = 0, prev_t0 = 0, prev_off = 0;
    auto flush = [&]() {                                                   // before: s_base set, a barrier
        uint32_t at = s_base + prev_off;
        for (uint32_t r = prev_keep; r; r &= r - 1u, at++)
            if (at < scratch_cap) scratch[at] = prev_t0 + (uint32_t)(__ffs(r) - 1);
    };
    auto publish = [&]() {                                                 // thread 0, before a barrier
        s_base = prev_base;
        tile_src[prev_tile] = prev_base;
        tile_count[prev_tile] = prev_total;
    };
    uint32_t tile = blockIdx.x;                                            // tiles blockIdx.x + k * gridDim.x
    __syncthreads();                                                       // the table is staged
    load_tile(tile);
    for (; tile < n_tiles; tile += gridDim.x) {
#pragma unroll
        for (int k = 0; k < kLoads; k++) {
            const int c = tid + k * kWeakThreads;
            if (c < kWeakChunks) {
                uint32_t *d = s_words + skew(4 * c);            // the four words of a chunk share one skew group
                d[0] = weak::word_mags(pre[k].x, s_lut); d[1] = weak::word_mags(pre[k].y, s_lut);
                d[2] = weak::word_mags(pre[k].z, s_lut); d[3] = weak::word_mags(pre[k].w, s_lut);
            }
        }
        if (tid == 0 && prev_tile != UINT32_MAX) publish();
        __syncthreads();
        if (prev_tile != UINT32_MAX) flush();
        load_tile(tile + gridDim.x);
        // conditions 1 and 2 for this thread's 16 positions: window = samples 16 tid + 2 .. + 31
        uint32_t win[kWeakWinWords];
#pragma unroll
        for (int k = 0; k < kWeakWinWords; k++) win[k] = s_words[skew(8 * tid + 1 + k)];
        const RegWindow rw{win};
        uint32_t mask = 0;
#pragma unroll
        for (int s = 0; s < kWeakPer; s++) mask |= weak::shape_and_contrast(rw, s) ? 1u << s : 0u;
        const uint32_t t0 = batch_tile(tile) * (uint32_t)kWeakTileSamples + (uint32_t)(kWeakPer * tid);
        const uint32_t j0 = t0 & (kBufSamples - 1);
        if (j0 + kWeakPer > kScanLimit) mask &= (1u << (kScanLimit - j0)) - 1u;      // j < 131070 (dump1090.c:1593)
        // conditions 3 and 4 for the survivors
        uint32_t keep = 0;
        for (uint32_t r = mask; r; r &= r - 1u) {
            const int s = __ffs(r) - 1;
            if (weak::weak_rest(SmemWindow{s_words, kWeakPer * tid + 2 + s}, 0)) keep |= 1u << s;
        }
        // the thread's offset inside the tile, and the tile's count
        const uint32_t cnt = __popc(keep);
        uint32_t incl = cnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t x = __shfl_up_sync(full, incl, o);
            if (lane >= o) incl += x;
        }
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();
        uint32_t before = 0, total = 0;
#pragma unroll
        for (int w = 0; w < kWeakWarps; w++) {
            const uint32_t x = s_warp[w];
            before += w < warp ? x : 0u;
            total += x;
        }
        if (tid == 0) prev_base = total ? atomicAdd(counters + 1, total) : 0u;
        prev_tile = tile; prev_total = total;
        prev_keep = keep; prev_t0 = t0; prev_off = before + (incl - cnt);
    }
    if (prev_tile != UINT32_MAX) {
        if (tid == 0) publish();
        __syncthreads();
        flush();
    }
}

// The tiles' offsets in the output list: an exclusive scan of their counts in stream order (one CTA).
// Each round covers 16 tiles per thread, read and written as four 16-byte words (n_tiles is a multiple
// of 32), so the loads are coalesced and few rounds are needed.
__global__ void __launch_bounds__(kOrderThreads)
weak_order_kernel(const uint32_t *tile_count, uint32_t n_tiles, uint32_t *tile_dst) {
    __shared__ uint32_t s_warp[kOrderThreads / 32];
    __shared__ uint32_t s_carry;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr uint32_t kPer = 16, kRound = kPer * kOrderThreads;
    if (tid == 0) s_carry = 0;
    const uint4 *in4 = reinterpret_cast<const uint4 *>(tile_count);
    uint4 *out4 = reinterpret_cast<uint4 *>(tile_dst);
    for (uint32_t base = 0; base < n_tiles; base += kRound) {
        uint4 v[4];
        uint32_t sum = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const uint32_t t = base + kPer * tid + 4 * k;
            v[k] = t < n_tiles ? in4[t / 4] : make_uint4(0, 0, 0, 0);
            sum += v[k].x + v[k].y + v[k].z + v[k].w;
        }
        uint32_t incl = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t x = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += x;
        }
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();                                    // also: s_carry of the last round is final
        uint32_t at = s_carry + incl - sum, round_total = 0;
        for (int w = 0; w < kOrderThreads / 32; w++) {
            const uint32_t x = s_warp[w];
            at += w < warp ? x : 0u;
            round_total += x;
        }
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const uint32_t t = base + kPer * tid + 4 * k;
            uint4 d;
            d.x = at; at += v[k].x;
            d.y = at; at += v[k].y;
            d.z = at; at += v[k].z;
            d.w = at; at += v[k].w;
            if (t < n_tiles) out4[t / 4] = d;
        }
        __syncthreads();                                    // every thread has read s_carry and s_warp
        if (tid == 0) s_carry += round_total;
    }
}

// Every tile's block of the scratch list to its place in the output list (a thread per tile); nothing
// when the scratch list overflowed.
__global__ void weak_gather_kernel(const uint32_t *tile_src, const uint32_t *tile_count, const uint32_t *tile_dst,
                                   uint32_t n_tiles, const uint32_t *counters, const uint32_t *scratch, uint32_t scratch_cap,
                                   uint32_t *out, uint32_t capacity) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_tiles || counters[1] > scratch_cap) return;
    const uint32_t src = tile_src[t], n = tile_count[t], dst = tile_dst[t];
    for (uint32_t e = 0; e < n && dst + e < capacity; e++) out[dst + e] = scratch[src + e];
}

}  // namespace

void launch_weak_scan(const BatchView &in, const DeviceTables &tab, const WeakOutputs &out, int sm_count, cudaStream_t stream) {
    const uint32_t n_tiles = weak_tiles_for(out.n_buffers);
    uint32_t *tile_src = out.tiles, *tile_count = out.tiles + n_tiles, *tile_dst = out.tiles + 2 * (size_t)n_tiles;
    cudaMemsetAsync(out.counters, 0, 2 * sizeof(uint32_t), stream);
    if (!n_tiles) return;
    // the opt-in to > 48 KB of dynamic shared memory is per device
    static bool configured[64] = {};
    static int per_sm[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) dev = 0;
    if (!configured[dev]) {
        cudaFuncSetAttribute(weak_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kWeakLutBytes);
        int b = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, weak_scan_kernel, kWeakThreads, kWeakLutBytes) != cudaSuccess || b < 1) {
            (void)cudaGetLastError();
            b = 1;
        }
        per_sm[dev] = b;
        configured[dev] = true;
    }
    // one wave: every CTA stages the table once and then takes tiles until none are left
    const uint32_t most = (uint32_t)sm_count * (uint32_t)per_sm[dev];
    weak_scan_kernel<<<n_tiles < most ? n_tiles : most, kWeakThreads, kWeakLutBytes, stream>>>(
        in, tab.lutn, n_tiles, out.first_buffer, out.buffer_step, tile_src, tile_count, out.counters, out.scratch, out.scratch_cap);
    weak_order_kernel<<<1, kOrderThreads, 0, stream>>>(tile_count, n_tiles, tile_dst);
    weak_gather_kernel<<<(n_tiles + 255) / 256, 256, 0, stream>>>(tile_src, tile_count, tile_dst, n_tiles, out.counters,
                                                                  out.scratch, out.scratch_cap, out.pos, out.capacity);
}

}  // namespace modes
