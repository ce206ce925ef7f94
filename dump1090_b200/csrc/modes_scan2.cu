// modes_scan2.cu — K1, the fused magnitude + preamble scan kernel (sm_90a).
//
// Replaces computeMagnitudeVector (dump1090.c:1454-1469) and the per-position tests of
// detectModeS (dump1090.c:1602-1650).  HBM-bound by design: 2 bytes read per sample, nothing
// written but the sparse candidate list; in practice the limit is the integer instruction rate,
// so the kernel is built around instructions per sample (modes_scan_core.cuh has the arithmetic)
// and around a loop body small enough to stay in the instruction cache.
//
// Work split.  One warp owns a tile of 7936 positions and walks it in 8 self-contained rows.  A
// row is 2 KB of I/Q = 1024 samples read as four 16-byte loads per lane (lane l: samples
// 32l .. 32l+31 of the row); lanes 0..30 each produce the pass flags of their 32 positions, lane
// 31 only supplies the 10 samples of lookahead lane 30 needs — its own positions belong to lane 0
// of the next row, which starts 31*32 = 992 samples later.  Paying 1/32 of redundant arithmetic
// removes every dependency between rows: a lane's lookahead is always the first five packed
// words of the next lane (one shuffle each), rows can be loaded and processed in any order, and
// the row step is one compact rolled loop: pack, reload the same registers with the next row,
// shuffle, compare.
//
// The 32-bit flag words go through 1 KB of shared memory so that lane j then holds 256
// consecutive positions; survivors of the ten comparisons (~1 % of positions) get the exact
// "high" tests of dump1090.c:1624-1642 on table magnitudes, 32 at a time from a queue of the
// non-empty flag words, their samples re-read through L1 where the row loads have just put them.  Tiles are handed out from a
// global counter, requested one tile ahead; a tile's slot in the candidate array costs one atomic,
// issued a tile before it is used.
#include <cstdint>
#include <cstdlib>
#include <cuda_runtime.h>
#include "modes_internal.h"
#include "modes_scan_core.cuh"

namespace modes {
namespace {

constexpr int kRows = kTileSamples / (31 * 32);          // rows per tile: 8
constexpr int kRowFresh = 31 * 32;                       // positions a row decides
constexpr int kTile = kRows * kRowFresh;                 // 7936 positions
constexpr int kRowStrideChunks = kRowFresh / 8;          // 124 16-byte chunks between row starts
constexpr int kTileChunks = kTile / 8;                   // 992
constexpr int kTileReach = (kRows - 1) * kRowStrideChunks + 128;   // chunks a tile's rows read: 996
constexpr int kEntryCap = 256;                           // non-empty flag words per tile the fast path holds
constexpr int kSurvivorCap = 512;                        // survivors per tile the fast path holds (dense path: per round)
constexpr int kOutCap = 256;                             // candidates per tile held back one tile
constexpr int kExactRounds = 3;                          // rounds of 32 exact tests whose loads are in flight together
static_assert(kTile == kTileSamples && kRows % 4 == 0 && 32 % kRows == 0, "tile geometry");

struct TileSrc {
    const uint4 *flat;           // chunk 0 of the tile when every row lies inside the body
    uint64_t c0;                 // first virtual chunk of the tile
    bool interior;
};

__device__ __forceinline__ TileSrc tile_source(const BatchView &in, uint32_t g, uint64_t n_vchunks) {
    TileSrc ts;
    ts.c0 = (uint64_t)g * kTileChunks;
    ts.interior = ts.c0 >= kHaloSamples / 8 && ts.c0 + kTileReach <= n_vchunks;
    ts.flat = reinterpret_cast<const uint4 *>(in.body) + (ts.c0 - kHaloSamples / 8);
    return ts;
}

// Chunk c of the virtual sample array (carry block, then the body); chunks past the end read as
// "no signal" (127,127).  Only the first and the last tiles of a batch come here.
// (Out-of-line helpers take plain values: a reference to a kernel-parameter struct or to a register
// array would force a copy in local memory, read back through L1 in the hot path.)
// The carry block may be the kernel's parameter: a generic load, not __ldg (global space only).
__device__ __noinline__ uint4 load_vchunk(const uint8_t *body, const uint8_t *halo, uint64_t c, uint64_t n_vchunks) {
    if (c >= n_vchunks) return make_uint4(0x7f7f7f7fu, 0x7f7f7f7fu, 0x7f7f7f7fu, 0x7f7f7f7fu);
    if (c < kHaloSamples / 8) return reinterpret_cast<const uint4 *>(halo)[c];
    return __ldg(reinterpret_cast<const uint4 *>(body) + (c - kHaloSamples / 8));
}

// Row r of a tile: this lane's 64 bytes.  Loaded through L1 (no L1::no_allocate): the exact tests
// re-read a few of the samples.
__device__ __forceinline__ void load_row(const BatchView &in, const TileSrc &t, int r, int lane, uint64_t n_vchunks, uint4 x[4]) {
    const int chunk = kRowStrideChunks * r + 4 * lane;
    if (t.interior) {
        const uint4 *p = t.flat + chunk;
        x[0] = __ldg(p); x[1] = __ldg(p + 1); x[2] = __ldg(p + 2); x[3] = __ldg(p + 3);
    } else {
#pragma unroll 1
        for (int k = 0; k < 4; k++) {
            const uint4 v = load_vchunk(in.body, in.halo, t.c0 + chunk + k, n_vchunks);
            if (k == 0) x[0] = v; else if (k == 1) x[1] = v; else if (k == 2) x[2] = v; else x[3] = v;
        }
    }
}

// Squared magnitude of one sample (I in byte 0, Q in byte 1, upper bytes zero: they come out of
// the byte-wise |x - 127| as 127 each, which the dot product's addend takes off again).
__device__ __forceinline__ uint32_t n_of(uint32_t iq16) {
    const uint32_t a = __vabsdiffu4(iq16, 0x7f7f7f7fu);
    return __dp4a(a, a, (uint32_t)(-2 * 127 * 127));
}

// dump1090.c:1624-1642 on exact magnitudes, given the squared magnitudes of m0, m2, m7, m9 and the
// largest of m4, m5, m11..m14:   high = (m0+m2+m7+m9)/6;  m4, m5, m11..m14 < high
// <=> 6*(max(m4,m5,m11..m14)+1) <= m0+m2+m7+m9.  The magnitude table is monotone in the squared
// magnitude, so the max is taken before the lookup: five lookups instead of ten.
__device__ __forceinline__ bool high_rule(uint32_t n0, uint32_t n2, uint32_t n7, uint32_t n9, uint32_t nx,
                                          const uint16_t *__restrict__ lutn) {
    const int sum = (int)__ldg(lutn + n0) + (int)__ldg(lutn + n2) + (int)__ldg(lutn + n7) + (int)__ldg(lutn + n9);
    const int mx = __ldg(lutn + nx);
    return 6 * (mx + 1) <= sum;
}

// The exact tests for the position whose first sample is at p (interior tiles: samples re-read
// through L1, where the row loads have just put them).
__device__ __forceinline__ bool high_tests_at(const uint16_t *__restrict__ p, const uint16_t *__restrict__ lutn) {
    const uint32_t n0 = n_of(__ldg(p)), n2 = n_of(__ldg(p + 2)), n7 = n_of(__ldg(p + 7)), n9 = n_of(__ldg(p + 9));
    const uint32_t n4 = n_of(__ldg(p + 4)), n5 = n_of(__ldg(p + 5)), n11 = n_of(__ldg(p + 11));
    const uint32_t n12 = n_of(__ldg(p + 12)), n13 = n_of(__ldg(p + 13)), n14 = n_of(__ldg(p + 14));
    return high_rule(n0, n2, n7, n9, max(max(max(n4, n5), max(n11, n12)), max(n13, n14)), lutn);
}

// The same for the first and last tiles of a batch (carry block, end of data), sample by sample.
__device__ __noinline__ bool high_tests_edge(const uint8_t *body, const uint8_t *halo, uint64_t n_samples, uint64_t v,
                                             const uint16_t *__restrict__ lutn) {
    uint32_t n[15];
#pragma unroll
    for (int d = 0; d < 15; d++) {
        const uint64_t vd = v + d;
        const uint8_t *p = (vd < (uint64_t)kHaloSamples) ? halo + 2 * vd : body + 2 * (vd - kHaloSamples);
        n[d] = n_of(vd < n_samples + kHaloSamples ? *reinterpret_cast<const uint16_t *>(p) : 0x7f7fu);
    }
    return high_rule(n[0], n[2], n[7], n[9], max(max(max(n[4], n[5]), max(n[11], n[12])), max(n[13], n[14])), lutn);
}

__device__ __forceinline__ bool high_tests(const BatchView &in, const TileSrc &t, int s, const uint16_t *__restrict__ lutn) {
    if (t.interior) return high_tests_at(reinterpret_cast<const uint16_t *>(t.flat) + s, lutn);
    return high_tests_edge(in.body, in.halo, in.n_samples, t.c0 * 8 + (uint64_t)s, lutn);
}

// This lane's survivors (bit i of w[q] = tile position base + 32q + i) -> the slots [excl, excl+cnt)
// of the tile-ordered survivor sequence; those in [round, round+kSurvivorCap) are listed.
__device__ __forceinline__ void list_survivors(const uint32_t w[kRows], int base, uint32_t excl, uint32_t round, uint16_t *surv) {
    uint32_t slot = excl - round;
#pragma unroll
    for (int q = 0; q < kRows; q++)
        for (uint32_t b = w[q]; b; b &= b - 1) {
            if (slot < (uint32_t)kSurvivorCap) surv[slot] = (uint16_t)(base + 32 * q + __ffs(b) - 1);
            slot++;
        }
}

// Copy a finished tile's candidate list (tile-local positions, position order) to its slot in the
// global candidate array and record the tile.  `base0` is the slot claimed one tile earlier.
__device__ __forceinline__ void emit_tile(const ScanOutputs &out, const uint16_t *olist, uint32_t tile, uint32_t base0,
                                          uint32_t total, int lane) {
    const uint32_t base = __shfl_sync(0xffffffffu, base0, 0);
    const uint32_t v0 = tile * (uint32_t)kTile;
    for (uint32_t i = lane; i < total; i += 32)
        if (base + i < out.cand_capacity) out.cand_v[base + i] = v0 + olist[i];
    if (lane == 0) {
        uint32_t stored = total;
        if (base + total > out.cand_capacity) {
            stored = base < out.cand_capacity ? out.cand_capacity - base : 0;
            out.counters[1] = 1;
        }
        modes_tile tl; tl.offset = base; tl.count = stored;
        out.tiles[tile] = tl;
    }
}

// A tile with more survivors or candidates than the fast path's buffers hold (periodic input that
// makes nearly every position a preamble): count, claim a slot in the candidate array, then write
// the candidates straight to it, survivors listed kSurvivorCap at a time.  Out of line: never
// executed on real traffic, and the hot loop should stay small.  The (validity-masked) flag words
// are handed over in shared memory, lane j's at s_words[kRows*j ..].
__device__ __noinline__ void dense_tile(const uint8_t *body, const uint8_t *halo, uint64_t n_samples, uint64_t n_vchunks,
                                        const uint16_t *__restrict__ lutn, uint32_t *cand_v, uint32_t cand_capacity,
                                        modes_tile *tiles, uint32_t *counters, uint32_t g, const uint32_t *s_words,
                                        uint16_t *surv, int lane) {
    const BatchView in{body, halo, n_samples};
    const TileSrc ts = tile_source(in, g, n_vchunks);
    uint32_t w[kRows];
    uint32_t cnt = 0;
#pragma unroll
    for (int q = 0; q < kRows; q++) { w[q] = s_words[kRows * lane + q]; cnt += __popc(w[q]); }
    uint32_t incl = cnt;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t o = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += o;
    }
    const uint32_t n_surv = __shfl_sync(0xffffffffu, incl, 31), excl = incl - cnt;
    const int base = kRowFresh * ((kRows * lane) >> 5) + 32 * ((kRows * lane) & 31);
    const uint32_t v_tile = g * (uint32_t)kTile;
    uint32_t total = 0;
    for (int pass_no = 0; pass_no < 2; pass_no++) {
        uint32_t gbase = 0, run = 0;
        if (pass_no == 1) {
            if (lane == 0 && total) gbase = atomicAdd(&counters[0], total);
            gbase = __shfl_sync(0xffffffffu, gbase, 0);
        }
        for (uint32_t round = 0; round < n_surv; round += kSurvivorCap) {
            __syncwarp();
            list_survivors(w, base, excl, round, surv);
            __syncwarp();
            const uint32_t n_here = min(n_surv - round, (uint32_t)kSurvivorCap);
            for (uint32_t i0 = 0; i0 < n_here; i0 += 32) {
                const uint32_t i = i0 + lane;
                const int spos = i < n_here ? surv[i] : 0;
                const bool pass = i < n_here && high_tests(in, ts, spos, lutn);
                const uint32_t bal = __ballot_sync(0xffffffffu, pass);
                if (pass_no == 1 && pass) {
                    const uint32_t idx = gbase + run + __popc(bal & ((1u << lane) - 1u));
                    if (idx < cand_capacity) cand_v[idx] = v_tile + spos;
                }
                run += __popc(bal);
            }
        }
        if (pass_no == 0) total = run;
        else if (lane == 0) {
            uint32_t stored = total;
            if (gbase + total > cand_capacity) {
                stored = gbase < cand_capacity ? cand_capacity - gbase : 0;
                counters[1] = 1;
            }
            modes_tile tl; tl.offset = gbase; tl.count = stored;
            tiles[g] = tl;
        }
    }
    __syncwarp();
}

struct alignas(16) CarryBlock { uint8_t b[kHaloAlloc]; };

// 12 warps per SM (3 per scheduler) at up to 168 registers: the kernel needs about 160 and then has no
// spill.  On the H100 that is faster than 16 warps at the 128-register cap with a spill (DESIGN §6).
// carry_in_param: the batch's carry block is `carry`, and CTA 0 stores it to batch.halo for the kernels
// after this one; else it is read at batch.halo.
__global__ void __launch_bounds__(32, 12)
scan_kernel(BatchView batch, __grid_constant__ const CarryBlock carry, uint32_t carry_in_param,
            const uint16_t *__restrict__ lutn, ScanOutputs out, uint32_t n_tiles, uint32_t one, uint32_t minus_one,
            uint32_t c65536) {
    __shared__ __align__(16) uint32_t s_mask[kRows * 32];
    __shared__ __align__(16) uint2 s_entry[kEntryCap];                // non-empty flag words: {word, position of bit 0 | first survivor slot << 16}
    __shared__ __align__(16) uint16_t s_surv[kSurvivorCap];           // survivor positions, position order
    __shared__ __align__(16) uint16_t s_olist[2 * kOutCap];
    uint32_t pend_tile = 0xffffffffu, pend_base = 0, pend_total = 0, pend_buf = 0;

    const int lane = threadIdx.x;
    const BatchView in{batch.body, carry_in_param ? carry.b : batch.halo, batch.n_samples};
    if (blockIdx.x == 0) {
        static_assert(kHaloAlloc == 32 * 16 && kCounterWords <= 32, "one 16-byte carry chunk and one counter per lane");
        if (carry_in_param)
            reinterpret_cast<uint4 *>(const_cast<uint8_t *>(batch.halo))[lane] = reinterpret_cast<const uint4 *>(carry.b)[lane];
        if (out.next_counters && lane < kCounterWords) out.next_counters[lane] = 0u;
    }
    const uint32_t lt_mask = (1u << lane) - 1u;
    const uint64_t n_vchunks = (in.n_samples + kHaloSamples) / 8;
    const uint64_t t_end = in.n_samples;

    uint32_t g = blockIdx.x;
    if (g >= n_tiles) return;
    TileSrc ts = tile_source(in, g, n_vchunks);
    uint4 x[8];                                           // the two rows in flight / being packed
    load_row(in, ts, 0, lane, n_vchunks, x);
    load_row(in, ts, 1, lane, n_vchunks, x + 4);

    // Tiles are handed out first come, first served (after one static tile per warp); the index
    // is requested a whole tile before it is needed, so the atomic's latency is never waited for.
    // (The returned counter is used untouched until the next tile: any arithmetic on it here would
    // wait for the atomic's round trip.)
    uint32_t g_ahead = 0;
    if (lane == 0) g_ahead = atomicAdd(&out.counters[2], 1u);

    for (int it = 0; g < n_tiles; ++it) {
        const int cur = it & 1;
        const TileSrc ts_cur = ts;
        const uint32_t g_next = gridDim.x + __shfl_sync(0xffffffffu, g_ahead, 0);
        // Both atomics of a tile are issued here, with the whole row loop between them and their
        // consumers: the request for the tile after next, and the previous tile's slot in the
        // candidate array (its list is copied out after this tile's rows).
        if (lane == 0) {
            if (g_next < n_tiles) g_ahead = atomicAdd(&out.counters[2], 1u);
            if (pend_tile != 0xffffffffu && pend_total) pend_base = atomicAdd(&out.counters[0], pend_total);
        }
        if (g_next < n_tiles) ts = tile_source(in, g_next, n_vchunks);

        // ---- the rows, two at a time (the halves of a register hold the same sample of both rows).
        // The registers the rows arrived in are reloaded with the next two as soon as they are
        // packed: that load has the whole comparison phase to complete.
#pragma unroll 1
        for (int r = 0; r < kRows; r += 2) {
            uint32_t X[32 + scan2::kPairLook];
#pragma unroll
            for (int p = 0; p < 4; p++) {
                scan2::npack2(x[p].x, x[4 + p].x, c65536, minus_one, X[8 * p + 0], X[8 * p + 1]);
                scan2::npack2(x[p].y, x[4 + p].y, c65536, minus_one, X[8 * p + 2], X[8 * p + 3]);
                scan2::npack2(x[p].z, x[4 + p].z, c65536, minus_one, X[8 * p + 4], X[8 * p + 5]);
                scan2::npack2(x[p].w, x[4 + p].w, c65536, minus_one, X[8 * p + 6], X[8 * p + 7]);
            }
            // Copy out the PREVIOUS tile's candidates here: its slot was claimed two steps ago, and
            // every older load has just been consumed, so nothing this waits on is still in flight.
            if (r == 2 && pend_tile != 0xffffffffu) {
                emit_tile(out, s_olist + kOutCap * pend_buf, pend_tile, pend_base, pend_total, lane);
                pend_tile = 0xffffffffu;
            }
            if (r + 2 < kRows) load_row(in, ts_cur, r + 2, lane, n_vchunks, x);
            else if (g_next < n_tiles) load_row(in, ts, 0, lane, n_vchunks, x);
            if (r + 2 < kRows) load_row(in, ts_cur, r + 3, lane, n_vchunks, x + 4);
            else if (g_next < n_tiles) load_row(in, ts, 1, lane, n_vchunks, x + 4);
#pragma unroll
            for (int k = 0; k < scan2::kPairLook; k++) X[32 + k] = __shfl_down_sync(0xffffffffu, X[k], 1);
            uint32_t ma, mb;
            scan2::rows2_mask(X, one, minus_one, ma, mb);
            s_mask[32 * r + lane] = lane == 31 ? 0u : ma;            // lane 31's positions belong to the next row
            s_mask[32 * r + 32 + lane] = lane == 31 ? 0u : mb;
        }
        __syncwarp();
        // lane j now takes words kRows*j .. kRows*j + kRows-1 = 32*kRows consecutive positions of one row
        uint32_t w[kRows];
#pragma unroll
        for (int q4 = 0; q4 < kRows / 4; q4++) {
            const uint4 m4 = reinterpret_cast<const uint4 *>(s_mask)[(kRows / 4) * lane + q4];
            w[4 * q4 + 0] = m4.x; w[4 * q4 + 1] = m4.y; w[4 * q4 + 2] = m4.z; w[4 * q4 + 3] = m4.w;
        }
        const int base = kRowFresh * ((kRows * lane) >> 5) + 32 * ((kRows * lane) & 31);   // tile position of bit 0 of w[0]

        // ---- positions the reference never tests (dump1090.c:1593): j >= 131070, i.e. the first
        // two positions v = 131072k, 131072k+1 of every buffer (v = t+2); the batch ends at t = N-1
        const uint32_t v_tile = g * (uint32_t)kTile;
        {
            const uint32_t o = v_tile & (kBufSamples - 1);
            if (o < 2u || o + (uint32_t)kTile > kBufSamples) {
#pragma unroll
                for (int d = 0; d < 2; d++) {
                    const int p = (int)(((uint32_t)d - o) & (kBufSamples - 1));      // tile position of v = 131072k + d
#pragma unroll
                    for (int q = 0; q < kRows; q++)
                        if (p >= base + 32 * q && p < base + 32 * q + 32) w[q] &= ~(1u << (p - base - 32 * q));
                }
            }
            if (t_end + 2 - v_tile < (uint64_t)kTile) {
                const int s_max = (int)(t_end + 2 - v_tile);
#pragma unroll
                for (int q = 0; q < kRows; q++) {
                    const int lo_pos = base + 32 * q;
                    if (lo_pos >= s_max) w[q] = 0;
                    else if (lo_pos + 32 > s_max) w[q] &= (1u << (s_max - lo_pos)) - 1u;
                }
            }
        }

        // ---- survivors of the ten comparisons (~1 % of positions) get the exact "high" tests,
        // 32 at a time in position order.  Listing them is balanced over the warp in two steps: the
        // owner lanes queue their non-empty flag words (most hold one survivor) with the slot of
        // their first survivor, then the words are spread one per lane and expanded.
        uint32_t nz = 0, cnt = 0;
#pragma unroll
        for (int q = 0; q < kRows; q++) { nz += w[q] != 0u; cnt += __popc(w[q]); }
        uint32_t incl = nz | (cnt << 16);                            // two prefix sums in one
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t o = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += o;
        }
        const uint32_t totals = __shfl_sync(0xffffffffu, incl, 31);
        const uint32_t n_surv = totals >> 16, n_words = totals & 0xffffu;
        uint16_t *olist = s_olist + kOutCap * cur;
        uint32_t n_out = 0;
        bool dense = n_surv > (uint32_t)kSurvivorCap || n_words > (uint32_t)kEntryCap;
        if (!dense) {
            uint32_t slot = (incl & 0xffffu) - nz, sslot = (incl >> 16) - cnt;
#pragma unroll
            for (int q = 0; q < kRows; q++)
                if (w[q]) {
                    s_entry[slot] = make_uint2(w[q], (uint32_t)(base + 32 * q) | (sslot << 16));
                    slot++; sslot += __popc(w[q]);
                }
            __syncwarp();
            for (uint32_t e0 = 0; e0 < n_words; e0 += 32) {
                if (e0 + lane < n_words) {
                    const uint2 e = s_entry[e0 + lane];
                    const uint32_t p0 = e.y & 0xffffu;
                    uint32_t sl = e.y >> 16;
                    for (uint32_t b = e.x; b; b &= b - 1) s_surv[sl++] = (uint16_t)(p0 + __ffs(b) - 1);
                }
            }
            __syncwarp();
            // Three rounds of 32 survivors at a time: the loads of all three are issued before the
            // first is used (30 sample loads, then 15 table lookups in flight per lane), so a tile
            // pays the two memory round trips of a round once, not once per round.
            for (uint32_t i0 = 0; i0 < n_surv; i0 += 32 * kExactRounds) {
                int spos[kExactRounds];
                bool pass[kExactRounds];
#pragma unroll
                for (int k = 0; k < kExactRounds; k++) {
                    const uint32_t i = i0 + 32 * k + lane;
                    spos[k] = i < n_surv ? s_surv[i] : 0;
                }
                if (ts_cur.interior) {
                    const uint16_t *tp = reinterpret_cast<const uint16_t *>(ts_cur.flat);
                    uint32_t raw[kExactRounds][10];
#pragma unroll
                    for (int k = 0; k < kExactRounds; k++) {
                        const uint16_t *p = tp + spos[k];
                        raw[k][0] = __ldg(p); raw[k][1] = __ldg(p + 2); raw[k][2] = __ldg(p + 7); raw[k][3] = __ldg(p + 9);
                        raw[k][4] = __ldg(p + 4); raw[k][5] = __ldg(p + 5); raw[k][6] = __ldg(p + 11);
                        raw[k][7] = __ldg(p + 12); raw[k][8] = __ldg(p + 13); raw[k][9] = __ldg(p + 14);
                    }
                    // Most survivors are noise and fail by a wide margin; those are decided on the squared
                    // magnitudes alone and skip the table (their lanes make no memory requests):
                    //   m = round(360 sqrt(n))  =>  6(mx+1) >= 2160 sqrt(nx) + 3  and
                    //   m0+m2+m7+m9 <= 360 (sqrt n0 + sqrt n2 + sqrt n7 + sqrt n9) + 2 <= 720 sqrt(n0+n2+n7+n9) + 2,
                    // so 9 nx >= n0+n2+n7+n9 implies 6(mx+1) > m0+m2+m7+m9: the test of dump1090.c:1624-1642 fails.
                    uint32_t m[kExactRounds][5];
                    bool undecided[kExactRounds];
#pragma unroll
                    for (int k = 0; k < kExactRounds; k++) {
                        uint32_t n[10];
#pragma unroll
                        for (int j = 0; j < 10; j++) n[j] = n_of(raw[k][j]);
                        const uint32_t nx = max(max(max(n[4], n[5]), max(n[6], n[7])), max(n[8], n[9]));
                        undecided[k] = 9u * nx < n[0] + n[1] + n[2] + n[3];
#pragma unroll
                        for (int j = 0; j < 5; j++) m[k][j] = 0u;
                        if (undecided[k]) {
#pragma unroll
                            for (int j = 0; j < 4; j++) m[k][j] = __ldg(lutn + n[j]);
                            m[k][4] = __ldg(lutn + nx);
                        }
                    }
#pragma unroll
                    for (int k = 0; k < kExactRounds; k++)                // dump1090.c:1624-1642, see high_rule
                        pass[k] = undecided[k] && 6 * ((int)m[k][4] + 1) <= (int)(m[k][0] + m[k][1] + m[k][2] + m[k][3]);
                } else {
#pragma unroll
                    for (int k = 0; k < kExactRounds; k++)
                        pass[k] = high_tests_edge(in.body, in.halo, in.n_samples, ts_cur.c0 * 8 + (uint64_t)spos[k], lutn);
                }
#pragma unroll
                for (int k = 0; k < kExactRounds; k++) {
                    const bool ok = pass[k] && i0 + 32 * k + lane < n_surv;
                    const uint32_t bal = __ballot_sync(0xffffffffu, ok);
                    const uint32_t oslot = n_out + __popc(bal & lt_mask);
                    if (ok && oslot < (uint32_t)kOutCap) olist[oslot] = (uint16_t)spos[k];
                    n_out += __popc(bal);
                }
            }
            dense = n_out > (uint32_t)kOutCap;
        }
        if (!dense) {
            pend_total = n_out; pend_tile = g; pend_buf = cur;       // its slot is claimed at the top of the next tile
        } else {
            __syncwarp();
#pragma unroll
            for (int q = 0; q < kRows; q++) s_mask[kRows * lane + q] = w[q];       // as masked above
            __syncwarp();
            dense_tile(in.body, in.halo, in.n_samples, n_vchunks, lutn, out.cand_v, out.cand_capacity, out.tiles, out.counters,
                       g, s_mask, s_surv, lane);
        }
        __syncwarp();                                    // the masks, the queue and the lists are reused by the next tile
        g = g_next;
    }
    if (pend_tile != 0xffffffffu) {
        if (lane == 0 && pend_total) pend_base = atomicAdd(&out.counters[0], pend_total);
        emit_tile(out, s_olist + kOutCap * pend_buf, pend_tile, pend_base, pend_total, lane);
    }
    // The last CTA to finish hands the final count and overflow flag to the host (lane 0 made every
    // write to counters[1]; counters[0] only ever changes by atomics).  No CTA waits for another.
    if (out.host_counts && lane == 0) {
        __threadfence();
        if (atomicAdd(&out.counters[4], 1u) == gridDim.x - 1) {
            const volatile uint32_t *c = out.counters;
            out.host_counts[0] = c[0];
            out.host_counts[1] = c[1];
            __threadfence_system();
        }
    }
}

}  // namespace

void launch_scan(const BatchView &in, const DeviceTables &tab, const ScanOutputs &out, int sm_count, cudaStream_t stream,
                 const uint8_t *carry_block) {
    // occupancy is a property of the device the context lives on
    static int ctas_per_sm[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) dev = 0;
    if (!ctas_per_sm[dev]) {
        int n = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, scan_kernel, 32, 0) != cudaSuccess || n < 1) n = 12;
        ctas_per_sm[dev] = n;
    }
    const uint32_t n_tiles = tiles_for(in.n_samples);
    uint32_t grid = (uint32_t)(sm_count * ctas_per_sm[dev]);   // persistent single-warp CTAs, all resident
    if (grid > n_tiles) grid = n_tiles;                         // (so that every CTA has a tile and reaches the end)
    CarryBlock carry = {};
    if (carry_block) memcpy(carry.b, carry_block, kHaloAlloc);
    scan_kernel<<<grid, 32, 0, stream>>>(in, carry, carry_block ? 1u : 0u, tab.lutn, out, n_tiles, 1u, 0xffffffffu, 65536u);
}

}  // namespace modes
