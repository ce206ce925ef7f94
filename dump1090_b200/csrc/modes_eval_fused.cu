// modes_eval_fused.cu — K2, frame evaluation as ONE walk per candidate (sm_90a).
//
// Replaces the body of detectModeS after the preamble test (dump1090.c:1653-1735) and the
// order-independent half of decodeModesMessage (:1099-1128), like eval_serial_kernel
// (modes_kernels.cu), with the per-candidate arithmetic of modes_eval_serial.cuh, namespace fused:
// the first attempt and the phase-corrected retry share one pass over the window, in the retry's
// walk direction, and nothing is written back.
//
// Thread = candidate, warp = 32 consecutive candidates.  What the kernel adds around the walk:
//  * The walk direction and scale factors depend on eight preamble samples only
//    (applyPhaseCorrection, :1498-1517).  Each lane's first seven window words are copied to a small
//    "preamble area" before the chunk's windows are staged (cp.async, behind the walk of the chunk
//    before it), so that when a chunk is staged every lane already knows which way it will walk.
//  * The windows are staged in WALK ORDER: the words of a backwards-walked candidate are written
//    reversed (the copy is a 4-byte cp.async per word anyway: windows are only 4-byte aligned).
//    Every lane then reads ascending slots at compile-time offsets; row stride odd: lane l's slot
//    k sits in bank (stride*l + k) mod 32, conflict free whatever the directions are.
//  * The next chunk's windows are copied while the current chunk's verdicts (mask assembly, CRC,
//    repair) are worked out: the rows are free as soon as every lane has finished its walk, and
//    the verdicts leave straight from registers.  Chunks of 32 candidates are handed out from a
//    global counter three ahead: chunk i+2's positions are loaded, its preamble words copied and
//    its windows prefetched into L2 while chunk i is walked.
//  * MODES_EVAL_VARIANT=fused2 stages half a window at a time into the same rows (57 slots, then
//    the other 57, slot 56 twice): 8.4 KB per warp instead of 15.6, 16 warps per SM instead of 12.
//    The second half's copy is exposed (it cannot start before all lanes finished the first half);
//    measured slightly slower than whole windows (0.170 against 0.166 ms).
#include <cstdint>
#include <cstdlib>
#include <cuda_runtime.h>
#include "modes_internal.h"
#include "modes_eval_serial.cuh"

namespace modes {
namespace {

constexpr int kPreStride = 9;                            // words per lane in the preamble area (7 used; odd: conflict free)
constexpr int kPreWords = 7;
constexpr int kNibWords = 28 * 16;
constexpr int kLutWords = serial::kIqLutEntries / 2;
constexpr int kTableWords = 112 + kFixHashSlots + kNibWords + kLutWords;
static_assert(serial::kIqLutStride == kLutIqStride && serial::kIqLutEntries % 8 == 0, "table geometry");
static_assert(kTableWords % 2 == 0, "record staging uses 8-byte stores");

// kFirst = blocks of the walk (of 4) whose slots are staged first; the rest follows into the same
// rows once every lane is through them.  4: the whole walk (113 slots) at once, 12 warps per SM;
// 3: 85 slots, then 29 (16 warps); 2: two halves of 57 (slot 56 twice: a part starts with the word
// its first pair begins in).
template <int kFirst, int kWarpsPerSm> struct Geom {
    static constexpr int kParts = kFirst == serial::fused::kBlocks ? 1 : 2;
    static constexpr int kSlots0 = serial::fused::kBlockBits * kFirst + 1;                              // slots of part 0
    static constexpr int kSlots1 = serial::fused::kBlockBits * (serial::fused::kBlocks - kFirst) + 1;   // slots of part 1 (from slot 28 * kFirst)
    static constexpr int kRow = kSlots0 > kSlots1 ? kSlots0 : kSlots1;                                  // 113, 85 or 57 words: odd
    static constexpr int kWarps = kWarpsPerSm;
    static constexpr int kThreads = 32 * kWarps;
    static constexpr int kWarpWords = 32 * kRow + 32 * kPreStride;
    static constexpr int kSmemBytes = 4 * (kTableWords + kWarps * kWarpWords);
    static_assert(kFirst >= 2 && kFirst <= serial::fused::kBlocks, "split");
    static_assert(kRow % 2 == 1 && (32 * kRow) % 2 == 0 && kWarpWords % 2 == 0, "row geometry");
    static_assert(kSmemBytes <= 227 * 1024, "shared memory");
};

__device__ __forceinline__ uint32_t raw_sample(const BatchView &in, uint64_t v) {
    const uint8_t *p = (v < (uint64_t)kHaloSamples) ? in.halo + 2 * v : in.body + 2 * (v - kHaloSamples);
    return *reinterpret_cast<const uint16_t *>(p);
}

__device__ __forceinline__ void cp_async4(uint32_t dst_shared, const uint32_t *src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst_shared), "l"(src) : "memory");
}

// One lane's atomic add.  For an atomic on a warp-uniform address in divergent code ptxas emits its
// aggregated form (leader election, population count, and a shuffle of the result right behind
// the atomic), and that shuffle waits for the atomic's round trip at the top of every chunk (3.7 %
// of the kernel).  The hand-out counter is therefore addressed as counters + 3 + lane * c_zero with
// c_zero = 0 from a kernel parameter: not provably uniform, so the atomic stays a plain one and its
// result is first touched a chunk later.
__device__ __forceinline__ uint32_t atom_add(uint32_t *p, uint32_t x) {
    uint32_t old;
    asm volatile("atom.global.add.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(x) : "memory");
    return old;
}

// Word w (0..120) of the window of the candidate at virtual position v, whatever it overlaps.
__device__ __noinline__ uint32_t window_word_slow(const uint8_t *body, const uint8_t *halo, uint64_t n_samples, uint32_t v, int w) {
    const BatchView in{body, halo, n_samples};
    if (v > (uint32_t)kHaloSamples)
        return __ldg(reinterpret_cast<const uint32_t *>(in.body) + ((v - 1 - kHaloSamples) >> 1) + w);
    // window reaches into the carry block (first 240 positions of a batch): sample by sample, odd = 0
    return raw_sample(in, (uint64_t)v - 1 + 2 * w) | (raw_sample(in, (uint64_t)v + 2 * w) << 16);
}

// The first seven window words of this lane's candidate -> its row of the preamble area.
__device__ __forceinline__ void prestage(const BatchView &in, const uint32_t *body32, uint32_t v, uint32_t *pre, uint32_t pre_s) {
    if (v > (uint32_t)kHaloSamples) {
        const uint32_t *wp = body32 + ((v - 1 - kHaloSamples) >> 1);
#pragma unroll
        for (int k = 0; k < kPreWords; k++) cp_async4(pre_s + 4u * k, wp + k);
    } else {
        for (int k = 0; k < kPreWords; k++) pre[k] = window_word_slow(in.body, in.halo, in.n_samples, v, k);
    }
}

// Slots [u0, u0 + kCount) of all 32 rows of a chunk -> shared memory (row c at rows + c * kRow,
// slot u at word u - u0).  Forwards slot u = window word 8 + u, backwards = window word 120 - u.
// `w0` = this lane's candidate's first window word as an index into the body's 32-bit words.
// Branch-free: a backwards row is copied by the mirrored lane assignment (lane l takes slots
// kCount-1-l, kCount-1-l-32, ...), so that in both directions a lane's source words are 32 apart
// ascending (compile-time offsets) and only the shared-memory side differs (a select per copy).
template <int kRow, int kCount>
__device__ __forceinline__ void stage_part(const BatchView &in, const uint32_t *body32, uint32_t my_v, uint32_t w0, uint32_t rev_mask,
                                           bool fast, uint32_t *rows, uint32_t rows_s, int u0, int lane) {
    if (fast) {
        // common case (no window in the carry block): asynchronous copies straight into shared
        // memory, all 32 rows in flight, one wait (the caller's)
        constexpr int kCopies = (kCount + 31) / 32;
        const uint32_t a_fwd = (uint32_t)(8 + u0 + lane), a_rev = (uint32_t)(121 - u0 - kCount + lane);
        uint32_t d_fwd[kCopies], d_rev[kCopies];
#pragma unroll
        for (int j = 0; j < kCopies; j++) {
            d_fwd[j] = rows_s + 4u * (uint32_t)(lane + 32 * j);
            d_rev[j] = rows_s + 4u * (uint32_t)(kCount - 1 - lane - 32 * j);
        }
        // rows in groups of eight: inside a group the row's offset is a compile-time immediate, between
        // groups the eight shared-memory bases move on
        uint32_t rm = rev_mask;
#pragma unroll 1
        for (int g = 0; g < 32; g += 8) {
#pragma unroll
            for (int ci = 0; ci < 8; ci++) {
                const uint32_t w = __shfl_sync(0xffffffffu, w0, g + ci);
                const bool rev = (rm >> ci) & 1u;
                const uint32_t *src = body32 + (w + (rev ? a_rev : a_fwd));
#pragma unroll
                for (int j = 0; j < kCopies; j++)
                    if (32 * j + 31 < kCount || lane + 32 * j < kCount)
                        cp_async4((rev ? d_rev[j] : d_fwd[j]) + 4u * (uint32_t)(ci * kRow), src + 32 * j);
            }
            rm >>= 8;
#pragma unroll
            for (int j = 0; j < kCopies; j++) { d_fwd[j] += 4u * 8u * (uint32_t)kRow; d_rev[j] += 4u * 8u * (uint32_t)kRow; }
        }
    } else {
        for (int c = 0; c < 32; c++) {
            const uint32_t v = __shfl_sync(0xffffffffu, my_v, c);
            const bool rev = (rev_mask >> c) & 1u;
            for (int k = lane; k < kCount; k += 32) {
                const int u = u0 + k;
                rows[c * kRow + k] = window_word_slow(in.body, in.halo, in.n_samples, v, rev ? 120 - u : 8 + u);
            }
        }
    }
}

template <int kFirst, int kWarpsPerSm>
__global__ void __launch_bounds__(Geom<kFirst, kWarpsPerSm>::kThreads, 1)
eval_fused_kernel(BatchView in, DeviceTables tab, const uint32_t *__restrict__ cand_v, uint32_t *counters,
                  uint32_t cand_capacity, modes_candidate *records, int fix_errors, int aggressive, uint32_t c_one,
                  uint32_t c_m1, uint32_t c_m16k, uint32_t c_zero) {
    using G = Geom<kFirst, kWarpsPerSm>;
    namespace fz = serial::fused;
    extern __shared__ __align__(16) uint32_t s_mem[];
    uint32_t *s_syn = s_mem, *s_hash = s_syn + 112, *s_nib = s_hash + kFixHashSlots;
    uint16_t *s_lut = reinterpret_cast<uint16_t *>(s_nib + kNibWords);
    uint32_t *s_warp = s_nib + kNibWords + kLutWords;
    for (int i = threadIdx.x; i < 112; i += G::kThreads) s_syn[i] = tab.bit_syn[i];
    for (int i = threadIdx.x; i < kFixHashSlots; i += G::kThreads) s_hash[i] = tab.fix_hash[i];
    for (int i = threadIdx.x; i < serial::kIqLutEntries / 8; i += G::kThreads)
        reinterpret_cast<uint4 *>(s_lut)[i] = __ldg(reinterpret_cast<const uint4 *>(tab.lut_iq) + i);
    __syncthreads();
    for (int i = threadIdx.x; i < kNibWords; i += G::kThreads) s_nib[i] = serial::nibble_syndrome(s_syn, i >> 4, i & 15);
    __syncthreads();

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t *rows = s_warp + warp * G::kWarpWords;
    uint32_t *pre = rows + 32 * G::kRow + kPreStride * lane;
    const uint32_t rows_s = (uint32_t)__cvta_generic_to_shared(rows);
    const uint32_t pre_s = (uint32_t)__cvta_generic_to_shared(pre);
    const serial::Tables T{s_lut, s_syn, s_nib, s_hash, tab.pair_hash};
    const fz::Lut lut{(uint32_t)__cvta_generic_to_shared(s_lut)};
    uint32_t n_cand = counters[0];
    if (n_cand > cand_capacity) n_cand = cand_capacity;
    const uint32_t n_chunks = (n_cand + 31) / 32;
    const uint32_t total_warps = gridDim.x * G::kWarps;
    const uint32_t *body32 = reinterpret_cast<const uint32_t *>(in.body);

    // Chunks of 32 candidates are handed out from a global counter, requested three chunks ahead:
    // while chunk i is evaluated, chunk i+1's first part is staged (behind the verdicts of chunk i),
    // chunk i+2's positions are loaded, its preamble words copied and its windows prefetched into L2.
    // (The counter values are used untouched until a chunk later: arithmetic on them right away
    // would wait for the atomic's round trip.)
    auto positions = [&](uint32_t c) -> uint32_t {
        if (c >= n_chunks) return 0u;
        const uint32_t nc = n_cand - c * 32 < 32u ? n_cand - c * 32 : 32u;   // idle lanes of the last chunk duplicate its last candidate
        return cand_v[c * 32 + ((uint32_t)lane < nc ? lane : nc - 1)];
    };
    auto look_ahead = [&](uint32_t c, uint32_t v) {      // chunk c (positions v): preamble words -> preamble area, windows -> L2
        if (c >= n_chunks) return;
        prestage(in, body32, v, pre, pre_s);
        if (v > (uint32_t)kHaloSamples) {
            // 484 bytes from a 4-byte aligned address: five 128-byte lines
            const uint8_t *wp = in.body + 4ull * ((v - 1 - kHaloSamples) >> 1);
            if ((uint64_t)(wp - in.body) + 640u <= 2ull * in.n_samples) {
#pragma unroll
                for (int k = 0; k < 5; k++) asm volatile("prefetch.global.L2 [%0];" ::"l"(wp + 128 * k));
            }
        }
    };
    // this lane's walk of the chunk whose preamble words are in the preamble area, and the chunk's first part on its way
    auto setup_and_stage = [&](uint32_t v, fz::Lane &L, uint32_t &rev_mask, bool &fast) {
        const uint32_t odd = v > (uint32_t)kHaloSamples ? ((v - 1 - kHaloSamples) & 1u) : 0u;
        fz::phase_setup(pre, odd, s_lut, c_one, c_m1, c_m16k, L);
        rev_mask = __ballot_sync(0xffffffffu, L.fwd == 0u);
        fast = __all_sync(0xffffffffu, v > (uint32_t)kHaloSamples);
        stage_part<G::kRow, G::kSlots0>(in, body32, v, (v - 1 - kHaloSamples) >> 1, rev_mask, fast, rows, rows_s, 0, lane);
    };

    uint32_t chunk = blockIdx.x * G::kWarps + warp;
    if (chunk >= n_chunks) return;
    uint32_t next1 = 0, next2_raw = 0;
    uint32_t *const hand_out = counters + 3 + lane * c_zero;
    if (lane == 0) { next1 = atom_add(hand_out, 1u); next2_raw = atom_add(hand_out, 1u); }
    next1 = total_warps + __shfl_sync(0xffffffffu, next1, 0);
    uint32_t my_v = positions(chunk), v1 = positions(next1);
    fz::Lane L;
    uint32_t rev_mask;
    bool fast;
    prestage(in, body32, my_v, pre, pre_s);
    asm volatile("cp.async.wait_all;" ::: "memory");
    setup_and_stage(my_v, L, rev_mask, fast);
    look_ahead(next1, v1);                                 // (the preamble area is free again: phase_setup has read it)
    asm volatile("cp.async.wait_all;" ::: "memory");
    __syncwarp();

    while (true) {
        // rows: part 0 of `chunk` (complete); L, rev_mask, fast: its walk; preamble area: chunk next1's words (arriving)
        const uint32_t next2 = total_warps + __shfl_sync(0xffffffffu, next2_raw, 0);
        if (lane == 0) next2_raw = atom_add(hand_out, 1u);
        const uint32_t v2 = positions(next2);              // used after the walk
        const uint32_t base = chunk * 32;
        const uint32_t n = n_cand - base < 32u ? n_cand - base : 32u;
        const uint32_t *row = rows + lane * G::kRow;
        fz::Walk W;
        fz::walk_begin(W, L, row[0]);
        constexpr int kU1 = fz::kBlockBits * kFirst;       // part 1 holds slots kU1 ..: the walk indexes slots from 0
#pragma unroll 1
        for (int h = 0; h < G::kParts; h++) {              // (a loop, so that the walk's code exists once)
            if (h) {
                __syncwarp();                              // every lane is done with part 0
                stage_part<G::kRow, G::kSlots1>(in, body32, my_v, (my_v - 1 - kHaloSamples) >> 1, rev_mask, fast, rows, rows_s, kU1, lane);
                asm volatile("cp.async.wait_all;" ::: "memory");
                __syncwarp();
            }
            fz::walk_blocks(W, L, h ? row - kU1 : row, h ? kFirst : 0, h ? fz::kBlocks : kFirst, lut);
        }
        __syncwarp();                                      // the rows are free
        const uint64_t t = (uint64_t)my_v - 2;
        const fz::Lane Lcur = L;
        const bool more = next1 < n_chunks;
        if (more) {
            // the next chunk's first part is copied while this chunk's verdicts are worked out
            asm volatile("cp.async.wait_all;" ::: "memory");   // its preamble words (issued a walk ago)
            setup_and_stage(v1, L, rev_mask, fast);
            look_ahead(next2, v2);
        }
        uint32_t rec[14];
        rec[0] = (uint32_t)t; rec[1] = (uint32_t)(t >> 32);
        fz::walk_finish(W, Lcur, (((uint32_t)t) & (kBufSamples - 1)) == 0, fix_errors, aggressive, T, rec + 2);
        if ((uint32_t)lane < n) {
            // 56-byte records, 8-byte aligned: straight from registers (the rows are being overwritten)
            uint2 *dst = reinterpret_cast<uint2 *>(records + base + lane);
#pragma unroll
            for (int k = 0; k < 7; k++) dst[k] = make_uint2(rec[2 * k], rec[2 * k + 1]);
        }
        if (!more) break;
        asm volatile("cp.async.wait_all;" ::: "memory");
        __syncwarp();
        chunk = next1; next1 = next2;
        my_v = v1; v1 = v2;
    }
}

template <int kFirst, int kWarpsPerSm>
void launch_fused(const BatchView &in, const DeviceTables &tab, const ScanOutputs &scan, modes_candidate *records,
                  int fix_errors, int aggressive, int sm_count, cudaStream_t stream) {
    using G = Geom<kFirst, kWarpsPerSm>;
    // the opt-in to > 48 KB of dynamic shared memory is per device
    static bool configured[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64 || !configured[dev]) {
        cudaFuncSetAttribute(eval_fused_kernel<kFirst, kWarpsPerSm>, cudaFuncAttributeMaxDynamicSharedMemorySize, G::kSmemBytes);
        if (dev >= 0 && dev < 64) configured[dev] = true;
    }
    eval_fused_kernel<kFirst, kWarpsPerSm><<<sm_count, G::kThreads, G::kSmemBytes, stream>>>(in, tab, scan.cand_v, scan.counters, scan.cand_capacity,
                                                                               records, fix_errors, aggressive, 1u, 0xffffffffu, (uint32_t)-16384, 0u);
}

}  // namespace

void launch_eval_fused(const BatchView &in, const DeviceTables &tab, const ScanOutputs &scan, modes_candidate *records,
                       int fix_errors, int aggressive, int sm_count, int parts, cudaStream_t stream) {
    // measured on an H100 (400 W) over the bench's 845 458 candidates: whole windows, 12 warps per SM 0.293 ms;
    // half windows, 16 warps 0.321 ms
    if (parts == 2) launch_fused<2, 16>(in, tab, scan, records, fix_errors, aggressive, sm_count, stream);
    else launch_fused<4, 12>(in, tab, scan, records, fix_errors, aggressive, sm_count, stream);
}

}  // namespace modes
