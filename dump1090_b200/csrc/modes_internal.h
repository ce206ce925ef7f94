// modes_internal.h — declarations shared by the CUDA kernels (modes_kernels.cu),
// the host resolve (modes_resolve.cpp) and the C-ABI glue (modes_api.cpp).
// Product code; never includes anything from oracle/.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>
#include "modes_b200.h"

namespace modes {

// ---- geometry of the "virtual" sample array a batch is scanned over --------
// A batch is n_buffers whole reference buffers (131072 new samples each,
// dump1090.c:54) resident in HBM, preceded by the 238 samples the reference
// carries over from the previous buffer (dump1090.c:481).  The carry lives in
// a separate 480-byte device block (2 unused samples + 238 carry) so that the
// body keeps its 16-byte alignment:
//     virtual index v in [0, 240)      -> halo[v]
//     virtual index v in [240, 240+N)  -> body[v-240]
// The reference's buffer-relative position of v is t = v - 2 = 131072*k + j,
// and the scan visits j in [0, 131070) (dump1090.c:1593).
constexpr int      kHaloSamples  = 240;
constexpr int      kHaloBytes    = 480;
constexpr int      kHaloAlloc    = 512;                         // + 16 bytes of "no signal" (127) after the carry: kernels read it for out-of-range chunks
constexpr int      kTileSamples  = MODES_TILE_SAMPLES;          // one scan tile: 8 rows of 31 lanes x 32 positions (modes_scan2.cu)
constexpr uint32_t kBufSamples   = MODES_BUFFER_SAMPLES;
constexpr uint32_t kScanLimit    = kBufSamples - 2;             // j < 131070
constexpr int      kNLutEntries  = 32769;                       // magnitude by i*i+q*q
constexpr int      kFixHashSlots = 256;
constexpr int      kPairHashBits = 14;                          // == serial::kPairHashBits
constexpr int      kPairHashSlots = 1 << kPairHashBits;          // two-bit patterns: 5671 entries
constexpr int      kPairHashMaxProbe = 16;                      // checked at table construction
constexpr int      kLutIqStride  = 136;                         // == serial::kIqLutStride (modes_eval_serial.cuh)
constexpr int      kLutIqEntries = 129 * kLutIqStride;

struct DeviceTables {
    const uint16_t *lutn;        // [32769] round(sqrt(n)*360), dump1090.c:362 keyed by n=i*i+q*q
    const uint16_t *lut_iq;      // [129 x kLutIqStride] the same keyed by (|I-127|, |Q-127|); 16-byte aligned
    const uint32_t *bit_syn;     // [112] syndrome of a single flipped bit (dump1090.c:683-698 + parity bits)
    const uint32_t *fix_hash;    // [256] open-addressed inverse of bit_syn: (syndrome<<8 | pos), 0xFFFFFFFF empty
    const uint32_t *pair_hash;   // [16384] two flipped bits p < q: (syndrome<<7 | p), 0xFFFFFFFF empty
};

struct BatchView {
    const uint8_t *body;         // n_samples*2 bytes, 16-byte aligned
    const uint8_t *halo;         // kHaloBytes, 16-byte aligned
    uint64_t       n_samples;    // N = n_buffers * 131072
};

struct ScanOutputs {
    uint32_t   *cand_v;          // virtual positions of candidates, tile by tile
    uint32_t    cand_capacity;
    modes_tile *tiles;           // [n_tiles]
    uint32_t   *counters;        // [0] candidates found (may exceed capacity), [1] overflow flag, [2]/[3] scan tile / eval chunk hand-out
};

inline uint32_t tiles_for(uint64_t n_samples) {
    return (uint32_t)((n_samples + kHaloSamples + kTileSamples - 1) / kTileSamples);
}

// Kernel launchers (launch_scan: modes_scan2.cu; the rest: modes_kernels.cu).  All asynchronous on `stream`.
void launch_scan(const BatchView &in, const DeviceTables &tab, const ScanOutputs &out, int sm_count,
                 cudaStream_t stream);
void launch_eval(const BatchView &in, const DeviceTables &tab, const ScanOutputs &scan,
                 modes_candidate *records, int fix_errors, int aggressive, int sm_count,
                 cudaStream_t stream);
// The single-walk frame evaluation (modes_eval_fused.cu); parts = 1: whole windows staged, 2: half windows.
void launch_eval_fused(const BatchView &in, const DeviceTables &tab, const ScanOutputs &scan, modes_candidate *records,
                       int fix_errors, int aggressive, int sm_count, int parts, cudaStream_t stream);
void launch_magnitude(const uint8_t *d_iq, uint16_t *d_mag, uint64_t n_samples, const uint16_t *lutn,
                      cudaStream_t stream);
// CRC / fix on raw frame bytes (hex door): n frames of 14 bytes -> n modes_frame_eval.
void launch_eval_frames(const uint8_t *d_frames, modes_frame_eval *d_out, uint32_t n, const DeviceTables &tab,
                        int fix_errors, int aggressive, cudaStream_t stream);
// Signal level of every decoded attempt (modes_signal.cu): writes pass[k].signal of the first
// min(counters[0], cand_capacity) records over the same windows the scan and frame evaluation read.
void launch_signal(const BatchView &in, const DeviceTables &tab, const ScanOutputs &scan, modes_candidate *records,
                   int sm_count, cudaStream_t stream);
// Levels of n_buffers whole buffers at d_iq + k * stride_bytes (modes_levels.cu): writes out[k],
// k < n_buffers, with buffer = k and n_samples = kBufSamples.
void launch_levels(const uint8_t *d_iq, uint32_t n_buffers, uint64_t stride_bytes, const DeviceTables &tab,
                   modes_level *out, int sm_count, cudaStream_t stream);
static_assert(sizeof(modes_level) == 40 && offsetof(modes_level, sum_mag) == 16 && offsetof(modes_level, peak) == 32,
              "level record layout");
// Recovery records (modes_recover.cu): writes out[k] for k < min(counters[0], capacity) from the
// candidate records and the windows the scan and frame evaluation read.
void launch_recover(const BatchView &in, const DeviceTables &tab, const ScanOutputs &scan, const modes_candidate *records,
                    uint32_t capacity, modes_recovered *out, int sm_count, cudaStream_t stream);
// Weak preambles (modes_weak.cu, three kernels): the positions of the scanned buffers of the batch
// (buffers first_buffer + i * buffer_step, i < n_buffers) that meet the weak-preamble definition
// (include/modes_b200.h), in stream order: pos[k] for k < min(counters[1], capacity).  counters[1] is
// the exact count; when it exceeds scratch_cap the list is not complete and nothing is written to pos
// (the caller repeats the batch with a larger scratch list).  tiles: 3 * weak_tiles_for(n_buffers)
// words of per-tile bookkeeping; counters (two words) are cleared on the stream by the launcher.
constexpr uint32_t kWeakTileSamples = 4096;
inline uint32_t weak_tiles_for(uint64_t n_buffers) { return (uint32_t)(n_buffers * (kBufSamples / kWeakTileSamples)); }
struct WeakOutputs {
    uint32_t  first_buffer, buffer_step, n_buffers;
    uint32_t *pos;
    uint32_t  capacity;
    uint32_t *scratch;           // the positions tile by tile, in no particular order of the tiles
    uint32_t  scratch_cap;
    uint32_t *tiles;
    uint32_t *counters;          // [1] weak positions found (may exceed both capacities); [0] is not used
};
void launch_weak_scan(const BatchView &in, const DeviceTables &tab, const WeakOutputs &out, int sm_count, cudaStream_t stream);
// The recovery records of the weak positions pos[k], k < min(*count, capacity), and none when *count
// exceeds scratch_cap (the positions were not all written) (modes_recover.cu: the same per-position
// search as launch_recover's).
void launch_recover_weak(const BatchView &in, const DeviceTables &tab, const uint32_t *count, uint32_t capacity,
                         uint32_t scratch_cap, const uint32_t *pos, modes_recovered *out, int sm_count, cudaStream_t stream);
// modes_weak_device over the buffers first_buffer + i * buffer_step of the last batch only (the
// receiver pool: its data buffers, never its pad buffers); modes_weak_device is (0, 1).
int weak_device_strided(modes_ctx *ctx, void *d_pos, void *d_rec, size_t capacity, uint32_t first_buffer, uint32_t buffer_step);
static_assert(sizeof(modes_recovered) == 20 && offsetof(modes_recovered, status) == 14 && offsetof(modes_recovered, signal) == 16,
              "recovery record layout");
static_assert(offsetof(modes_message, recovered) == 14 && offsetof(modes_message, msgbits) == 16, "message layout");

// The record layouts are ABI: the signal field took the two bytes every evaluation kernel already wrote as zero.
static_assert(sizeof(modes_frame_eval) == 24 && offsetof(modes_frame_eval, signal) == 18 && offsetof(modes_frame_eval, crc) == 20,
              "frame evaluation record layout");
static_assert(sizeof(modes_candidate) == 56, "candidate record layout");

// Host-side table construction (modes_tables.cpp).
void build_lutn(uint16_t *out /*[32769]*/);
void build_lut_iq(uint16_t *out /*[kLutIqEntries]*/);
void build_bit_syndromes(uint32_t *out /*[112]*/);
bool build_fix_hash(const uint32_t *bit_syn, uint32_t *out /*[256]*/);
bool build_pair_hash(const uint32_t *bit_syn, uint32_t *out /*[kPairHashSlots]*/);

// ---- device resolve (modes_resolve_gpu.cu) ----------------------------------
// One delivered message as the device resolve hands it over: position, the evaluated frame, and
// what the sequential half decided.  bits = crcok | phase_corrected << 8 | extra_is_ap << 16;
// extra = DF11 interrogator id, or the address recovered from an address/parity field.
struct modes_delivery { int64_t t; modes_frame_eval eval; uint32_t extra; uint32_t bits; };
static_assert(sizeof(modes_delivery) == 40, "delivery record layout");
// Replay + hand-over rounds before the in-order fallback (which then does nothing) and the emit pass.
// Two suffice on real traffic; a chain through the address cache over n buffers needs about n.
constexpr int kGpuResolveRounds = 4;

struct GpuResolve {
    uint32_t *start, *end;       // [n_buffers][1024] address cache at the start / end of each buffer
    uint32_t *written, *readfirst;   // [n_buffers][32]  slots a buffer wrote / read before writing
    uint32_t *rerun, *n_deliv, *offsets;   // [n_buffers] (+1 for offsets)
    uint32_t *flags;             // [0] a buffer still needed another replay (0 after the fallback), [1] delivery capacity exceeded, [2] deliveries
    const uint32_t *cache_in;    // [1024] cache at the start of the batch
    uint32_t *cache_out;         // [1024] cache at its end
    uint64_t *stats_out;         // [8]
    modes_delivery *out;         // deliveries in stream order
    uint32_t capacity;           // entries of `out`
};
void launch_gpu_resolve(const GpuResolve &g, const modes_candidate *records, const modes_tile *tiles, uint32_t n_tiles,
                        uint32_t n_buffers, int check_crc, int sm_count, cudaStream_t stream);

// ---- sequential resolve (modes_resolve.cpp) --------------------------------
struct ResolveState {
    uint32_t icao[1024];         // dump1090.c:335: address per slot (TTL: never expires within a run)
    int64_t  stats[8];
    int64_t  cur_buffer;         // buffer whose skip state is live, -1 = none
    uint32_t next_j;             // first position not skipped in cur_buffer
    uint32_t next_j_recovered;   // first position of cur_buffer not inside a recovered message (recovery only)
    modes_recovery_stats rstats;
    modes_recovery_stats wstats; // recoveries at weak preambles (modes_set_weak_preambles)
    void reset();
};

// recover_signal: recovered messages carry their record's signal (else 0)
struct ResolveConfig { int fix_errors, aggressive, check_crc; int recover_signal; };

// Where delivered messages go: a callback, and/or a caller-owned array that is
// filled in place (count keeps running past capacity).
struct MessageOut {
    modes_sink_fn sink = nullptr; void *user = nullptr;
    modes_message *array = nullptr; size_t capacity = 0; size_t count = 0;
};

// Working memory of the resolve (verdict lists, per-shard runs), owned by a context / resolver and
// kept between calls: grown once, never handed back (re-faulting ~14 MB of verdicts per GiB in every
// call costs more than the verdicts themselves).
struct ResolveScratch;
ResolveScratch *scratch_create();
void scratch_destroy(ResolveScratch *s);

// The weak positions of a record array (sorted t, as the candidates' t) and their recovery records.
struct WeakList { const uint32_t *t = nullptr; const modes_recovered *rec = nullptr; size_t n = 0; };

// recovered: one record per candidate (modes_recover.cu), or nullptr with recovery off; weak: the
// weak positions merged into the walk (only with recovered)
void resolve_candidates(ResolveState &st, const ResolveConfig &cfg, const modes_candidate *cands,
                        const modes_tile *tiles, size_t n_tiles, int64_t buffer_base, MessageOut &out,
                        ResolveScratch *scratch, const modes_recovered *recovered = nullptr, const WeakList &weak = WeakList());
void resolve_shards(ResolveState &st, const ResolveConfig &cfg, size_t n_shards, const modes_candidate *const *cands,
                    const modes_tile *const *tiles, const size_t *n_tiles, const int64_t *buffer_base,
                    MessageOut &out, ResolveScratch *scratch, const modes_recovered *const *recovered = nullptr,
                    const WeakList *weak = nullptr);
// A shard resolved from a GUESSED address cache (one rank / one GPU thread of a sharded decode):
// verdicts only, deliveries held back in the scratch until the guess is verified.
void resolve_tentative(ResolveState &st, const ResolveConfig &cfg, const modes_candidate *cands, const modes_tile *tiles,
                       size_t n_tiles, int64_t buffer_base, ResolveScratch *scratch);
void resolve_commit(MessageOut &out, ResolveScratch *scratch);
// Messages from the device resolve's delivery records (structs built in parallel, sink called in order).
void deliver_gpu(const modes_delivery *d, size_t n, int64_t buffer_base, MessageOut &out);
// The order-dependent tail of decodeModesMessage + field decode for one evaluated frame.
int finish_message(ResolveState &st, const modes_frame_eval &p, modes_message *out);
void add_recovery_stats(modes_recovery_stats &to, const modes_recovery_stats &from);

}  // namespace modes
