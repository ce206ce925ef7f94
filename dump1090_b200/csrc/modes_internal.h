// modes_internal.h — declarations shared by the CUDA kernels (modes_kernels.cu),
// the host resolve (modes_resolve.cpp) and the C-ABI glue (modes_api.cpp).
// Product code; never includes anything from oracle/.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>
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

// One batch's counters: [0] candidates found (may exceed capacity), [1] overflow flag, [2]/[3] scan tile /
// eval chunk hand-out, [4] scan CTAs finished (only with host_counts).  The scan starts from a zeroed set.
constexpr int kCounterWords = 8;

struct ScanOutputs {
    uint32_t   *cand_v;          // virtual positions of candidates, tile by tile
    uint32_t    cand_capacity;
    modes_tile *tiles;           // [n_tiles]
    uint32_t   *counters;        // kCounterWords (the first four without host_counts)
    // A context's slot alternates between two counter sets, so that no memset or copy sits between its
    // batches: the scan zeroes next_counters (the set of the slot's next batch) and its last CTA writes
    // counters[0..1] to host_counts (mapped pinned host memory).  nullptr: neither.
    uint32_t   *next_counters = nullptr;
    uint32_t   *host_counts = nullptr;
};

inline uint32_t tiles_for(uint64_t n_samples) {
    return (uint32_t)((n_samples + kHaloSamples + kTileSamples - 1) / kTileSamples);
}

// Kernel launchers (launch_scan: modes_scan2.cu; the rest: modes_kernels.cu).  All asynchronous on `stream`.
// carry_block: nullptr, the batch's carry block is in.halo (device); else kHaloAlloc host bytes that travel
// as a kernel parameter, and the scan stores them to in.halo for the batch's later kernels.
void launch_scan(const BatchView &in, const DeviceTables &tab, const ScanOutputs &out, int sm_count,
                 cudaStream_t stream, const uint8_t *carry_block = nullptr);
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
// Signal level, arrival code and carrier record of every decoded attempt (modes_signal.cu): writes
// pass[k].signal (signal), bits 4-7 of pass[k].flags (arrival) and carrier[i] (carrier != nullptr: the
// record of every candidate i with a decoded attempt) of the first min(counters[0], cand_capacity)
// records over the same windows the scan and frame evaluation read.  Launches nothing when all are off.
void launch_signal(const BatchView &in, const DeviceTables &tab, const ScanOutputs &scan, modes_candidate *records,
                   int sm_count, cudaStream_t stream, bool signal = true, bool arrival = false,
                   modes_carrier *carrier = nullptr);
static_assert(sizeof(modes_carrier) == 16, "carrier record layout");
// Levels of n_buffers whole buffers at d_iq + k * stride_bytes (modes_levels.cu): writes out[k],
// k < n_buffers, with buffer = k and n_samples = kBufSamples.
void launch_levels(const uint8_t *d_iq, uint32_t n_buffers, uint64_t stride_bytes, const DeviceTables &tab,
                   modes_level *out, int sm_count, cudaStream_t stream);
static_assert(sizeof(modes_level) == 40 && offsetof(modes_level, sum_mag) == 16 && offsetof(modes_level, peak) == 32,
              "level record layout");
// 2.4 MS/s UC8 input resampled to 2 MHz bytes (modes_resample.cu, arithmetic in modes_resample_core.cuh).
// Output sample n (stream index, 2 MHz) reads the input samples around 1.2 n; the job holds the stream's
// input bytes [2 in_first, 2 in_first + in_bytes) and every other input byte reads as 127.
struct ResampleJob {
    const uint8_t *in;           // 16-byte aligned
    uint64_t       in_bytes;
    int64_t        in_first;     // stream input sample of in[0]
    int64_t        out_first;    // stream output sample of body[0]: a multiple of 8
    uint64_t       out_samples;
    int64_t        out_end;      // output samples at or past it are written as 127 (the EOF buffer's padding)
    uint8_t       *body;         // 2 * out_samples bytes, 16-byte aligned
    uint8_t       *halo;         // kHaloAlloc bytes laid out as a batch's carry block (the 238 samples before
                                 // body[0] at kHaloBytes - MODES_CARRY_BYTES, 127 elsewhere), or nullptr
};
void launch_resample(const ResampleJob &j, cudaStream_t stream);
// 16-bit input (modes_set_input_format, arithmetic in modes_input_core.cuh): the same job over int16 I/Q,
// in[0] the first byte of input sample in_first (4 bytes a sample, a trailing partial sample not in the
// span), converted with the shift and then resampled (K9, 2.4 MS/s) or converted only (K10, 2 MHz:
// output sample n is input sample n; in_first a multiple of 4, so that its 16-byte loads are aligned).
void launch_resample_sc16(const ResampleJob &j, int shift, cudaStream_t stream);
void launch_convert_sc16(const ResampleJob &j, int shift, cudaStream_t stream);
// 4, 6, 8 and 10 MS/s (K11): the same job decimated by m = 2..5, the input UC8 (shift < 0) or int16
// converted with the shift; any in_first, out_first a multiple of 8.  step != 0 (K12): each input sample
// is first rotated by shift::step's phase at its stream index (modes_set_input_offset); step 0 is K11.
void launch_decimate(const ResampleJob &j, int m, int shift, uint32_t step, cudaStream_t stream);
// The receiver pool's 2.4 MS/s receivers (modes_pool.cpp): one launch for one job per pair of the pool's
// batch.  A job's input is its receiver's stream bytes [hist0, call0) at hist (the receiver's device input
// history) and [call0, call0 + MODES_BUFFER_BYTES) at stage (the call's bytes); every other input byte
// reads as 127.  hist0 and call0 are multiples of 16, hist and stage 16-byte aligned.
struct PoolResampleJob {
    const uint8_t *hist;
    const uint8_t *stage;
    int64_t        hist0, call0;
    int64_t        out_first;    // the 2 MHz buffer's first sample (a multiple of MODES_BUFFER_SAMPLES);
                                 // negative: a 2 MHz receiver, stage is copied to data as it is
    uint8_t       *pad_tail;     // MODES_CARRY_BYTES: samples out_first - 238 ... out_first - 1
    uint8_t       *data;         // MODES_BUFFER_BYTES, 16-byte aligned: samples out_first ...
};
// The history step of the same receivers: their stream bytes [keep, call0 + MODES_BUFFER_BYTES), read as
// a PoolResampleJob reads them, to out (the other half of the history; keep a multiple of 16).
struct PoolHistoryJob {
    const uint8_t *hist;
    const uint8_t *stage;
    int64_t        hist0, call0, keep;
    uint8_t       *out;
};
// d_jobs: device memory; max_bytes: the most bytes one history job writes.
void launch_resample_pool(const PoolResampleJob *d_jobs, uint32_t n_jobs, cudaStream_t stream);
void launch_history_pool(const PoolHistoryJob *d_jobs, uint32_t n_jobs, uint64_t max_bytes, cudaStream_t stream);
// The receiver pool's 16-bit receivers (modes_pool_set_input_format): one launch for one job per such
// receiver of the batch, ahead of the two above.  A job converts one whole buffer, MODES_BUFFER_SAMPLES
// int16 I/Q samples at in (2 x MODES_BUFFER_BYTES bytes), to its MODES_BUFFER_BYTES UC8 bytes at out
// (modes_input_core.cuh at the shift); in and out 16-byte aligned.
struct PoolConvertJob {
    const uint8_t *in;
    uint8_t       *out;
    int32_t        shift;
};
void launch_convert_pool(const PoolConvertJob *d_jobs, uint32_t n_jobs, cudaStream_t stream);
// The receiver pool's device-fed 2 MHz receivers (modes_pool_submit_device): one launch for one job per such
// pair of the batch, after the conversion.  A job copies the MODES_BUFFER_BYTES UC8 bytes at in (the caller's
// buffer; nullptr: data already holds them, converted) to data, writes the pad tail from carry_in (the
// receiver's device carry; nullptr: its stream starts, the tail is no signal) and stores the last
// MODES_CARRY_BYTES of the buffer to carry_out.  in and data are 16-byte aligned, the three carry spans
// 4-byte aligned; carry_out is never carry_in.
struct PoolGatherJob {
    const uint8_t *in;
    uint8_t       *data;
    const uint8_t *carry_in;
    uint8_t       *carry_out;
    uint8_t       *pad_tail;
};
void launch_gather_pool(const PoolGatherJob *d_jobs, uint32_t n_jobs, cudaStream_t stream);
// A device-fed call's refusal of memory that is not device memory of `device` (modes_process_device,
// modes_pool_submit_device): empty when p is such memory, else what it is, for the caller's message
// (`owner`: whose device; `host_call`: the call for host memory).
std::string device_input_refusal(const void *p, int device, const char *owner, const char *host_call);
// The input spectrum pass (modes_spectrum.cu, K13; arithmetic in modes_spectrum_core.cuh): out[k] = the record of
// reference buffer first_buffer + k, k < n_buffers, of a stream at the ratio out : in (InputRate) whose input
// span the job holds (in, in_bytes, in_first: as launch_decimate reads them, UC8 with shift < 0, else int16
// converted with the shift).  The records must be zero: each block adds its frames' power into its buffer's.
void launch_spectrum(const ResampleJob &j, int shift, int out, int in, int64_t first_buffer, uint32_t n_buffers,
                     modes_spectrum *records, cudaStream_t stream);
// The receiver pool's form: one job per pair of a batch, record k from job k.  A job's input is read as a
// PoolResampleJob's ([hist0, call0) at hist, [call0, call0 + MODES_BUFFER_BYTES) at stage, UC8 stream bytes):
// its buffer's frames of `frames` start at stream sample `first`.  A 2 MHz receiver's job has hist0 = call0 =
// 2 first and stage = its pair's data buffer.  max_frames: the most frames of a job.
struct PoolSpectrumJob {
    const uint8_t *hist;
    const uint8_t *stage;
    int64_t        hist0, call0;
    int64_t        buffer;       // the receiver's own buffer index
    int64_t        first;
    uint32_t       frames;
    uint32_t       pad;
};
void launch_spectrum_pool(const PoolSpectrumJob *d_jobs, uint32_t n_jobs, uint32_t max_frames, modes_spectrum *records,
                          cudaStream_t stream);
static_assert(sizeof(modes_spectrum) == 16 + 8 * MODES_SPECTRUM_BINS && offsetof(modes_spectrum, power) == 16,
              "spectrum record layout");
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
static_assert(offsetof(modes_message, recovered) == 14 && offsetof(modes_message, arrival) == 15 &&
              offsetof(modes_message, msgbits) == 16 && offsetof(modes_message, carrier) == 106 &&
              offsetof(modes_message, ew_dir) == 108 && sizeof(modes_message) == 200, "message layout");

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
    // A part of the stream judged on its own after `from`: from's cache and skip state, totals zeroed;
    // at_buffer: the part starts at a buffer boundary (no skip state).
    void start_part(const ResolveState &from, bool at_buffer);
    // Take over a finished part's cache and add its totals.  The skip state is left to the caller.
    void fold_part(const ResolveState &part);
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

// One record array as the resolve takes it: a batch's candidate records and tile table, and the stream's
// buffer number of the array's buffer 0 (buffer numbers in the records: t >> 17).  recovered: one record
// per candidate (modes_recover.cu), or nullptr with recovery off; weak: the weak positions merged into the
// walk (only with recovered); carrier: one carrier record per candidate (modes_signal.cu), or nullptr with
// carrier measurement off.  Only the candidates and weak positions of the buffers [b_lo, b_hi) are judged.
struct Shard {
    const modes_candidate *cands = nullptr;
    const modes_tile *tiles = nullptr;
    size_t n_tiles = 0;
    int64_t buffer_base = 0;
    const modes_recovered *recovered = nullptr;
    WeakList weak{};
    const modes_carrier *carrier = nullptr;
    uint32_t b_lo = 0, b_hi = UINT32_MAX;
};

void resolve_candidates(ResolveState &st, const ResolveConfig &cfg, const Shard &shard, MessageOut &out, ResolveScratch *scratch);
void resolve_shards(ResolveState &st, const ResolveConfig &cfg, const Shard *shards, size_t n_shards, MessageOut &out,
                    ResolveScratch *scratch);
// A shard resolved from a GUESSED address cache (one rank / one GPU thread of a sharded decode):
// verdicts only, deliveries held back in the scratch until the guess is verified.
void resolve_tentative(ResolveState &st, const ResolveConfig &cfg, const Shard &shard, ResolveScratch *scratch);
void resolve_commit(MessageOut &out, ResolveScratch *scratch);
// Messages from the device resolve's delivery records (structs built in parallel, sink called in order).
void deliver_gpu(const modes_delivery *d, size_t n, int64_t buffer_base, MessageOut &out);
// The order-dependent tail of decodeModesMessage + field decode for one evaluated frame.
int finish_message(ResolveState &st, const modes_frame_eval &p, modes_message *out);

// ---- host glue shared by the context (modes_api.cpp) and the receiver pool (modes_pool.cpp) ----
// An owning, grow-only array of T in device memory (DevBuf) or pinned host memory (PinnedBuf).
// ensure(n) replaces the array with one of exactly n elements when n exceeds its capacity, without
// keeping the contents; the caller chooses n, so each growth policy stays where the array is used.
template <typename T, bool Pinned>
class CudaBuf {
public:
    CudaBuf() = default;
    CudaBuf(CudaBuf &&o) noexcept : p_(o.p_), cap_(o.cap_) { o.p_ = nullptr; o.cap_ = 0; }
    CudaBuf &operator=(CudaBuf &&o) noexcept {
        if (this != &o) { release(); p_ = o.p_; cap_ = o.cap_; o.p_ = nullptr; o.cap_ = 0; }
        return *this;
    }
    ~CudaBuf() { release(); }
    cudaError_t ensure(size_t n) {
        if (n <= cap_) return cudaSuccess;
        release();
        void *p = nullptr;
        const cudaError_t e = Pinned ? cudaMallocHost(&p, n * sizeof(T)) : cudaMalloc(&p, n * sizeof(T));
        if (e != cudaSuccess) return e;
        p_ = static_cast<T *>(p);
        cap_ = n;
        return cudaSuccess;
    }
    T *get() const { return p_; }
    T &operator[](size_t i) const { return p_[i]; }
    size_t capacity() const { return cap_; }
private:
    void release() {
        if (p_) { if (Pinned) cudaFreeHost(p_); else cudaFree(p_); }
        p_ = nullptr;
        cap_ = 0;
    }
    T *p_ = nullptr;
    size_t cap_ = 0;
};
template <typename T> using DevBuf = CudaBuf<T, false>;
template <typename T> using PinnedBuf = CudaBuf<T, true>;

// The optional measurements and searches of a decode (modes_set_* / modes_pool_set_*).
struct Features { bool signal = false, arrival = false, levels = false, recover = false, weak = false, spectrum = false, carrier = false; };

// The last modes_detect_device batch's records (the receiver pool's slot contexts), in the context's pinned
// memory, with those of the passes it ran with its own arrays (recovery, weak preambles, carrier): waits for
// the batch, copies them and waits once.  The shard is valid until the context's next batch.
int detect_shard(modes_ctx *ctx, Shard &shard);

// Level or spectrum records not taken yet, oldest first.
template <typename T>
class RecordQueue {
public:
    void push(const T &r) { q_.push_back(r); }
    void clear() { q_.clear(); head_ = 0; }
    // Moves up to cap of the oldest records to out; out == nullptr: how many are queued.
    size_t take(T *out, size_t cap) {
        const size_t queued = q_.size() - head_;
        if (!out) return queued;
        const size_t n = cap < queued ? cap : queued;
        if (n) memcpy(out, q_.data() + head_, n * sizeof(T));
        head_ += n;
        if (head_ == q_.size()) clear();
        else if (head_ >= 4096 && 2 * head_ >= q_.size()) {   // compact when the taken records are half the queue
            q_.erase(q_.begin(), q_.begin() + (ptrdiff_t)head_);
            head_ = 0;
        }
        return n;
    }
private:
    std::vector<T> q_;
    size_t head_ = 0;
};
using LevelQueue = RecordQueue<modes_level>;
using SpectrumQueue = RecordQueue<modes_spectrum>;

}  // namespace modes
