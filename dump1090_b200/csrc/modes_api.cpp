// modes_api.cpp — the C ABI declared in include/modes_b200.h: context, device
// workspaces, the two-slot host->device pipeline, and glue to the kernels
// (modes_kernels.cu) and the sequential resolve (modes_resolve.cpp).
//
// No CPU fallback: every entry point that computes runs the CUDA kernels, and
// modes_create() fails when no device is usable.
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <new>
#include <string>
#include <vector>
#include "modes_internal.h"
#include "modes_input_core.cuh"
#include "modes_resample_core.cuh"

using namespace modes;

namespace {

thread_local std::string g_create_error;

// Pinned room for a host copy of n records, with half as much again to spare so that slowly rising
// counts do not reallocate every batch.
template <typename T>
cudaError_t ensure_spare(PinnedBuf<T> &b, size_t n) { return b.capacity() >= n ? cudaSuccess : b.ensure(n + n / 2 + 1024); }

struct Slot {
    cudaStream_t stream = nullptr;
    DevBuf<uint8_t> d_iq;
    DevBuf<uint8_t> d_halo;
    DevBuf<uint8_t> d_in;             // 2.4 MS/s or 16-bit input: the input bytes the batch is made from
    DevBuf<uint32_t> d_cand_v;       // its capacity is the slot's candidate capacity
    DevBuf<modes_candidate> d_records;
    DevBuf<modes_tile> d_tiles;
    // two counter sets (ScanOutputs), used in turn: `set` is the last batch's, and its scan zeroed the
    // other one for the slot's next batch (whose scan runs after every pass that reads this batch's set)
    DevBuf<uint32_t> d_counters;     // 2 x kCounterWords
    unsigned set = 1;
    uint32_t *counters() const { return d_counters.get() + kCounterWords * set; }
    // the last batch's candidate count and overflow flag, written by its scan (mapped pinned memory)
    uint32_t *h_counts = nullptr;
    // the batch's carry block, passed to the scan by value (carry_on_host), or already on the device in
    // d_halo (the resampler writes it there)
    uint8_t carry[kHaloAlloc];
    bool carry_on_host = false;
    PinnedBuf<modes_candidate> h_records;
    PinnedBuf<modes_tile> h_tiles;
    // the batch's last operation on the stream (what wait_batch waits for); never timed, so that recording it
    // costs the stream no timestamp
    cudaEvent_t done = nullptr;
    // cfg.gpu_resolve: workspace of the device resolve (the storage behind a GpuResolve view)
    DevBuf<uint32_t> gr_start, gr_end, gr_written, gr_readfirst, gr_rerun, gr_n_deliv, gr_offsets, gr_flags;
    DevBuf<uint64_t> gr_stats;
    DevBuf<modes_delivery> gr_out;
    PinnedBuf<uint32_t> h_gr_flags;  // flags[3] + pad, then stats[8] as u64, then the end cache [1024]
    PinnedBuf<modes_delivery> h_deliveries;
    // modes_set_levels: one record per buffer of the batch (device, and its pinned host copy)
    DevBuf<modes_level> d_levels;
    PinnedBuf<modes_level> h_levels;
    // modes_set_spectrum: one record per buffer of the batch (device, pinned host copy), and the input span
    // the batch was made from (spec_shift < 0: UC8, else int16 with that shift)
    DevBuf<modes_spectrum> d_spectra;
    PinnedBuf<modes_spectrum> h_spectra;
    ResampleJob spec_in{};
    int spec_shift = -1;
    // modes_set_recovery / modes_recover_device: one record per candidate (device, and its pinned host copy)
    DevBuf<modes_recovered> d_recovered;
    PinnedBuf<modes_recovered> h_recovered;
    // modes_set_carrier: one record per candidate (device, and its pinned host copy)
    DevBuf<modes_carrier> d_carrier;
    PinnedBuf<modes_carrier> h_carrier;
    // modes_set_weak_preambles / modes_weak_device: the weak positions and their records (device), the
    // scan's unordered scratch list (its capacity is the slot's weak capacity), its per-tile words
    // (source, count and destination of every tile's block) and counters, and pinned host copies
    DevBuf<uint32_t> d_weak_pos;
    DevBuf<modes_recovered> d_weak_rec;
    DevBuf<uint32_t> d_weak_scratch;
    uint32_t want_weak_cap = 0;
    DevBuf<uint32_t> d_weak_tiles;
    DevBuf<uint32_t> d_weak_counters;
    PinnedBuf<uint32_t> h_weak_counters;
    PinnedBuf<uint32_t> h_weak_pos;
    PinnedBuf<modes_recovered> h_weak_rec;
    // in-flight batch
    bool busy = false;
    size_t n_buffers = 0;
    int64_t buffer_base = 0;
    const void *batch_iq = nullptr;   // device address the batch was scanned from
    bool own_outputs = true;          // results in this slot's own buffers (growable)
    // the batch's passes: the switches as they were at submit (the stage level adds recovery and weak
    // preambles with modes_recover_device / modes_weak_device)
    Features feat;
    uint32_t *weak_pos_ext = nullptr; modes_recovered *weak_rec_ext = nullptr; uint32_t weak_ext_cap = 0;   // modes_weak_device's buffers
    uint32_t weak_first = 0, weak_step = 1;   // the buffers the weak scan reads: weak_first + i * weak_step
    modes_recovered *rec_ext = nullptr; uint32_t rec_ext_cap = 0;   // modes_recover_device's d_out (nullptr: own buffer)
    uint32_t want_cap = 0;            // grow the candidate buffers to at least this on the next ensure
    // where this batch's results live (own workspace unless the caller supplied memory)
    modes_candidate *out_records = nullptr;
    modes_tile *out_tiles = nullptr;
    uint32_t out_cap = 0;
    uint32_t cand_cap() const { return (uint32_t)d_cand_v.capacity(); }
    uint32_t weak_cap() const { return (uint32_t)d_weak_scratch.capacity(); }
};

}  // namespace

struct modes_ctx {
    modes_config cfg;
    int sm_count = 132;
    DevBuf<uint16_t> d_lutn, d_lut_iq;
    DevBuf<uint32_t> d_bit_syn, d_fix_hash, d_pair_hash;
    DeviceTables tab{};
    Slot slot[2];
    Slot detect;                      // stage-level API workspace
    // cfg.n_gpus > 1: this context is the front of a multi-GPU decode and owns one single-GPU
    // context per device; it keeps the stream state, the resolve state and the outputs itself
    // cfg.gpu_resolve: the address cache lives on the device, handed from batch to batch
    DevBuf<uint32_t> d_cache[2];
    int cache_cur = 0;
    cudaEvent_t ev_resolved = nullptr;    // the last batch's device resolve has finished (its cache_out is valid)
    bool resolved_pending = false;
    // hex door staging (modes_decode_frames)
    DevBuf<uint8_t> d_frames;
    DevBuf<modes_frame_eval> d_frame_evals;
    PinnedBuf<modes_frame_eval> h_frame_evals;
    std::vector<modes_ctx *> gpus;
    size_t group_n[2] = {0, 0};       // batches in flight per slot parity
    uint64_t last_detect_count = 0;
    // stream state
    PinnedBuf<uint8_t> pending;       // one reference buffer
    size_t pending_len = 0;
    uint8_t carry[MODES_CARRY_BYTES];
    // which memory the stream is fed from (modes_process or modes_process_device), fixed by its first call
    enum class Feed { none, host, device } feed = Feed::none;
    // a device-fed stream's twins of pending, carry and hold, on cfg.device: created by its first call.  The
    // hold lives in two halves used in turn, so that keeping its tail never copies a range onto itself.
    DevBuf<uint8_t> d_pending;
    DevBuf<uint8_t> d_carry;
    DevBuf<uint8_t> d_hold[2];
    int hold_cur = 0;
    int64_t buffers_done = 0;
    bool finished = false;
    bool started = false;                 // modes_process or modes_finish since create / reset
    // modes_set_input_rate / modes_set_input_format: at 2.4 MS/s or more, or in a 16-bit format, each batch's
    // 2 MHz UC8 bytes are made on the device (K9 resamples, K11 decimates, K10 converts) from the stream's
    // input bytes; they never exist on the host.  hold keeps the stream bytes [hold0, in_total) that later
    // batches read (the filter's history and a buffer not yet complete).  input_shift: the format's shift,
    // default resolved.
    const InputRate *rate = find_input_rate(2000000);
    uint32_t input_format = input::kUC8;
    int input_shift = 0;
    // modes_set_input_offset: where 1090 MHz sits in the capture's baseband (0 unless rate->m); K12 rotates
    // the input by it as it decimates.  The pair (rate, input_offset) is always one the setters accept.
    int32_t input_offset = 0;
    int64_t in_total = 0;
    PinnedBuf<uint8_t> hold;
    int64_t hold0 = 0;
    // modes_resample_device: the carry block (device, pinned host copy)
    DevBuf<uint8_t> d_rs_halo;
    PinnedBuf<uint8_t> h_rs_halo;
    ResolveState rs;
    ResolveScratch *scratch = nullptr;
    MessageOut out;                       // modes_set_sink / modes_set_output
    cudaStream_t own_detect_stream = nullptr;
    std::string err;
    uint64_t launches = 0;                // this context's own; a multi-GPU front adds its GPUs' (modes_launch_count)
    // signal, arrival: measured on decoded attempts; levels: of every decoded buffer; recover:
    // soft-decision recovery of weak DF17/18 frames; weak: recovery at weak preambles too
    Features feat;
    LevelQueue level_q;
    SpectrumQueue spectrum_q;
    int64_t eof_buffer = -1;              // modes_finish: stream index of the EOF buffer and its real samples
    uint32_t eof_samples = 0;
    // modes_levels_device: the records of the last call (device, pinned host copy)
    DevBuf<modes_level> d_lv;
    PinnedBuf<modes_level> h_lv;
    size_t lv_n = 0;
    bool lv_fetched = true;               // no copy of them is pending
    // cfg.profile: ring of CUDA-event triplets, one per batch, recorded on the launching stream
    static constexpr int kProfRing = 512;
    cudaEvent_t prof_ev[kProfRing][3];
    bool prof_ready = false;
    uint64_t prof_head = 0, prof_tail = 0;   // batches recorded / batches already reported
};

namespace {

int fail(modes_ctx *ctx, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    if (ctx) ctx->err = buf; else g_create_error = buf;
    return -1;
}

#define CK(ctx, call)                                                                   \
    do {                                                                                \
        cudaError_t e_ = (call);                                                        \
        if (e_ != cudaSuccess)                                                          \
            return fail(ctx, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
    } while (0)

// How host threads wait for the GPU.  0 (default): the CUDA runtime's own choice, which spins on a
// many-core host — lowest latency, one core busy per waiting thread.  1: sleep until the GPU signals
// (events with cudaEventBlockingSync) — for hosts that run more ranks than they have cores to burn,
// e.g. eight one-GPU processes under a small cgroup CPU quota.  Process-wide; contexts pick it up
// when they are created.  MODES_HOST_WAIT=block sets the initial value.
std::atomic<int> g_host_wait{-1};

int host_wait_mode() {
    int m = g_host_wait.load(std::memory_order_relaxed);
    if (m < 0) {
        const char *e = std::getenv("MODES_HOST_WAIT");
        m = (e && (*e == 'b' || *e == 'B' || *e == '1')) ? 1 : 0;
        g_host_wait.store(m, std::memory_order_relaxed);
    }
    return m;
}

unsigned event_flags(bool timing) {
    return (timing ? 0u : (unsigned)cudaEventDisableTiming) | (host_wait_mode() ? (unsigned)cudaEventBlockingSync : 0u);
}

// cudaStreamSynchronize, or its sleeping equivalent (the stream must belong to the current device).
cudaError_t wait_stream(cudaStream_t st) {
    if (!host_wait_mode()) return cudaStreamSynchronize(st);
    static thread_local cudaEvent_t ev[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return cudaStreamSynchronize(st);
    if (!ev[dev] && cudaEventCreateWithFlags(&ev[dev], cudaEventDisableTiming | cudaEventBlockingSync) != cudaSuccess) {
        ev[dev] = nullptr;
        (void)cudaGetLastError();
        return cudaStreamSynchronize(st);
    }
    if (cudaEventRecord(ev[dev], st) != cudaSuccess) { (void)cudaGetLastError(); return cudaStreamSynchronize(st); }
    return cudaEventSynchronize(ev[dev]);
}

uint32_t default_cand_capacity(uint64_t n_samples) {
    uint64_t c = n_samples / 64 + 4096;
    return c > 0xFFFFFFF0ull ? 0xFFFFFFF0u : (uint32_t)c;
}

int slot_init(modes_ctx *ctx, Slot &s) {
    CK(ctx, cudaStreamCreateWithFlags(&s.stream, cudaStreamNonBlocking));
    CK(ctx, s.d_halo.ensure(kHaloAlloc));
    CK(ctx, s.d_counters.ensure(2 * kCounterWords));
    CK(ctx, cudaMemsetAsync(s.d_counters.get(), 0, 2 * kCounterWords * sizeof(uint32_t), s.stream));
    CK(ctx, cudaStreamSynchronize(s.stream));
    void *h = nullptr;
    CK(ctx, cudaHostAlloc(&h, 2 * sizeof(uint32_t), cudaHostAllocMapped));
    s.h_counts = static_cast<uint32_t *>(h);
    s.h_counts[0] = s.h_counts[1] = 0;
    CK(ctx, cudaEventCreateWithFlags(&s.done, event_flags(false)));
    return 0;
}

void slot_free(Slot &s) {
    if (s.stream) wait_stream(s.stream);
    if (s.done) cudaEventDestroy(s.done);
    if (s.h_counts) cudaFreeHost(s.h_counts);
    if (s.stream) cudaStreamDestroy(s.stream);
    s = Slot();                       // releases its buffers: nothing queued uses them any more
}

// Make sure the slot can hold a batch of n_samples (device staging only if need_iq).
int slot_ensure(modes_ctx *ctx, Slot &s, uint64_t n_samples, bool need_iq, bool need_records) {
    if (need_iq) CK(ctx, s.d_iq.ensure(n_samples * 2));
    uint32_t cap = default_cand_capacity(n_samples);
    if (cap < s.want_cap) cap = s.want_cap;
    CK(ctx, s.d_cand_v.ensure(cap));
    if (need_records) CK(ctx, s.d_records.ensure(s.cand_cap()));
    CK(ctx, s.d_tiles.ensure(tiles_for(n_samples)));
    return 0;
}

int launch_batch(modes_ctx *ctx, Slot &s);

// Queue the level records of the slot's finished batch, re-based to stream buffer indices.
void append_levels(modes_ctx *ctx, const Slot &s) {
    if (!s.feat.levels) return;
    for (size_t k = 0; k < s.n_buffers; k++) {
        modes_level r = s.h_levels[k];
        r.buffer = s.buffer_base + (int64_t)k;
        if (r.buffer == ctx->eof_buffer) r.n_samples = ctx->eof_samples;
        ctx->level_q.push(r);
    }
}

// Queue the spectrum records of the slot's finished batch (the kernel wrote their stream buffer indices).
void append_spectra(modes_ctx *ctx, const Slot &s) {
    if (!s.feat.spectrum) return;
    for (size_t k = 0; k < s.n_buffers; k++) ctx->spectrum_q.push(s.h_spectra[k]);
}

// The device resolve's view of the slot's workspace, grown for its current batch.
int gpu_resolve_ensure(modes_ctx *ctx, Slot &s, GpuResolve &g) {
    const size_t nb = s.n_buffers;
    CK(ctx, s.gr_start.ensure(nb * 1024)); CK(ctx, s.gr_end.ensure(nb * 1024));
    CK(ctx, s.gr_written.ensure(nb * 32)); CK(ctx, s.gr_readfirst.ensure(nb * 32));
    CK(ctx, s.gr_rerun.ensure(nb)); CK(ctx, s.gr_n_deliv.ensure(nb)); CK(ctx, s.gr_offsets.ensure(nb + 1));
    CK(ctx, s.gr_flags.ensure(4));
    CK(ctx, s.gr_stats.ensure(8));
    CK(ctx, s.h_gr_flags.ensure(20 + 1024));
    // at most two deliveries per candidate (check_crc = 0 delivers a failed first attempt and its
    // retry), so the deliveries fit whenever the candidates do
    CK(ctx, s.gr_out.ensure(2 * (size_t)s.cand_cap()));
    g = GpuResolve{s.gr_start.get(), s.gr_end.get(), s.gr_written.get(), s.gr_readfirst.get(), s.gr_rerun.get(),
                   s.gr_n_deliv.get(), s.gr_offsets.get(), s.gr_flags.get(), nullptr, nullptr, s.gr_stats.get(),
                   s.gr_out.get(), (uint32_t)s.gr_out.capacity()};
    return 0;
}

// Queue one batch on the slot's stream: (optional H2D) + scan + frame evaluation.  halo_on_device: the
// slot's carry block is already queued on the stream (the resampler writes it), so carry476 is unused.
int submit(modes_ctx *ctx, Slot &s, const uint8_t *host_iq, const void *d_iq, size_t n_buffers,
           const uint8_t *carry476, modes_candidate *d_records_ext, uint32_t cap_ext, modes_tile *d_tiles_ext,
           bool halo_on_device = false) {
    const uint64_t n_samples = (uint64_t)n_buffers * kBufSamples;
    if (n_samples + kHaloSamples >= (1ull << 32)) return fail(ctx, "batch too large: %zu buffers", n_buffers);
    // caller-supplied record buffers: the slot's own position list must hold as many candidates
    if (d_records_ext && cap_ext > s.want_cap) s.want_cap = cap_ext;
    if (slot_ensure(ctx, s, n_samples, host_iq != nullptr, d_records_ext == nullptr)) return -1;
    s.feat = ctx->feat;
    s.feat.levels &= &s != &ctx->detect;
    s.feat.spectrum &= &s != &ctx->detect;
    s.feat.recover &= &s != &ctx->detect;                 // the stage level asks with modes_recover_device
    s.rec_ext = nullptr; s.rec_ext_cap = 0;
    s.feat.weak &= s.feat.recover;                        // the stage level asks with modes_weak_device
    s.weak_pos_ext = nullptr; s.weak_rec_ext = nullptr; s.weak_ext_cap = 0;
    s.weak_first = 0; s.weak_step = 1;
    if (s.feat.levels) {                                  // the slot's previous batch is collected: no copy is queued
        CK(ctx, s.d_levels.ensure(n_buffers));
        CK(ctx, s.h_levels.ensure(n_buffers));
    }
    if (s.feat.spectrum) {
        CK(ctx, s.d_spectra.ensure(n_buffers));
        CK(ctx, s.h_spectra.ensure(n_buffers));
    }
    if (host_iq) {
        CK(ctx, cudaMemcpyAsync(s.d_iq.get(), host_iq, n_samples * 2, cudaMemcpyHostToDevice, s.stream));
        d_iq = s.d_iq.get();
    }
    if ((reinterpret_cast<uintptr_t>(d_iq) & 15) != 0) return fail(ctx, "device I/Q pointer must be 16-byte aligned");
    s.carry_on_host = !halo_on_device;
    if (s.carry_on_host) {
        memset(s.carry, 127, kHaloAlloc);                                 // dump1090.c:344 no-signal
        if (carry476) memcpy(s.carry + (kHaloBytes - MODES_CARRY_BYTES), carry476, MODES_CARRY_BYTES);
    }
    s.batch_iq = d_iq;
    s.n_buffers = n_buffers;
    s.own_outputs = d_records_ext == nullptr;
    s.out_records = d_records_ext ? d_records_ext : s.d_records.get();
    s.out_tiles = d_tiles_ext ? d_tiles_ext : s.d_tiles.get();
    s.out_cap = d_records_ext ? (cap_ext < s.cand_cap() ? cap_ext : s.cand_cap()) : s.cand_cap();
    return launch_batch(ctx, s);
}

// The recovery pass over the slot's batch and records, into the caller's array or the slot's own
// (grown to the record capacity).
int launch_recovery(modes_ctx *ctx, Slot &s, const BatchView &in, const ScanOutputs &so) {
    modes_recovered *dst = s.rec_ext;
    uint32_t cap = s.rec_ext_cap < s.out_cap ? s.rec_ext_cap : s.out_cap;
    if (!dst) {
        CK(ctx, s.d_recovered.ensure(s.out_cap));
        dst = s.d_recovered.get();
        cap = s.out_cap;
    }
    launch_recover(in, ctx->tab, so, s.out_records, cap, dst, ctx->sm_count, s.stream);
    CK(ctx, cudaGetLastError());
    ctx->launches++;
    return 0;
}

// The weak-preamble scan and the search at its positions over the slot's batch, into the caller's
// arrays or the slot's own, and the count to pinned memory.  The slot's own arrays (the scan's scratch
// list always) are grown to want_weak_cap.
int launch_weak(modes_ctx *ctx, Slot &s, const BatchView &in) {
    const uint32_t n_scan = s.weak_first < s.n_buffers ? (uint32_t)((s.n_buffers - 1 - s.weak_first) / s.weak_step + 1) : 0u;
    const uint64_t scan_samples = (uint64_t)n_scan * kBufSamples;
    CK(ctx, s.d_weak_tiles.ensure(3 * (size_t)weak_tiles_for(n_scan)));
    CK(ctx, s.d_weak_counters.ensure(2));
    CK(ctx, s.h_weak_counters.ensure(2));
    // a weak position passes the shape test, which two neighbours never both pass: at most one in two
    uint64_t want = scan_samples / 512 + 4096;
    if (want < s.want_weak_cap) want = s.want_weak_cap;
    if (want > scan_samples / 2 + 1) want = scan_samples / 2 + 1;
    CK(ctx, s.d_weak_pos.ensure(want));
    CK(ctx, s.d_weak_rec.ensure(want));
    CK(ctx, s.d_weak_scratch.ensure(want));
    uint32_t *pos = s.weak_pos_ext ? s.weak_pos_ext : s.d_weak_pos.get();
    modes_recovered *rec = s.weak_pos_ext ? s.weak_rec_ext : s.d_weak_rec.get();
    const uint32_t cap = s.weak_pos_ext ? s.weak_ext_cap : s.weak_cap();
    launch_weak_scan(in, ctx->tab,
                     WeakOutputs{s.weak_first, s.weak_step, n_scan, pos, cap, s.d_weak_scratch.get(), s.weak_cap(),
                                 s.d_weak_tiles.get(), s.d_weak_counters.get()},
                     ctx->sm_count, s.stream);
    launch_recover_weak(in, ctx->tab, s.d_weak_counters.get() + 1, cap, s.weak_cap(), pos, rec, ctx->sm_count, s.stream);
    CK(ctx, cudaGetLastError());
    ctx->launches += 4;
    CK(ctx, cudaMemcpyAsync(s.h_weak_counters.get(), s.d_weak_counters.get(), 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s.stream));
    return 0;
}

// The weak positions of the slot's last batch exceed its scratch list (and its own output arrays):
// the batch is repeated with larger ones.  A caller's smaller arrays only report the count.
bool weak_overflowed(const Slot &s) {
    return s.feat.weak && s.h_weak_counters[1] > s.weak_cap();
}

// The two kernels over the slot's staged batch (also used to repeat a batch that overflowed).
int launch_batch(modes_ctx *ctx, Slot &s) {
    const uint64_t n_samples = (uint64_t)s.n_buffers * kBufSamples;
    // a repeated batch takes the other set too: the first run's scan zeroed it
    s.set ^= 1;
    BatchView in{static_cast<const uint8_t *>(s.batch_iq), s.d_halo.get(), n_samples};
    ScanOutputs so{s.d_cand_v.get(), s.out_cap, s.out_tiles, s.counters(),
                   s.d_counters.get() + kCounterWords * (s.set ^ 1), s.h_counts};

    cudaEvent_t *pe = nullptr;
    if (ctx->cfg.profile) {
        if (!ctx->prof_ready) {
            for (auto &trip : ctx->prof_ev) for (auto &e : trip) CK(ctx, cudaEventCreateWithFlags(&e, event_flags(true)));
            ctx->prof_ready = true;
        }
        if (ctx->prof_head - ctx->prof_tail >= (uint64_t)modes_ctx::kProfRing) ctx->prof_tail = ctx->prof_head - modes_ctx::kProfRing + 1;
        pe = ctx->prof_ev[ctx->prof_head % modes_ctx::kProfRing];
        ctx->prof_head++;
    }
    if (pe) CK(ctx, cudaEventRecord(pe[0], s.stream));
    launch_scan(in, ctx->tab, so, ctx->sm_count, s.stream, s.carry_on_host ? s.carry : nullptr);
    if (pe) CK(ctx, cudaEventRecord(pe[1], s.stream));
    launch_eval(in, ctx->tab, so, s.out_records, ctx->cfg.fix_errors, ctx->cfg.aggressive, ctx->sm_count, s.stream);
    if (pe) CK(ctx, cudaEventRecord(pe[2], s.stream));
    // after pe[2]: the kernel times keep their meaning; before the device resolve, which copies the field
    const Features &f = s.feat;
    if (f.carrier) CK(ctx, s.d_carrier.ensure(s.out_cap));
    if (f.signal || f.arrival || f.carrier)
        launch_signal(in, ctx->tab, so, s.out_records, ctx->sm_count, s.stream, f.signal, f.arrival, f.carrier ? s.d_carrier.get() : nullptr);
    // the buffers' own bytes (the body, not the carry block); one writer per record, so a repeated
    // batch writes the same records
    if (f.levels)
        launch_levels(in.body, (uint32_t)s.n_buffers, MODES_BUFFER_BYTES, ctx->tab, s.d_levels.get(), ctx->sm_count, s.stream);
    // the input the buffers stand for, where the batch was made from; the records start from zero
    if (f.spectrum) {
        CK(ctx, cudaMemsetAsync(s.d_spectra.get(), 0, s.n_buffers * sizeof(modes_spectrum), s.stream));
        launch_spectrum(s.spec_in, s.spec_shift, ctx->rate->out, ctx->rate->in, s.buffer_base, (uint32_t)s.n_buffers,
                        s.d_spectra.get(), s.stream);
    }
    CK(ctx, cudaGetLastError());
    ctx->launches += (f.signal || f.arrival || f.carrier ? 3 : 2) + (f.levels ? 1 : 0) + (f.spectrum ? 1 : 0);
    if (f.recover && launch_recovery(ctx, s, in, so)) return -1;
    if (f.weak && launch_weak(ctx, s, in)) return -1;
    if (ctx->cfg.gpu_resolve && s.own_outputs && &s != &ctx->detect) {
        GpuResolve g;
        if (gpu_resolve_ensure(ctx, s, g)) return -1;
        // the address cache comes from the previous batch's resolve (other slot, other stream)
        if (ctx->resolved_pending) CK(ctx, cudaStreamWaitEvent(s.stream, ctx->ev_resolved, 0));
        g.cache_in = ctx->d_cache[ctx->cache_cur].get();
        g.cache_out = ctx->d_cache[ctx->cache_cur ^ 1].get();
        ctx->cache_cur ^= 1;
        launch_gpu_resolve(g, s.out_records, s.out_tiles, tiles_for(n_samples), (uint32_t)s.n_buffers, ctx->cfg.check_crc,
                           ctx->sm_count, s.stream);
        CK(ctx, cudaGetLastError());
        ctx->launches += 4 + 2 * kGpuResolveRounds;
        CK(ctx, cudaEventRecord(ctx->ev_resolved, s.stream));
        ctx->resolved_pending = true;
        uint32_t *h = s.h_gr_flags.get();
        CK(ctx, cudaMemcpyAsync(h, g.flags, 4 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s.stream));
        CK(ctx, cudaMemcpyAsync(h + 4, g.stats_out, 8 * sizeof(uint64_t), cudaMemcpyDeviceToHost, s.stream));
        CK(ctx, cudaMemcpyAsync(h + 20, g.cache_out, 1024 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s.stream));
    }
    if (f.levels)
        CK(ctx, cudaMemcpyAsync(s.h_levels.get(), s.d_levels.get(), s.n_buffers * sizeof(modes_level), cudaMemcpyDeviceToHost, s.stream));
    if (f.spectrum)
        CK(ctx, cudaMemcpyAsync(s.h_spectra.get(), s.d_spectra.get(), s.n_buffers * sizeof(modes_spectrum), cudaMemcpyDeviceToHost,
                                s.stream));
    CK(ctx, cudaEventRecord(s.done, s.stream));
    s.busy = true;
    return 0;
}

// Wait for the slot's batch; returns the number of candidates stored.  A batch denser than the
// candidate buffers (default: one candidate per 64 samples) is repeated with larger buffers when
// they are the slot's own; caller-supplied buffers cannot grow and report the overflow.
int wait_batch(modes_ctx *ctx, Slot &s, uint64_t *n_out) {
    for (;;) {
        CK(ctx, cudaEventSynchronize(s.done));
        const bool cand_over = s.h_counts[1] || s.h_counts[0] > s.out_cap;
        if (!cand_over && !weak_overflowed(s)) break;
        if (ctx->cfg.gpu_resolve && &s != &ctx->detect) break;           // reported by collect(): the device resolve ran on a truncated list
        if (cand_over) {
            const uint32_t found = s.h_counts[0];
            if (!s.own_outputs)
                return fail(ctx, "candidate capacity exceeded: %u found, room for %u", found, s.out_cap);
            s.want_cap = found + found / 8 + 1024;
            if (slot_ensure(ctx, s, (uint64_t)s.n_buffers * kBufSamples, false, true)) return -1;
            s.out_records = s.d_records.get();
            s.out_cap = s.cand_cap();
        }
        if (weak_overflowed(s)) s.want_weak_cap = s.h_weak_counters[1] + s.h_weak_counters[1] / 8 + 1024;
        if (launch_batch(ctx, s)) return -1;
    }
    *n_out = s.h_counts[0];
    return 0;
}

// Queue the copies of the slot's finished batch (n candidate records) to pinned memory on its
// stream; the shard is valid once the stream has been waited for.
int fetch_async(modes_ctx *ctx, Slot &s, uint64_t n, Shard &v) {
    const size_t nt = tiles_for((uint64_t)s.n_buffers * kBufSamples);
    CK(ctx, ensure_spare(s.h_records, n));
    CK(ctx, s.h_tiles.ensure(nt));
    if (n) CK(ctx, cudaMemcpyAsync(s.h_records.get(), s.out_records, n * sizeof(modes_candidate), cudaMemcpyDeviceToHost, s.stream));
    if (s.feat.recover) {
        CK(ctx, ensure_spare(s.h_recovered, n));
        if (n) CK(ctx, cudaMemcpyAsync(s.h_recovered.get(), s.d_recovered.get(), n * sizeof(modes_recovered), cudaMemcpyDeviceToHost, s.stream));
    }
    WeakList wl;
    if (s.feat.weak) {
        const size_t nw = s.h_weak_counters[1];
        CK(ctx, ensure_spare(s.h_weak_pos, nw));
        CK(ctx, ensure_spare(s.h_weak_rec, nw));
        if (nw) {
            CK(ctx, cudaMemcpyAsync(s.h_weak_pos.get(), s.d_weak_pos.get(), nw * sizeof(uint32_t), cudaMemcpyDeviceToHost, s.stream));
            CK(ctx, cudaMemcpyAsync(s.h_weak_rec.get(), s.d_weak_rec.get(), nw * sizeof(modes_recovered), cudaMemcpyDeviceToHost, s.stream));
        }
        wl = WeakList{s.h_weak_pos.get(), s.h_weak_rec.get(), nw};
    }
    if (s.feat.carrier) {
        CK(ctx, ensure_spare(s.h_carrier, n));
        if (n) CK(ctx, cudaMemcpyAsync(s.h_carrier.get(), s.d_carrier.get(), n * sizeof(modes_carrier), cudaMemcpyDeviceToHost, s.stream));
    }
    CK(ctx, cudaMemcpyAsync(s.h_tiles.get(), s.out_tiles, nt * sizeof(modes_tile), cudaMemcpyDeviceToHost, s.stream));
    v = Shard{s.h_records.get(), s.h_tiles.get(), nt, s.buffer_base, s.feat.recover ? s.h_recovered.get() : nullptr, wl,
              s.feat.carrier ? s.h_carrier.get() : nullptr};
    return 0;
}

// Fetch the slot's results to pinned host memory and run the sequential resolve.
double now_ms() {
    timespec t; clock_gettime(CLOCK_MONOTONIC, &t);
    return t.tv_sec * 1e3 + t.tv_nsec * 1e-6;
}

int collect(modes_ctx *ctx, Slot &s) {
    if (!s.busy) return 0;
    s.busy = false;
    uint64_t n = 0;
    const bool dbg = getenv("MODES_DEBUG_TIMING") != nullptr;
    const double t0 = dbg ? now_ms() : 0;
    if (wait_batch(ctx, s, &n)) return -1;
    s.busy = false;                                     // a repeated (overflowed) batch re-arms the flag
    append_levels(ctx, s);                              // copied with the counters: on the host since s.done
    append_spectra(ctx, s);
    const double t1 = dbg ? now_ms() : 0;
    if (ctx->cfg.gpu_resolve) {
        // the verdicts were taken on the device: fetch the deliveries, build the structs
        if (s.h_counts[1] || s.h_counts[0] > s.out_cap) return fail(ctx, "gpu_resolve: candidate capacity exceeded (%u found)", s.h_counts[0]);
        // internal check: the in-order fallback leaves every buffer's cache as the hand-over computes it
        if (s.h_gr_flags[0]) return fail(ctx, "gpu_resolve: internal error: address caches did not settle after the in-order replay");
        if (s.h_gr_flags[1]) return fail(ctx, "gpu_resolve: delivery capacity exceeded (%u messages)", s.h_gr_flags[2]);
        const size_t nd = s.h_gr_flags[2];
        CK(ctx, ensure_spare(s.h_deliveries, nd));
        if (nd) CK(ctx, cudaMemcpyAsync(s.h_deliveries.get(), s.gr_out.get(), nd * sizeof(modes_delivery), cudaMemcpyDeviceToHost, s.stream));
        CK(ctx, wait_stream(s.stream));
        uint64_t st8[8];
        memcpy(st8, s.h_gr_flags.get() + 4, sizeof(st8));
        for (int i = 0; i < 8; i++) ctx->rs.stats[i] += (int64_t)st8[i];
        memcpy(ctx->rs.icao, s.h_gr_flags.get() + 20, sizeof(ctx->rs.icao));    // host copy for the hex door / a later host resolve
        deliver_gpu(s.h_deliveries.get(), nd, s.buffer_base, ctx->out);
        return 0;
    }
    Shard v;
    if (fetch_async(ctx, s, n, v)) return -1;
    CK(ctx, wait_stream(s.stream));
    const double t2 = dbg ? now_ms() : 0;
    ResolveConfig rc{ctx->cfg.fix_errors, ctx->cfg.aggressive, ctx->cfg.check_crc, s.feat.signal ? 1 : 0};
    resolve_candidates(ctx->rs, rc, v, ctx->out, ctx->scratch);
    if (dbg) fprintf(stderr, "[collect] %zu buffers, %llu cands: wait %.3f ms, d2h %.3f ms, resolve %.3f ms (t=%.3f)\n",
                     s.n_buffers, (unsigned long long)n, t1 - t0, t2 - t1, now_ms() - t2, now_ms());
    return 0;
}

// Multi-GPU: wait for the group of batches in slot `parity` (one per GPU), bring their records to
// the host over every GPU's own link at once, and resolve the group exactly, shards in parallel.
int collect_group(modes_ctx *ctx, int parity) {
    const size_t n = ctx->group_n[parity];
    if (!n) return 0;
    ctx->group_n[parity] = 0;
    std::vector<Shard> shards(n);
    bool signal = false;
    for (size_t k = 0; k < n; k++) {
        modes_ctx *g = ctx->gpus[k];
        Slot &s = g->slot[parity];
        CK(ctx, cudaSetDevice(g->cfg.device));
        uint64_t nc = 0;
        s.busy = false;
        if (wait_batch(g, s, &nc)) return fail(ctx, "GPU %d: %s", g->cfg.device, g->err.c_str());
        s.busy = false;
        append_levels(ctx, s);                          // groups and GPUs in stream order
        append_spectra(ctx, s);
        if (fetch_async(g, s, nc, shards[k])) return fail(ctx, "GPU %d: %s", g->cfg.device, g->err.c_str());
        signal = s.feat.signal;
    }
    for (size_t k = 0; k < n; k++) {
        CK(ctx, cudaSetDevice(ctx->gpus[k]->cfg.device));
        CK(ctx, wait_stream(ctx->gpus[k]->slot[parity].stream));
    }
    // the switches are the same on every GPU of a group: all or none of the shards have records
    for (size_t k = 1; k < n; k++)
        if (!shards[k].recovered != !shards[0].recovered || !shards[k].carrier != !shards[0].carrier)
            return fail(ctx, "internal: recovery or carrier records of GPU %d and GPU %d differ", ctx->gpus[0]->cfg.device,
                        ctx->gpus[k]->cfg.device);
    ResolveConfig rc{ctx->cfg.fix_errors, ctx->cfg.aggressive, ctx->cfg.check_crc, signal ? 1 : 0};
    resolve_shards(ctx->rs, rc, shards.data(), n, ctx->out, ctx->scratch);
    return 0;
}

// Where the batches of a run read their input, host memory or (device) the leading context's device memory.
// 2 MHz UC8: the run's whole reference buffers at iq.
// 2.4 MS/s or a 16-bit format (iq == nullptr): the stream's input bytes [hold0, call0) at hold and
// [call0, end) at call; every later byte is no signal, and output samples at or past out_end are the EOF
// buffer's padding.
struct Source {
    const uint8_t *iq = nullptr;
    const uint8_t *carry = nullptr;   // device: the stream's 476 bytes before iq (host: the context's carry)
    bool device = false;              // every pointer is device memory of the context's device
    const uint8_t *hold = nullptr;
    int64_t hold0 = 0;
    const uint8_t *call = nullptr;
    int64_t call0 = 0, end = 0;
    int64_t out_end = INT64_MAX;
};

// The input paths through the hold: any rate but 2 MHz (resampled, K9, or decimated, K11) or a 16-bit
// format (converted, K10; at the other rates converted as the resampling or decimation loads it).
bool held_input(const modes_ctx *ctx) { return ctx->rate->hz != 2000000 || ctx->input_format != input::kUC8; }

// The input samples [batch_in_lo(o0), batch_in_hi(o1)) that the 2 MHz output samples [o0, o1) of a batch
// and its carry block read (at 2 MHz the carry block's 240 samples, so that a 16-bit upload starts on a
// 16-byte boundary).
int64_t batch_in_lo(const modes_ctx *ctx, int64_t o0) { return in_lo(*ctx->rate, o0 - ctx->rate->carry); }
int64_t batch_in_hi(const modes_ctx *ctx, int64_t o1) { return in_hi(*ctx->rate, o1 - 1); }

// Upload the input bytes the slot's batch (nb buffers from s.buffer_base, and the carry before them) reads,
// straight from where they are (a device source: to this GPU's slot, from the leading context's device), and
// make the slot's body and carry block from them on the device.
int stage_held(modes_ctx *ctx, Slot &s, const Source &src, size_t nb) {
    const cudaMemcpyKind kind = src.device ? cudaMemcpyDefault : cudaMemcpyHostToDevice;
    const int bps = input::sample_bytes(ctx->input_format);
    const int64_t o0 = s.buffer_base * (int64_t)kBufSamples;
    const int64_t o1 = o0 + (int64_t)nb * kBufSamples;
    int64_t lo = bps * batch_in_lo(ctx, o0);
    int64_t hi = bps * batch_in_hi(ctx, o1);
    if (lo < 0) lo = 0;
    if (hi > src.end) hi = src.end;
    if (hi < lo) hi = lo;
    if (lo < src.hold0) return fail(ctx, "internal: input history starts at byte %lld, batch reads from %lld",
                                    (long long)src.hold0, (long long)lo);
    CK(ctx, s.d_iq.ensure((size_t)(o1 - o0) * 2));
    CK(ctx, s.d_in.ensure((size_t)(hi - lo) + 16));
    if (lo < src.call0) {
        const int64_t n = (hi < src.call0 ? hi : src.call0) - lo;
        if (n) CK(ctx, cudaMemcpyAsync(s.d_in.get(), src.hold + (lo - src.hold0), (size_t)n, kind, s.stream));
    }
    if (hi > src.call0) {
        const int64_t from = lo > src.call0 ? lo : src.call0;
        CK(ctx, cudaMemcpyAsync(s.d_in.get() + (from - lo), src.call + (from - src.call0), (size_t)(hi - from), kind,
                                s.stream));
    }
    const ResampleJob j{s.d_in.get(), (uint64_t)(hi - lo), lo / bps, o0, (uint64_t)(o1 - o0), src.out_end,
                        s.d_iq.get(), s.d_halo.get()};
    const int shift = ctx->input_format == input::kUC8 ? -1 : ctx->input_shift;
    s.spec_in = j;
    s.spec_shift = shift;
    if (ctx->rate->m) launch_decimate(j, ctx->rate->m, shift, shift::step(ctx->input_offset, ctx->rate->hz), s.stream);
    else if (ctx->input_format == input::kUC8) launch_resample(j, s.stream);
    else if (ctx->rate->hz == 2400000) launch_resample_sc16(j, ctx->input_shift, s.stream);
    else launch_convert_sc16(j, ctx->input_shift, s.stream);
    CK(ctx, cudaGetLastError());
    ctx->launches++;
    return 0;
}

// Queue the run's next nb buffers (from s.buffer_base) on slot s of context g, whose run ctx leads (g is
// ctx itself, or one of its GPUs), and move src past them.
int submit_next(modes_ctx *ctx, modes_ctx *g, Slot &s, Source &src, size_t nb) {
    if (!src.iq) {
        if (stage_held(g, s, src, nb)) return -1;
        return submit(g, s, nullptr, s.d_iq.get(), nb, nullptr, nullptr, 0, nullptr, true);
    }
    // the batch bytes, uploaded to d_iq, are the input: the span of its own buffers
    CK(g, s.d_iq.ensure((size_t)nb * MODES_BUFFER_BYTES));
    s.spec_in = ResampleJob{};
    s.spec_in.in = s.d_iq.get();
    s.spec_in.in_bytes = (uint64_t)nb * MODES_BUFFER_BYTES;
    s.spec_in.in_first = s.buffer_base * (int64_t)kBufSamples;
    s.spec_shift = -1;
    if (src.device) {
        // copied to the slot (its 16-byte alignment is the kernels'), the carry block built beside it: the
        // stream's bytes never pass through the host
        CK(g, cudaMemcpyAsync(s.d_iq.get(), src.iq, (size_t)nb * MODES_BUFFER_BYTES, cudaMemcpyDefault, s.stream));
        CK(g, cudaMemsetAsync(s.d_halo.get(), 127, kHaloAlloc, s.stream));                  // dump1090.c:344 no-signal
        CK(g, cudaMemcpyAsync(s.d_halo.get() + (kHaloBytes - MODES_CARRY_BYTES), src.carry, MODES_CARRY_BYTES,
                              cudaMemcpyDefault, s.stream));
        if (submit(g, s, nullptr, s.d_iq.get(), nb, nullptr, nullptr, 0, nullptr, true)) return -1;
        src.carry = src.iq + nb * MODES_BUFFER_BYTES - MODES_CARRY_BYTES;
    } else {
        if (submit(g, s, src.iq, nullptr, nb, ctx->carry, nullptr, 0, nullptr)) return -1;
        memcpy(ctx->carry, src.iq + nb * MODES_BUFFER_BYTES - MODES_CARRY_BYTES, MODES_CARRY_BYTES);
    }
    src.iq += nb * MODES_BUFFER_BYTES;
    return 0;
}

// Multi-GPU streaming decode: batches of whole buffers dealt round-robin to the GPUs, one group of
// gpus.size() batches in flight per slot parity; group g-1 is resolved while group g uploads and runs.
int run_buffers_multi(modes_ctx *ctx, Source src, size_t n_buffers) {
    size_t max_b = (size_t)(ctx->cfg.max_batch_bytes / MODES_BUFFER_BYTES);
    if (max_b < 1) max_b = 1;
    int cur = 0;
    bool have_prev = false;
    while (n_buffers) {
        size_t k = 0;
        for (; k < ctx->gpus.size() && n_buffers; k++) {
            // an even share of what is left, so that a short call still uses every GPU
            size_t nb = (n_buffers + (ctx->gpus.size() - k) - 1) / (ctx->gpus.size() - k);
            if (nb > max_b) nb = max_b;
            modes_ctx *g = ctx->gpus[k];
            Slot &s = g->slot[cur];
            CK(ctx, cudaSetDevice(g->cfg.device));
            s.buffer_base = ctx->buffers_done;
            if (submit_next(ctx, g, s, src, nb)) return fail(ctx, "GPU %d: %s", g->cfg.device, g->err.c_str());
            ctx->buffers_done += (int64_t)nb;
            n_buffers -= nb;
        }
        ctx->group_n[cur] = k;
        if (have_prev && collect_group(ctx, cur ^ 1)) return -1;
        have_prev = true;
        cur ^= 1;
    }
    if (collect_group(ctx, cur ^ 1)) return -1;
    return cudaSetDevice(ctx->cfg.device) == cudaSuccess ? 0 : fail(ctx, "cudaSetDevice failed");
}

// Decode the next n_buffers whole reference buffers of the stream from src.
int run_buffers(modes_ctx *ctx, Source src, size_t n_buffers) {
    if (!ctx->gpus.empty()) return run_buffers_multi(ctx, src, n_buffers);
    size_t max_b = (size_t)(ctx->cfg.max_batch_bytes / MODES_BUFFER_BYTES);
    if (max_b < 1) max_b = 1;
    int cur = 0;
    constexpr size_t kTaperFloor = 16;                   // buffers (4 MiB)
    while (n_buffers) {
        size_t nb = n_buffers < max_b ? n_buffers : max_b;
        // The last batches of a call halve in size: what remains to be done after the final upload
        // (its kernels, record download and resolve) then belongs to a small batch, not a full one.
        if (n_buffers <= max_b && n_buffers > kTaperFloor) nb = (n_buffers + 1) / 2;
        Slot &s = ctx->slot[cur];
        if (collect(ctx, s)) return -1;                                  // slot may still hold batch b-2
        s.buffer_base = ctx->buffers_done;
        if (submit_next(ctx, ctx, s, src, nb)) return -1;
        ctx->buffers_done += (int64_t)nb;
        n_buffers -= nb;
        cur ^= 1;
        if (collect(ctx, ctx->slot[cur])) return -1;                     // resolve batch b-1 while b runs
    }
    if (collect(ctx, ctx->slot[cur])) return -1;
    if (collect(ctx, ctx->slot[cur ^ 1])) return -1;
    return 0;
}

Source host_buffers(const uint8_t *iq) {
    Source src;
    src.iq = iq;
    return src;
}

Source device_buffers(const uint8_t *iq, const uint8_t *carry) {
    Source src;
    src.iq = iq;
    src.carry = carry;
    src.device = true;
    return src;
}

// A device-fed stream's own copies (pending, carry, hold) are queued on slot 0's stream and waited for
// before anything reads them: a multi-GPU run's first batch reads them from another device's stream.
cudaError_t copy_on_device(modes_ctx *ctx, void *dst, const void *src, size_t n) {
    return n ? cudaMemcpyAsync(dst, src, n, cudaMemcpyDeviceToDevice, ctx->slot[0].stream) : cudaSuccess;
}

// The most the hold can need: the input of one reference buffer and of the carry before it, with the
// filter's reach on both sides where there is a filter (a whole buffer's input would have run).
size_t hold_bytes(const modes_ctx *ctx) {
    const InputRate &r = *ctx->rate;
    const size_t reach = (size_t)r.in * (kBufSamples + r.carry) / r.out + (r.taps > 1 ? 2 * r.taps : 0);
    return (size_t)input::sample_bytes(ctx->input_format) * (reach + 16);
}

// Run every whole buffer whose input (at 2.4 MS/s with the filter's lookahead) has arrived, reading the
// hold and the caller's bytes where they are (run_buffers returns with every copy done), then keep in
// the hold what later batches read, a sample split across calls included.
int process_held(modes_ctx *ctx, const uint8_t *iq, size_t nbytes) {
    const bool dev = ctx->feed == modes_ctx::Feed::device;
    if (dev) for (auto &h : ctx->d_hold) CK(ctx, h.ensure(hold_bytes(ctx)));
    else CK(ctx, ctx->hold.ensure(hold_bytes(ctx)));
    const int64_t call0 = ctx->in_total;
    ctx->in_total += (int64_t)nbytes;
    const int64_t avail = ctx->in_total / input::sample_bytes(ctx->input_format);   // whole input samples
    const int64_t B = kBufSamples;
    int64_t m = ctx->rate->out * avail / ctx->rate->in / B;                    // buffers [0, m) are ready
    while (m > ctx->buffers_done && batch_in_hi(ctx, m * B) > avail) m--;
    while (batch_in_hi(ctx, (m + 1) * B) <= avail) m++;
    if (m > ctx->buffers_done) {
        Source src;
        src.hold = dev ? ctx->d_hold[ctx->hold_cur].get() : ctx->hold.get(); src.hold0 = ctx->hold0;
        src.call = iq; src.call0 = call0; src.end = ctx->in_total;
        src.device = dev;
        if (run_buffers(ctx, src, (size_t)(m - ctx->buffers_done))) return -1;
    }
    int64_t keep = input::sample_bytes(ctx->input_format) * batch_in_lo(ctx, ctx->buffers_done * B);
    if (keep < ctx->hold0) keep = ctx->hold0;
    if ((size_t)(ctx->in_total - keep) > (dev ? ctx->d_hold[0].capacity() : ctx->hold.capacity()))
        return fail(ctx, "internal: input history of %lld bytes", (long long)(ctx->in_total - keep));
    if (dev) {
        // into the other half: what it keeps of the hold, then of the call
        const uint8_t *old = ctx->d_hold[ctx->hold_cur].get();
        uint8_t *h = ctx->d_hold[ctx->hold_cur ^ 1].get();
        if (keep < call0) {
            CK(ctx, copy_on_device(ctx, h, old + (keep - ctx->hold0), (size_t)(call0 - keep)));
            CK(ctx, copy_on_device(ctx, h + (call0 - keep), iq, nbytes));
        } else {
            CK(ctx, copy_on_device(ctx, h, iq + (keep - call0), (size_t)(ctx->in_total - keep)));
        }
        CK(ctx, wait_stream(ctx->slot[0].stream));
        ctx->hold_cur ^= 1;
        ctx->hold0 = keep;
        return 0;
    }
    uint8_t *h = ctx->hold.get();
    if (keep < call0) {
        memmove(h, h + (keep - ctx->hold0), (size_t)(call0 - keep));
        memcpy(h + (call0 - keep), iq, nbytes);
    } else {
        memcpy(h, iq + (keep - call0), (size_t)(ctx->in_total - keep));
    }
    ctx->hold0 = keep;
    return 0;
}

// The end of a held stream: n_in input samples (UC8: ceil(bytes / 2), a trailing odd byte an I whose Q is
// 127; 16-bit: floor(bytes / 4)) make N_out = n_in (2 MHz), ceil(5 n_in / 6) (2.4 MS/s) or ceil(n_in / M)
// (2 M MS/s) output samples;
// the remaining whole buffers and the EOF buffer (127 past N_out) run from the hold, the input 127-padded
// past its end.
int finish_held(modes_ctx *ctx) {
    const int64_t n_in = ctx->input_format == input::kUC8 ? (ctx->in_total + 1) / 2 : ctx->in_total / 4;
    const int64_t n_out = modes::n_out(*ctx->rate, n_in);
    ctx->eof_buffer = n_out / kBufSamples;                                  // its level record counts the real samples only
    ctx->eof_samples = (uint32_t)(n_out % kBufSamples);
    const int64_t last = ctx->eof_buffer + (ctx->cfg.drop_eof_buffer ? 0 : 1);
    if (last <= ctx->buffers_done) return 0;
    Source src;
    src.device = ctx->feed == modes_ctx::Feed::device;
    src.hold = src.device ? ctx->d_hold[ctx->hold_cur].get() : ctx->hold.get(); src.hold0 = ctx->hold0;
    src.call0 = src.end = ctx->in_total;
    src.out_end = n_out;
    return run_buffers(ctx, src, (size_t)(last - ctx->buffers_done));
}

// One switch of the context and of its GPUs' contexts; each batch runs as the switches were at submit.
int set_feature(modes_ctx *ctx, bool Features::*f, int on) {
    if (!ctx) return -1;
    ctx->feat.*f = on != 0;
    for (modes_ctx *g : ctx->gpus) g->feat.*f = on != 0;
    return 0;
}

}  // namespace

// ------------------------------------------------------------------- C ABI

extern "C" {

int modes_abi_version(void) { return MODES_B200_ABI_VERSION; }

void modes_default_config(modes_config *cfg) {
    memset(cfg, 0, sizeof(*cfg));
    cfg->fix_errors = 1;
    cfg->aggressive = 0;
    cfg->check_crc = 1;
    cfg->drop_eof_buffer = 0;
    cfg->device = 0;
    cfg->profile = 0;
    cfg->max_batch_bytes = 64ull << 20;
    cfg->n_gpus = 1;
}

const char *modes_last_error(const modes_ctx *ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }

void modes_destroy(modes_ctx *ctx) {
    if (!ctx) return;
    for (modes_ctx *g : ctx->gpus) modes_destroy(g);
    ctx->gpus.clear();
    cudaSetDevice(ctx->cfg.device);
    if (ctx->own_detect_stream) { wait_stream(ctx->detect.stream); ctx->detect.stream = ctx->own_detect_stream; }
    slot_free(ctx->slot[0]); slot_free(ctx->slot[1]); slot_free(ctx->detect);
    if (ctx->ev_resolved) cudaEventDestroy(ctx->ev_resolved);
    if (ctx->prof_ready) for (auto &trip : ctx->prof_ev) for (auto &e : trip) cudaEventDestroy(e);
    scratch_destroy(ctx->scratch);
    delete ctx;                       // and with it the context's own buffers
}

static int create_impl(modes_ctx *ctx) {
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return fail(nullptr, "no CUDA device available (%s); this library has no CPU path",
                    e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
    if (ctx->cfg.device < 0 || ctx->cfg.device >= ndev) return fail(nullptr, "device %d out of range", ctx->cfg.device);
    CK(nullptr, cudaSetDevice(ctx->cfg.device));
    cudaDeviceProp prop;
    CK(nullptr, cudaGetDeviceProperties(&prop, ctx->cfg.device));
    if (prop.major != 9 || prop.minor != 0)          // sm_90a code runs on compute capability 9.0 only
        return fail(nullptr, "device %d is sm_%d%d; kernels are built for sm_90a only", ctx->cfg.device, prop.major, prop.minor);
    ctx->sm_count = prop.multiProcessorCount;
    ctx->scratch = scratch_create();
    if (!ctx->scratch) return fail(nullptr, "out of memory");

    std::vector<uint16_t> lutn(kNLutEntries);
    uint32_t syn[112], hash[kFixHashSlots];
    build_lutn(lutn.data());
    std::vector<uint16_t> lut_iq(kLutIqEntries);
    build_lut_iq(lut_iq.data());
    build_bit_syndromes(syn);
    if (!build_fix_hash(syn, hash)) return fail(nullptr, "internal: syndrome hash construction failed");
    CK(nullptr, ctx->d_lutn.ensure(kNLutEntries));
    CK(nullptr, ctx->d_lut_iq.ensure(kLutIqEntries));
    CK(nullptr, cudaMemcpy(ctx->d_lut_iq.get(), lut_iq.data(), kLutIqEntries * sizeof(uint16_t), cudaMemcpyHostToDevice));
    CK(nullptr, ctx->d_bit_syn.ensure(112));
    CK(nullptr, ctx->d_fix_hash.ensure(kFixHashSlots));
    CK(nullptr, cudaMemcpy(ctx->d_lutn.get(), lutn.data(), kNLutEntries * sizeof(uint16_t), cudaMemcpyHostToDevice));
    CK(nullptr, cudaMemcpy(ctx->d_bit_syn.get(), syn, sizeof(syn), cudaMemcpyHostToDevice));
    CK(nullptr, cudaMemcpy(ctx->d_fix_hash.get(), hash, sizeof(hash), cudaMemcpyHostToDevice));
    std::vector<uint32_t> pair(kPairHashSlots);
    if (!build_pair_hash(syn, pair.data())) return fail(nullptr, "internal: two-bit syndrome table construction failed");
    CK(nullptr, ctx->d_pair_hash.ensure(pair.size()));
    CK(nullptr, cudaMemcpy(ctx->d_pair_hash.get(), pair.data(), pair.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
    ctx->tab = DeviceTables{ctx->d_lutn.get(), ctx->d_lut_iq.get(), ctx->d_bit_syn.get(), ctx->d_fix_hash.get(),
                            ctx->d_pair_hash.get()};
    CK(nullptr, ctx->pending.ensure(MODES_BUFFER_BYTES));
    if (ctx->cfg.gpu_resolve) {
        if (ctx->cfg.n_gpus > 1) return fail(nullptr, "gpu_resolve and n_gpus > 1 cannot be combined");
        for (auto &c : ctx->d_cache) { CK(nullptr, c.ensure(1024)); CK(nullptr, cudaMemset(c.get(), 0, 4096)); }
        CK(nullptr, cudaEventCreateWithFlags(&ctx->ev_resolved, cudaEventDisableTiming));
    }
    for (Slot *s : {&ctx->slot[0], &ctx->slot[1], &ctx->detect})
        if (slot_init(ctx, *s)) { g_create_error = ctx->err; return -1; }
    return 0;
}

modes_ctx *modes_create(const modes_config *cfg) {
    modes_ctx *ctx = new (std::nothrow) modes_ctx();
    if (!ctx) { g_create_error = "out of memory"; return nullptr; }
    if (cfg) ctx->cfg = *cfg; else modes_default_config(&ctx->cfg);
    if (ctx->cfg.max_batch_bytes == 0) ctx->cfg.max_batch_bytes = 64ull << 20;
    ctx->rs.reset();
    memset(ctx->carry, 127, sizeof(ctx->carry));
    if (create_impl(ctx)) { modes_destroy(ctx); return nullptr; }
    if (ctx->cfg.n_gpus > 1) {
        int ndev = 0;
        cudaGetDeviceCount(&ndev);
        for (int k = 0; k < ctx->cfg.n_gpus; k++) {
            modes_config c = ctx->cfg;
            c.n_gpus = 1;
            c.profile = 0;
            c.device = (ctx->cfg.device + k) % (ndev > 0 ? ndev : 1);   // fewer devices than shards: reuse them round-robin
            modes_ctx *g = modes_create(&c);
            if (!g) { modes_destroy(ctx); return nullptr; }               // g_create_error holds the reason
            ctx->gpus.push_back(g);
        }
        cudaSetDevice(ctx->cfg.device);
    }
    return ctx;
}

int modes_set_signal(modes_ctx *ctx, int on) { return set_feature(ctx, &Features::signal, on); }

int modes_set_arrival(modes_ctx *ctx, int on) { return set_feature(ctx, &Features::arrival, on); }

int modes_set_levels(modes_ctx *ctx, int on) { return set_feature(ctx, &Features::levels, on); }

int modes_set_carrier(modes_ctx *ctx, int on) {
    // the device resolve's 40-byte delivery records have no room for the carrier
    if (ctx && on && ctx->cfg.gpu_resolve) return fail(ctx, "modes_set_carrier: carrier measurement cannot be combined with gpu_resolve");
    return set_feature(ctx, &Features::carrier, on);
}

size_t modes_take_levels(modes_ctx *ctx, modes_level *out, size_t cap) { return ctx ? ctx->level_q.take(out, cap) : 0; }

int modes_set_spectrum(modes_ctx *ctx, int on) { return set_feature(ctx, &Features::spectrum, on); }

size_t modes_take_spectra(modes_ctx *ctx, modes_spectrum *out, size_t cap) { return ctx ? ctx->spectrum_q.take(out, cap) : 0; }

int modes_levels_device(modes_ctx *ctx, const void *d_iq, size_t n_buffers, size_t stride_bytes) {
    if (!ctx) return -1;
    if (!d_iq || !n_buffers) return fail(ctx, "modes_levels_device: empty input");
    if (n_buffers > 0xFFFFFFFFu) return fail(ctx, "modes_levels_device: too many buffers: %zu", n_buffers);
    if (!stride_bytes) stride_bytes = MODES_BUFFER_BYTES;
    if (((reinterpret_cast<uintptr_t>(d_iq) | stride_bytes) & 15) != 0)
        return fail(ctx, "modes_levels_device: buffers must be 16-byte aligned");
    CK(ctx, cudaSetDevice(ctx->cfg.device));
    cudaStream_t st = ctx->detect.stream;
    // a copy into the pinned block may still be queued: wait for it before the block is replaced
    if (!ctx->lv_fetched && ctx->h_lv.capacity() < n_buffers) CK(ctx, wait_stream(st));
    CK(ctx, ctx->d_lv.ensure(n_buffers));
    CK(ctx, ctx->h_lv.ensure(n_buffers));
    launch_levels(static_cast<const uint8_t *>(d_iq), (uint32_t)n_buffers, stride_bytes, ctx->tab, ctx->d_lv.get(), ctx->sm_count, st);
    CK(ctx, cudaGetLastError());
    ctx->launches++;
    CK(ctx, cudaMemcpyAsync(ctx->h_lv.get(), ctx->d_lv.get(), n_buffers * sizeof(modes_level), cudaMemcpyDeviceToHost, st));
    ctx->lv_n = n_buffers;
    ctx->lv_fetched = false;
    return 0;
}

int modes_levels_fetch(modes_ctx *ctx, modes_level *out) {
    if (!ctx) return -1;
    if (!ctx->lv_n) return fail(ctx, "modes_levels_fetch without modes_levels_device");
    if (!out) return fail(ctx, "modes_levels_fetch: no output array");
    CK(ctx, cudaSetDevice(ctx->cfg.device));
    CK(ctx, wait_stream(ctx->detect.stream));
    ctx->lv_fetched = true;
    memcpy(out, ctx->h_lv.get(), ctx->lv_n * sizeof(modes_level));
    return 0;
}

int modes_set_recovery(modes_ctx *ctx, int on) {
    // the device resolve's read-set bookkeeping has no recovery rule
    if (ctx && on && ctx->cfg.gpu_resolve) return fail(ctx, "modes_set_recovery: recovery cannot be combined with gpu_resolve");
    return set_feature(ctx, &Features::recover, on);
}

int modes_get_recovery_stats(const modes_ctx *ctx, modes_recovery_stats *out) {
    if (!ctx || !out) return -1;
    *out = ctx->rs.rstats;
    return 0;
}

int modes_set_weak_preambles(modes_ctx *ctx, int on) {
    if (ctx && on && ctx->cfg.gpu_resolve) return fail(ctx, "modes_set_weak_preambles: recovery cannot be combined with gpu_resolve");
    return set_feature(ctx, &Features::weak, on);
}

int modes_get_weak_recovery_stats(const modes_ctx *ctx, modes_recovery_stats *out) {
    if (!ctx || !out) return -1;
    *out = ctx->rs.wstats;
    return 0;
}

int modes_weak_device(modes_ctx *ctx, void *d_pos, void *d_rec, size_t capacity) {
    return modes::weak_device_strided(ctx, d_pos, d_rec, capacity, 0, 1);
}

}  // extern "C"

int modes::weak_device_strided(modes_ctx *ctx, void *d_pos, void *d_rec, size_t capacity, uint32_t first_buffer,
                               uint32_t buffer_step) {
    if (!ctx) return -1;
    Slot &s = ctx->detect;
    if (!s.batch_iq) return fail(ctx, "modes_weak_device without modes_detect_device");
    if (!buffer_step) return fail(ctx, "modes_weak_device: buffer step 0");
    if ((d_pos == nullptr) != (d_rec == nullptr)) return fail(ctx, "modes_weak_device: give both output arrays or neither");
    if (d_pos && !capacity) return fail(ctx, "modes_weak_device: capacity 0");
    if (((reinterpret_cast<uintptr_t>(d_pos) | reinterpret_cast<uintptr_t>(d_rec)) & 3) != 0)
        return fail(ctx, "modes_weak_device: outputs must be 4-byte aligned");
    CK(ctx, cudaSetDevice(ctx->cfg.device));
    s.feat.weak = true;
    s.weak_pos_ext = static_cast<uint32_t *>(d_pos);
    s.weak_rec_ext = static_cast<modes_recovered *>(d_rec);
    s.weak_ext_cap = !d_pos ? 0 : (capacity > 0xFFFFFFF0ull ? 0xFFFFFFF0u : (uint32_t)capacity);
    s.weak_first = first_buffer; s.weak_step = buffer_step;
    // a batch that wait_batch repeats (after a candidate or weak overflow) runs the passes again (launch_batch)
    BatchView in{static_cast<const uint8_t *>(s.batch_iq), s.d_halo.get(), (uint64_t)s.n_buffers * kBufSamples};
    if (launch_weak(ctx, s, in)) return -1;
    CK(ctx, cudaEventRecord(s.done, s.stream));            // wait_batch sees the weak count too
    return 0;
}

extern "C" {

int modes_weak_fetch(modes_ctx *ctx, uint32_t *t, modes_recovered *rec, uint64_t *n) {
    if (!ctx) return -1;
    Slot &s = ctx->detect;
    if (!s.feat.weak) return fail(ctx, "modes_weak_fetch without modes_weak_device");
    CK(ctx, cudaSetDevice(ctx->cfg.device));
    uint64_t nc = 0;
    if (wait_batch(ctx, s, &nc)) return -1;
    const uint64_t nw = s.h_weak_counters[1];
    if (n) *n = nw;
    if (!s.weak_pos_ext && nw) {
        if (t) CK(ctx, cudaMemcpyAsync(t, s.d_weak_pos.get(), nw * sizeof(uint32_t), cudaMemcpyDeviceToHost, s.stream));
        if (rec) CK(ctx, cudaMemcpyAsync(rec, s.d_weak_rec.get(), nw * sizeof(modes_recovered), cudaMemcpyDeviceToHost, s.stream));
    }
    CK(ctx, wait_stream(s.stream));
    return 0;
}

int modes_recover_device(modes_ctx *ctx, void *d_out, size_t capacity) {
    if (!ctx) return -1;
    Slot &s = ctx->detect;
    if (!s.batch_iq) return fail(ctx, "modes_recover_device without modes_detect_device");
    if (d_out && !capacity) return fail(ctx, "modes_recover_device: capacity 0");
    if ((reinterpret_cast<uintptr_t>(d_out) & 3) != 0) return fail(ctx, "modes_recover_device: output must be 4-byte aligned");
    CK(ctx, cudaSetDevice(ctx->cfg.device));
    s.feat.recover = true;
    s.rec_ext = static_cast<modes_recovered *>(d_out);
    s.rec_ext_cap = capacity > 0xFFFFFFF0ull ? 0xFFFFFFF0u : (uint32_t)capacity;
    // a batch that wait_batch repeats after an overflow runs the pass again (launch_batch)
    BatchView in{static_cast<const uint8_t *>(s.batch_iq), s.d_halo.get(), (uint64_t)s.n_buffers * kBufSamples};
    ScanOutputs so{s.d_cand_v.get(), s.out_cap, s.out_tiles, s.counters()};
    return launch_recovery(ctx, s, in, so);
}

}  // extern "C"

int modes::detect_shard(modes_ctx *ctx, Shard &shard) {
    if (!ctx) return -1;
    Slot &s = ctx->detect;
    if (!s.busy) return fail(ctx, "the batch's records without modes_detect_device");
    CK(ctx, cudaSetDevice(ctx->cfg.device));
    uint64_t n = 0;
    if (wait_batch(ctx, s, &n) || fetch_async(ctx, s, n, shard)) return -1;
    CK(ctx, wait_stream(s.stream));
    return 0;
}

extern "C" {

int modes_recover_fetch(modes_ctx *ctx, modes_recovered *out) {
    if (!ctx) return -1;
    Slot &s = ctx->detect;
    if (!s.feat.recover || s.rec_ext) return fail(ctx, "modes_recover_fetch without modes_recover_device(ctx, NULL, ...)");
    if (!out) return fail(ctx, "modes_recover_fetch: no output array");
    CK(ctx, cudaSetDevice(ctx->cfg.device));
    uint64_t n = 0;
    if (wait_batch(ctx, s, &n)) return -1;
    if (n) CK(ctx, cudaMemcpyAsync(out, s.d_recovered.get(), n * sizeof(modes_recovered), cudaMemcpyDeviceToHost, s.stream));
    CK(ctx, wait_stream(s.stream));
    return 0;
}

int modes_set_sink(modes_ctx *ctx, modes_sink_fn fn, void *user) {
    if (!ctx) return -1;
    ctx->out.sink = fn; ctx->out.user = user;
    return 0;
}

int modes_set_output(modes_ctx *ctx, modes_message *out, size_t capacity) {
    if (!ctx) return -1;
    ctx->out.array = capacity ? out : nullptr;
    ctx->out.capacity = out ? capacity : 0;
    ctx->out.count = 0;
    return 0;
}

size_t modes_output_count(const modes_ctx *ctx) { return ctx ? ctx->out.count : 0; }

int modes_set_stream(modes_ctx *ctx, void *cuda_stream) {
    if (!ctx) return -1;
    if (ctx->detect.busy) wait_stream(ctx->detect.stream);
    if (!ctx->own_detect_stream) ctx->own_detect_stream = ctx->detect.stream;
    ctx->detect.stream = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : ctx->own_detect_stream;
    return 0;
}

int modes_reset(modes_ctx *ctx) {
    if (!ctx) return -1;
    ctx->rs.reset();
    if (ctx->cfg.gpu_resolve) {
        cudaSetDevice(ctx->cfg.device);
        cudaDeviceSynchronize();
        for (auto &c : ctx->d_cache) cudaMemset(c.get(), 0, 4096);
        ctx->resolved_pending = false;
    }
    ctx->pending_len = 0;
    ctx->buffers_done = 0;
    ctx->finished = false;
    ctx->started = false;
    ctx->feed = modes_ctx::Feed::none;
    ctx->in_total = 0;
    ctx->hold0 = 0;
    ctx->level_q.clear();
    ctx->spectrum_q.clear();
    ctx->eof_buffer = -1;
    memset(ctx->carry, 127, sizeof(ctx->carry));
    return 0;
}

int modes_set_input_rate(modes_ctx *ctx, uint32_t hz) {
    if (!ctx) return -1;
    const InputRate *r = find_input_rate(hz);
    if (!r)
        return fail(ctx, "modes_set_input_rate: %u samples/s is not supported (2000000, 2400000, 4000000, 6000000, "
                         "8000000 or 10000000)", hz);
    if (!offset_fits(*r, ctx->input_offset))
        return fail(ctx, "modes_set_input_rate: %u samples/s is not supported with the input offset of %d Hz (at most "
                         "%d Hz); set the offset to 0 first", hz, (int)ctx->input_offset, (int)max_offset(*r));
    if (ctx->started && !ctx->finished)
        return fail(ctx, "modes_set_input_rate: a stream is in progress; call modes_finish or modes_reset first");
    ctx->rate = r;
    for (modes_ctx *g : ctx->gpus) g->rate = r;
    return 0;
}

int modes_set_input_offset(modes_ctx *ctx, int32_t offset_hz) {
    if (!ctx) return -1;
    if (!offset_fits(*ctx->rate, offset_hz))
        return fail(ctx, "modes_set_input_offset: %d Hz is not supported at %u samples/s (at most %d Hz; 4000000 to "
                         "10000000 samples/s take fs / 2 - 1 MHz, the other rates only 0)",
                    (int)offset_hz, ctx->rate->hz, (int)max_offset(*ctx->rate));
    if (ctx->started && !ctx->finished)
        return fail(ctx, "modes_set_input_offset: a stream is in progress; call modes_finish or modes_reset first");
    ctx->input_offset = offset_hz;
    for (modes_ctx *g : ctx->gpus) g->input_offset = offset_hz;
    return 0;
}

int modes_set_input_format(modes_ctx *ctx, uint32_t format, int32_t shift) {
    if (!ctx) return -1;
    if (!input::known(format))
        return fail(ctx, "modes_set_input_format: format %u is not supported (MODES_INPUT_UC8, MODES_INPUT_SC16 or "
                         "MODES_INPUT_SC16Q11)", format);
    if (shift > input::kMaxShift)
        return fail(ctx, "modes_set_input_format: shift %d is not supported (0 to %d, or negative for the format's default)",
                    (int)shift, input::kMaxShift);
    if (format == input::kUC8 && shift > 0)
        return fail(ctx, "modes_set_input_format: shift %d is not supported with UC8 (0, or negative)", (int)shift);
    if (ctx->started && !ctx->finished)
        return fail(ctx, "modes_set_input_format: a stream is in progress; call modes_finish or modes_reset first");
    const int s = shift < 0 ? input::default_shift(format) : (int)shift;
    ctx->input_format = format;
    ctx->input_shift = s;
    for (modes_ctx *g : ctx->gpus) {
        g->input_format = format;
        g->input_shift = s;
    }
    return 0;
}

int modes_process(modes_ctx *ctx, const uint8_t *iq, size_t nbytes) {
    if (!ctx) return -1;
    if (ctx->finished) return fail(ctx, "modes_process after modes_finish; call modes_reset first");
    if (ctx->feed == modes_ctx::Feed::device)
        return fail(ctx, "modes_process: a stream fed from device memory is in progress; call modes_finish or modes_reset first");
    CK(ctx, cudaSetDevice(ctx->cfg.device));
    ctx->started = true;
    ctx->feed = modes_ctx::Feed::host;
    if (held_input(ctx)) return process_held(ctx, iq, nbytes);
    if (ctx->pending_len) {
        size_t take = MODES_BUFFER_BYTES - ctx->pending_len;
        if (take > nbytes) take = nbytes;
        memcpy(ctx->pending.get() + ctx->pending_len, iq, take);
        ctx->pending_len += take; iq += take; nbytes -= take;
        if (ctx->pending_len < MODES_BUFFER_BYTES) return 0;
        if (run_buffers(ctx, host_buffers(ctx->pending.get()), 1)) return -1;
        ctx->pending_len = 0;
    }
    size_t whole = nbytes / MODES_BUFFER_BYTES;
    if (whole && run_buffers(ctx, host_buffers(iq), whole)) return -1;
    iq += whole * MODES_BUFFER_BYTES; nbytes -= whole * MODES_BUFFER_BYTES;
    if (nbytes) { memcpy(ctx->pending.get(), iq, nbytes); ctx->pending_len = nbytes; }
    return 0;
}

int modes_finish(modes_ctx *ctx) {
    if (!ctx) return -1;
    if (ctx->finished) return 0;
    CK(ctx, cudaSetDevice(ctx->cfg.device));
    ctx->finished = true;
    ctx->started = true;
    if (held_input(ctx)) return finish_held(ctx);
    // The read that hits EOF still hands a 127-padded buffer to the decoder (dump1090.c:496-510);
    // whether it is decoded is the reference's race, made a switch here.
    const bool dev = ctx->feed == modes_ctx::Feed::device;
    if (dev) {
        if (modes_device_memset(ctx->d_pending.get() + ctx->pending_len, 127, MODES_BUFFER_BYTES - ctx->pending_len))
            return fail(ctx, "modes_finish: padding the EOF buffer failed: %s", cudaGetErrorString(cudaGetLastError()));
    } else {
        memset(ctx->pending.get() + ctx->pending_len, 127, MODES_BUFFER_BYTES - ctx->pending_len);
    }
    ctx->eof_buffer = ctx->buffers_done;                 // its level record counts the real samples only
    ctx->eof_samples = (uint32_t)((ctx->pending_len + 1) / 2);
    ctx->pending_len = 0;
    if (ctx->cfg.drop_eof_buffer) return 0;
    return run_buffers(ctx, dev ? device_buffers(ctx->d_pending.get(), ctx->d_carry.get()) : host_buffers(ctx->pending.get()), 1);
}

}  // extern "C"

namespace modes {

std::string device_input_refusal(const void *p, int device, const char *owner, const char *host_call) {
    char buf[256];
    cudaPointerAttributes a;
    const cudaError_t e = cudaPointerGetAttributes(&a, p);
    if (e != cudaSuccess) {
        (void)cudaGetLastError();
        snprintf(buf, sizeof buf, "cudaPointerGetAttributes failed: %s", cudaGetErrorString(e));
        return buf;
    }
    const char *what = nullptr;
    switch (a.type) {
    case cudaMemoryTypeDevice:
        if (a.device == device) return std::string();
        snprintf(buf, sizeof buf, "the bytes are in memory of device %d, not of the %s's device %d", a.device, owner, device);
        return buf;
    case cudaMemoryTypeManaged: what = "managed memory"; break;
    case cudaMemoryTypeHost: what = "pinned host memory"; break;
    default: what = "host memory"; break;
    }
    snprintf(buf, sizeof buf, "the bytes are in %s, not in memory of the %s's device %d (use %s)", what, owner, device, host_call);
    return buf;
}

}  // namespace modes

extern "C" {

// modes_process_device's refusal of memory that is not the context's device memory, naming what it is.
static int check_device_input(modes_ctx *ctx, const void *p) {
    const std::string no = modes::device_input_refusal(p, ctx->cfg.device, "context", "modes_process");
    return no.empty() ? 0 : fail(ctx, "modes_process_device: %s", no.c_str());
}

int modes_process_device(modes_ctx *ctx, const void *d_iq, size_t nbytes) {
    if (!ctx) return -1;
    if (ctx->finished) return fail(ctx, "modes_process_device after modes_finish; call modes_reset first");
    if (!d_iq && nbytes) return fail(ctx, "modes_process_device: null pointer with %zu bytes", nbytes);
    if (ctx->feed == modes_ctx::Feed::host)
        return fail(ctx, "modes_process_device: a stream fed from host memory is in progress; call modes_finish or "
                         "modes_reset first");
    CK(ctx, cudaSetDevice(ctx->cfg.device));
    if (d_iq && check_device_input(ctx, d_iq)) return -1;
    const bool first = ctx->feed == modes_ctx::Feed::none;
    ctx->started = true;
    ctx->feed = modes_ctx::Feed::device;
    const uint8_t *iq = static_cast<const uint8_t *>(d_iq);
    if (held_input(ctx)) return process_held(ctx, iq, nbytes);
    CK(ctx, ctx->d_pending.ensure(MODES_BUFFER_BYTES));
    CK(ctx, ctx->d_carry.ensure(MODES_CARRY_BYTES));
    const cudaStream_t st = ctx->slot[0].stream;
    if (first) CK(ctx, cudaMemsetAsync(ctx->d_carry.get(), 127, MODES_CARRY_BYTES, st));
    // as modes_process, with the pending buffer and the carry on the device: the carry of a run's first batch
    // is d_carry or the pending buffer's tail, of every later one the caller's bytes before it
    const uint8_t *carry = ctx->d_carry.get();
    if (ctx->pending_len) {
        size_t take = MODES_BUFFER_BYTES - ctx->pending_len;
        if (take > nbytes) take = nbytes;
        CK(ctx, copy_on_device(ctx, ctx->d_pending.get() + ctx->pending_len, iq, take));
        ctx->pending_len += take; iq += take; nbytes -= take;
        CK(ctx, wait_stream(st));
        if (ctx->pending_len < MODES_BUFFER_BYTES) return 0;
        if (run_buffers(ctx, device_buffers(ctx->d_pending.get(), carry), 1)) return -1;
        carry = ctx->d_pending.get() + MODES_BUFFER_BYTES - MODES_CARRY_BYTES;
        ctx->pending_len = 0;
    } else if (first) {
        CK(ctx, wait_stream(st));
    }
    const size_t whole = nbytes / MODES_BUFFER_BYTES;
    if (whole) {
        if (run_buffers(ctx, device_buffers(iq, carry), whole)) return -1;
        carry = iq + whole * MODES_BUFFER_BYTES - MODES_CARRY_BYTES;
    }
    iq += whole * MODES_BUFFER_BYTES; nbytes -= whole * MODES_BUFFER_BYTES;
    // the next call's carry, then its partial buffer (on one stream: in that order)
    if (carry != ctx->d_carry.get()) CK(ctx, copy_on_device(ctx, ctx->d_carry.get(), carry, MODES_CARRY_BYTES));
    CK(ctx, copy_on_device(ctx, ctx->d_pending.get(), iq, nbytes));
    ctx->pending_len = nbytes;
    CK(ctx, wait_stream(st));
    return 0;
}

int modes_get_stats(const modes_ctx *ctx, modes_stats *out) {
    if (!ctx || !out) return -1;
    memcpy(out->v, ctx->rs.stats, sizeof(out->v));
    return 0;
}

int modes_compute_magnitude(modes_ctx *ctx, const uint8_t *iq, size_t nsamples, uint16_t *mag) {
    if (!ctx) return -1;
    if (!nsamples) return 0;
    CK(ctx, cudaSetDevice(ctx->cfg.device));
    DevBuf<uint8_t> d_iq;
    DevBuf<uint16_t> d_mag;
    cudaStream_t st = ctx->detect.stream;
    cudaError_t e = d_iq.ensure(nsamples * 2);
    if (e == cudaSuccess) e = d_mag.ensure(nsamples);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_iq.get(), iq, nsamples * 2, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) {
        launch_magnitude(d_iq.get(), d_mag.get(), nsamples, ctx->d_lutn.get(), st);
        ctx->launches++;
        e = cudaMemcpyAsync(mag, d_mag.get(), nsamples * 2, cudaMemcpyDeviceToHost, st);
    }
    if (e == cudaSuccess) e = wait_stream(st);
    if (e != cudaSuccess) return fail(ctx, "magnitude kernel failed: %s", cudaGetErrorString(e));
    return 0;
}

int modes_detect_device(modes_ctx *ctx, const void *d_iq, size_t n_buffers, const uint8_t *carry476,
                        void *d_candidates, size_t cand_capacity, void *d_tiles) {
    if (!ctx) return -1;
    if (!d_iq || !n_buffers) return fail(ctx, "modes_detect_device: empty input");
    CK(ctx, cudaSetDevice(ctx->cfg.device));
    uint32_t cap = cand_capacity > 0xFFFFFFF0ull ? 0xFFFFFFF0u : (uint32_t)cand_capacity;
    return submit(ctx, ctx->detect, nullptr, d_iq, n_buffers, carry476,
                  static_cast<modes_candidate *>(d_candidates), cap, static_cast<modes_tile *>(d_tiles));
}

int modes_detect_host(modes_ctx *ctx, const uint8_t *iq, size_t n_buffers, const uint8_t *carry476,
                      void *d_candidates, size_t cand_capacity, void *d_tiles) {
    if (!ctx) return -1;
    if (!iq || !n_buffers) return fail(ctx, "modes_detect_host: empty input");
    CK(ctx, cudaSetDevice(ctx->cfg.device));
    uint32_t cap = cand_capacity > 0xFFFFFFF0ull ? 0xFFFFFFF0u : (uint32_t)cand_capacity;
    return submit(ctx, ctx->detect, iq, nullptr, n_buffers, carry476,
                  static_cast<modes_candidate *>(d_candidates), cap, static_cast<modes_tile *>(d_tiles));
}

int modes_resample_device(modes_ctx *ctx, const void *d_in, size_t in_bytes, int64_t in_first_sample,
                          int64_t first_buffer, size_t n_buffers, int64_t out_end, void *d_out, uint8_t *carry476) {
    return modes_resample_device_at(ctx, 2400000, d_in, in_bytes, in_first_sample, first_buffer, n_buffers, out_end,
                                    d_out, carry476);
}

int modes_resample_device_at(modes_ctx *ctx, uint32_t hz, const void *d_in, size_t in_bytes, int64_t in_first_sample,
                             int64_t first_buffer, size_t n_buffers, int64_t out_end, void *d_out, uint8_t *carry476) {
    return modes_resample_device_shift(ctx, hz, 0, d_in, in_bytes, in_first_sample, first_buffer, n_buffers, out_end,
                                       d_out, carry476);
}

int modes_resample_device_shift(modes_ctx *ctx, uint32_t hz, int32_t offset_hz, const void *d_in, size_t in_bytes,
                                int64_t in_first_sample, int64_t first_buffer, size_t n_buffers, int64_t out_end,
                                void *d_out, uint8_t *carry476) {
    if (!ctx) return -1;
    const InputRate *r = find_input_rate(hz);
    if (!r || hz == 2000000)
        return fail(ctx, "modes_resample_device: %u samples/s is not supported (2400000, 4000000, 6000000, 8000000 or "
                         "10000000)", hz);
    if (!offset_fits(*r, offset_hz))
        return fail(ctx, "modes_resample_device: an input offset of %d Hz is not supported at %u samples/s (at most %d Hz)",
                    (int)offset_hz, hz, (int)max_offset(*r));
    if (!d_out || !n_buffers) return fail(ctx, "modes_resample_device: empty output");
    if (!d_in && in_bytes) return fail(ctx, "modes_resample_device: no input");
    if (first_buffer < 0) return fail(ctx, "modes_resample_device: buffer index %lld", (long long)first_buffer);
    if (((reinterpret_cast<uintptr_t>(d_in) | reinterpret_cast<uintptr_t>(d_out)) & 15) != 0)
        return fail(ctx, "modes_resample_device: input and output must be 16-byte aligned");
    CK(ctx, cudaSetDevice(ctx->cfg.device));
    cudaStream_t st = ctx->detect.stream;
    if (carry476) {
        CK(ctx, ctx->d_rs_halo.ensure(kHaloAlloc));
        CK(ctx, ctx->h_rs_halo.ensure(kHaloAlloc));
    }
    const ResampleJob j{static_cast<const uint8_t *>(d_in), in_bytes, in_first_sample, first_buffer * (int64_t)kBufSamples,
                        (uint64_t)n_buffers * kBufSamples, out_end < 0 ? INT64_MAX : out_end,
                        static_cast<uint8_t *>(d_out), carry476 ? ctx->d_rs_halo.get() : nullptr};
    if (r->m) launch_decimate(j, r->m, -1, shift::step(offset_hz, hz), st);
    else launch_resample(j, st);
    CK(ctx, cudaGetLastError());
    ctx->launches++;
    if (!carry476) return 0;
    CK(ctx, cudaMemcpyAsync(ctx->h_rs_halo.get(), ctx->d_rs_halo.get(), kHaloAlloc, cudaMemcpyDeviceToHost, st));
    CK(ctx, wait_stream(st));
    memcpy(carry476, ctx->h_rs_halo.get() + (kHaloBytes - MODES_CARRY_BYTES), MODES_CARRY_BYTES);
    return 0;
}

int modes_detect_wait(modes_ctx *ctx, uint64_t *n_candidates) {
    if (!ctx) return -1;
    if (!ctx->detect.busy) return fail(ctx, "modes_detect_wait without modes_detect_device");
    uint64_t n = 0;
    if (wait_batch(ctx, ctx->detect, &n)) return -1;
    ctx->last_detect_count = n;
    if (n_candidates) *n_candidates = n;
    return 0;
}

int modes_detect_fetch(modes_ctx *ctx, modes_candidate *candidates, modes_tile *tiles) {
    if (!ctx) return -1;
    Slot &s = ctx->detect;
    if (!s.busy) return fail(ctx, "modes_detect_fetch without modes_detect_device");
    uint64_t n = 0;
    if (wait_batch(ctx, s, &n)) return -1;
    const size_t nt = tiles_for((uint64_t)s.n_buffers * kBufSamples);
    if (n && candidates)
        CK(ctx, cudaMemcpyAsync(candidates, s.out_records, n * sizeof(modes_candidate), cudaMemcpyDeviceToHost, s.stream));
    if (tiles) CK(ctx, cudaMemcpyAsync(tiles, s.out_tiles, nt * sizeof(modes_tile), cudaMemcpyDeviceToHost, s.stream));
    CK(ctx, wait_stream(s.stream));
    return 0;
}

int modes_resolve(modes_ctx *ctx, const modes_candidate *candidates, const modes_tile *tiles, size_t n_tiles,
                  int64_t buffer_base) {
    if (!ctx || !tiles) return -1;
    ResolveConfig rc{ctx->cfg.fix_errors, ctx->cfg.aggressive, ctx->cfg.check_crc, 0};
    resolve_candidates(ctx->rs, rc, Shard{candidates, tiles, n_tiles, buffer_base}, ctx->out, ctx->scratch);
    return 0;
}

struct modes_resolver {
    ResolveState rs; ResolveConfig rc; MessageOut out; ResolveScratch *scratch = nullptr;
    ResolveState tentative;             // end state of the last modes_resolver_run_tentative
    bool has_tentative = false;
};

modes_resolver *modes_resolver_create(const modes_config *cfg) {
    modes_resolver *r = new (std::nothrow) modes_resolver();
    if (!r) return nullptr;
    modes_config c;
    if (cfg) c = *cfg; else modes_default_config(&c);
    r->rc = ResolveConfig{c.fix_errors, c.aggressive, c.check_crc, 1};
    r->rs.reset();
    r->scratch = scratch_create();
    if (!r->scratch) { delete r; return nullptr; }
    return r;
}

void modes_resolver_destroy(modes_resolver *r) { if (r) { scratch_destroy(r->scratch); delete r; } }

int modes_resolver_run(modes_resolver *r, const modes_candidate *candidates, const modes_tile *tiles,
                       size_t n_tiles, int64_t buffer_base, modes_sink_fn sink, void *user) {
    if (!r || !tiles) return -1;
    r->out.sink = sink; r->out.user = user;
    resolve_candidates(r->rs, r->rc, Shard{candidates, tiles, n_tiles, buffer_base}, r->out, r->scratch);
    return 0;
}

int modes_resolver_run_recovered(modes_resolver *r, const modes_candidate *candidates, const modes_recovered *recovered,
                                 const modes_tile *tiles, size_t n_tiles, int64_t buffer_base, modes_sink_fn sink, void *user) {
    if (!r || !tiles) return -1;
    r->out.sink = sink; r->out.user = user;
    resolve_candidates(r->rs, r->rc, Shard{candidates, tiles, n_tiles, buffer_base, recovered}, r->out, r->scratch);
    return 0;
}

int modes_resolver_run_shards_recovered(modes_resolver *r, size_t n_shards, const modes_candidate *const *candidates,
                                        const modes_recovered *const *recovered, const modes_tile *const *tiles,
                                        const size_t *n_tiles, const int64_t *buffer_base, modes_sink_fn sink, void *user) {
    if (!r || (n_shards && (!candidates || !tiles || !n_tiles || !buffer_base))) return -1;
    std::vector<Shard> shards(n_shards);
    for (size_t k = 0; k < n_shards; k++) {
        if (recovered && !recovered[k]) return -1;
        shards[k] = Shard{candidates[k], tiles[k], n_tiles[k], buffer_base[k], recovered ? recovered[k] : nullptr};
    }
    r->out.sink = sink; r->out.user = user;
    resolve_shards(r->rs, r->rc, shards.data(), n_shards, r->out, r->scratch);
    return 0;
}

int modes_resolver_recovery_stats(const modes_resolver *r, modes_recovery_stats *out) {
    if (!r || !out) return -1;
    *out = r->rs.rstats;
    return 0;
}

int modes_resolver_run_weak(modes_resolver *r, const modes_candidate *candidates, const modes_recovered *recovered,
                            const modes_tile *tiles, size_t n_tiles, int64_t buffer_base, const uint32_t *weak_t,
                            const modes_recovered *weak_rec, size_t n_weak, modes_sink_fn sink, void *user) {
    if (!r || !tiles || (n_weak && (!recovered || !weak_t || !weak_rec))) return -1;
    for (size_t k = 1; k < n_weak; k++)
        if (weak_t[k] <= weak_t[k - 1]) return -1;                   // stream order, each position once
    r->out.sink = sink; r->out.user = user;
    resolve_candidates(r->rs, r->rc, Shard{candidates, tiles, n_tiles, buffer_base, recovered, WeakList{weak_t, weak_rec, n_weak}},
                       r->out, r->scratch);
    return 0;
}

int modes_resolver_run_shards_weak(modes_resolver *r, size_t n_shards, const modes_candidate *const *candidates,
                                   const modes_recovered *const *recovered, const modes_tile *const *tiles,
                                   const size_t *n_tiles, const int64_t *buffer_base, const uint32_t *const *weak_t,
                                   const modes_recovered *const *weak_rec, const size_t *n_weak, modes_sink_fn sink,
                                   void *user) {
    if (!r || (n_shards && (!candidates || !tiles || !n_tiles || !buffer_base || !recovered || !weak_t || !weak_rec || !n_weak)))
        return -1;
    std::vector<Shard> shards(n_shards);
    for (size_t k = 0; k < n_shards; k++) {
        if (!recovered[k] || (n_weak[k] && (!weak_t[k] || !weak_rec[k]))) return -1;
        for (size_t i = 1; i < n_weak[k]; i++)
            if (weak_t[k][i] <= weak_t[k][i - 1]) return -1;
        shards[k] = Shard{candidates[k], tiles[k], n_tiles[k], buffer_base[k], recovered[k], WeakList{weak_t[k], weak_rec[k], n_weak[k]}};
    }
    r->out.sink = sink; r->out.user = user;
    resolve_shards(r->rs, r->rc, shards.data(), n_shards, r->out, r->scratch);
    return 0;
}

int modes_resolver_weak_stats(const modes_resolver *r, modes_recovery_stats *out) {
    if (!r || !out) return -1;
    *out = r->rs.wstats;
    return 0;
}

int modes_resolver_run_shards(modes_resolver *r, size_t n_shards, const modes_candidate *const *candidates,
                              const modes_tile *const *tiles, const size_t *n_tiles, const int64_t *buffer_base,
                              modes_sink_fn sink, void *user) {
    if (!r || (n_shards && (!candidates || !tiles || !n_tiles || !buffer_base))) return -1;
    std::vector<Shard> shards(n_shards);
    for (size_t k = 0; k < n_shards; k++) shards[k] = Shard{candidates[k], tiles[k], n_tiles[k], buffer_base[k]};
    r->out.sink = sink; r->out.user = user;
    resolve_shards(r->rs, r->rc, shards.data(), n_shards, r->out, r->scratch);
    return 0;
}

int modes_resolver_get_cache(const modes_resolver *r, uint32_t cache[MODES_ICAO_CACHE_SLOTS]) {
    if (!r || !cache) return -1;
    memcpy(cache, r->has_tentative ? r->tentative.icao : r->rs.icao, sizeof(r->rs.icao));
    return 0;
}

int modes_resolver_set_cache(modes_resolver *r, const uint32_t cache[MODES_ICAO_CACHE_SLOTS]) {
    if (!r) return -1;
    if (cache) memcpy(r->rs.icao, cache, sizeof(r->rs.icao)); else memset(r->rs.icao, 0, sizeof(r->rs.icao));
    r->rs.cur_buffer = -1; r->rs.next_j = 0; r->rs.next_j_recovered = 0;
    r->has_tentative = false;
    return 0;
}

int modes_resolver_tail_cache(const modes_resolver *r, const modes_candidate *candidates, const modes_tile *tiles,
                              size_t n_tiles, int64_t buffer_base, size_t n_tail_tiles, uint32_t cache[MODES_ICAO_CACHE_SLOTS]) {
    if (!r || !tiles || !cache) return -1;
    ResolveState st;
    st.reset();
    ResolveScratch *tmp = scratch_create();
    if (!tmp) return -1;
    if (n_tail_tiles > n_tiles) n_tail_tiles = n_tiles;
    resolve_tentative(st, r->rc, Shard{candidates, tiles + (n_tiles - n_tail_tiles), n_tail_tiles, buffer_base}, tmp);
    scratch_destroy(tmp);
    memcpy(cache, st.icao, sizeof(st.icao));
    return 0;
}

int modes_resolver_run_tentative(modes_resolver *r, const modes_candidate *candidates, const modes_tile *tiles,
                                 size_t n_tiles, int64_t buffer_base) {
    if (!r || !tiles) return -1;
    r->tentative.start_part(r->rs, true);
    resolve_tentative(r->tentative, r->rc, Shard{candidates, tiles, n_tiles, buffer_base}, r->scratch);
    r->has_tentative = true;
    return 0;
}

int modes_resolver_commit(modes_resolver *r, modes_sink_fn sink, void *user) {
    if (!r || !r->has_tentative) return -1;
    r->out.sink = sink; r->out.user = user;
    r->rs.fold_part(r->tentative);
    r->rs.cur_buffer = r->tentative.cur_buffer; r->rs.next_j = r->tentative.next_j;
    r->rs.next_j_recovered = r->tentative.next_j_recovered;
    resolve_commit(r->out, r->scratch);
    r->has_tentative = false;
    return 0;
}

int modes_resolver_set_output(modes_resolver *r, modes_message *out, size_t capacity) {
    if (!r) return -1;
    r->out.array = capacity ? out : nullptr;
    r->out.capacity = out ? capacity : 0;
    r->out.count = 0;
    return 0;
}

size_t modes_resolver_output_count(const modes_resolver *r) { return r ? r->out.count : 0; }

int modes_resolver_reset(modes_resolver *r) {
    if (!r) return -1;
    r->rs.reset();
    return 0;
}

int modes_resolver_stats(const modes_resolver *r, modes_stats *out) {
    if (!r || !out) return -1;
    memcpy(out->v, r->rs.stats, sizeof(out->v));
    return 0;
}

int modes_decode_frames(modes_ctx *ctx, const uint8_t *frames, size_t n, modes_message *out) {
    if (!ctx || (n && (!frames || !out))) return -1;
    if (!n) return 0;
    if (n > 0x7fffffffu) return fail(ctx, "too many frames");
    CK(ctx, cudaSetDevice(ctx->cfg.device));
    // persistent device / pinned staging, grown on demand (the hex door is called per line by a
    // network feeder: no allocation per call)
    if (ctx->h_frame_evals.capacity() < n) {
        const size_t cap = n < 64 ? 64 : n + n / 2;
        CK(ctx, ctx->d_frames.ensure(cap * 14));
        CK(ctx, ctx->d_frame_evals.ensure(cap));
        CK(ctx, ctx->h_frame_evals.ensure(cap));
    }
    cudaStream_t st = ctx->detect.stream;
    CK(ctx, cudaMemcpyAsync(ctx->d_frames.get(), frames, n * 14, cudaMemcpyHostToDevice, st));
    launch_eval_frames(ctx->d_frames.get(), ctx->d_frame_evals.get(), (uint32_t)n, ctx->tab, ctx->cfg.fix_errors,
                       ctx->cfg.aggressive, st);
    ctx->launches++;
    CK(ctx, cudaMemcpyAsync(ctx->h_frame_evals.get(), ctx->d_frame_evals.get(), n * sizeof(modes_frame_eval),
                            cudaMemcpyDeviceToHost, st));
    CK(ctx, wait_stream(st));
    for (size_t i = 0; i < n; i++) {                       // in order: the address cache is sequential
        finish_message(ctx->rs, ctx->h_frame_evals[i], &out[i]);
        out[i].sample_pos = -1;
    }
    if (ctx->cfg.gpu_resolve) {
        // The device resolve reads the next batch's cache from d_cache[cache_cur], not from rs.icao: hand
        // the frames' writes over.  No batch is in flight here (run_buffers collects both slots before
        // modes_process / modes_finish return), so nothing else reads or writes the device cache.  Queued
        // on the detect stream and waited for: the slot streams are non-blocking, so a copy on the legacy
        // default stream would not be ordered before their next batch.
        CK(ctx, cudaMemcpyAsync(ctx->d_cache[ctx->cache_cur].get(), ctx->rs.icao, sizeof(ctx->rs.icao), cudaMemcpyHostToDevice, st));
        CK(ctx, wait_stream(st));
    }
    return 0;
}

int modes_decode_frame(modes_ctx *ctx, const uint8_t msg[14], modes_message *out) {
    return modes_decode_frames(ctx, msg, 1, out);
}

void *modes_stream(modes_ctx *ctx) { return ctx ? (void *)ctx->detect.stream : nullptr; }

void *modes_device_alloc(size_t nbytes) {
    void *p = nullptr;
    if (cudaMalloc(&p, nbytes ? nbytes : 1) != cudaSuccess) return nullptr;
    return p;
}

void modes_device_free(void *p) { if (p) cudaFree(p); }

int modes_ipc_export(const void *dptr, uint8_t handle[64]) {
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handle size");
    cudaIpcMemHandle_t h;
    if (!dptr || cudaIpcGetMemHandle(&h, const_cast<void *>(dptr)) != cudaSuccess) return -1;
    memcpy(handle, &h, 64);
    return 0;
}

void *modes_ipc_open(const uint8_t handle[64]) {
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, 64);
    void *p = nullptr;
    if (cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return p;
}

int modes_ipc_close(void *mapped) { return mapped && cudaIpcCloseMemHandle(mapped) == cudaSuccess ? 0 : -1; }

int modes_copy_to_host(void *dst_host, const void *src_device, size_t nbytes) {
    // own non-blocking stream per calling thread: never serialises with the caller's other streams
    static thread_local cudaStream_t st = nullptr;
    static thread_local int st_dev = -1;
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, src_device) != cudaSuccess) return -1;
    if (cudaSetDevice(at.device) != cudaSuccess) return -1;
    if (!st || st_dev != at.device) {
        if (cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) != cudaSuccess) return -1;
        st_dev = at.device;
    }
    if (cudaMemcpyAsync(dst_host, src_device, nbytes, cudaMemcpyDeviceToHost, st) != cudaSuccess) return -1;
    return wait_stream(st) == cudaSuccess ? 0 : -1;
}

int modes_set_host_wait(int mode) {
    if (mode != 0 && mode != 1) return -1;
    g_host_wait.store(mode, std::memory_order_relaxed);
    return 0;
}

int modes_device_memset(void *dst_device, int value, size_t nbytes) {
    if (cudaMemset(dst_device, value, nbytes) != cudaSuccess) return -1;
    return cudaDeviceSynchronize() == cudaSuccess ? 0 : -1;
}

int modes_detect_publish_count(modes_ctx *ctx, void *dst) {
    if (!ctx || !dst) return -1;
    CK(ctx, cudaMemcpyAsync(dst, ctx->detect.counters(), 4 * sizeof(uint32_t), cudaMemcpyDeviceToDevice, ctx->detect.stream));
    return 0;
}

void *modes_host_alloc(size_t nbytes) {
    void *p = nullptr;
    if (cudaMallocHost(&p, nbytes ? nbytes : 1) != cudaSuccess) return nullptr;
    return p;
}

void modes_host_free(void *p) { if (p) cudaFreeHost(p); }

int modes_get_kernel_times(modes_ctx *ctx, float ms[4]) {
    if (!ctx || !ms) return -1;
    ms[0] = ms[1] = ms[2] = ms[3] = 0.f;
    if (!ctx->prof_ready) return 0;
    double a = 0, b = 0, c = 0; int n = 0;
    for (; ctx->prof_tail < ctx->prof_head; ctx->prof_tail++) {
        cudaEvent_t *pe = ctx->prof_ev[ctx->prof_tail % modes_ctx::kProfRing];
        if (cudaEventSynchronize(pe[2]) != cudaSuccess) continue;
        float x = 0, y = 0, z = 0;
        cudaEventElapsedTime(&x, pe[0], pe[1]); cudaEventElapsedTime(&y, pe[1], pe[2]); cudaEventElapsedTime(&z, pe[0], pe[2]);
        a += x; b += y; c += z; n++;
    }
    if (n) { ms[0] = (float)(a / n); ms[1] = (float)(b / n); ms[2] = (float)(c / n); ms[3] = (float)n; }
    return 0;
}

uint64_t modes_launch_count(const modes_ctx *ctx) {
    if (!ctx) return 0;
    uint64_t n = ctx->launches;
    for (const modes_ctx *g : ctx->gpus) n += g->launches;
    return n;
}

size_t modes_tile_count(size_t n_buffers) { return tiles_for((uint64_t)n_buffers * kBufSamples); }

}  // extern "C"
