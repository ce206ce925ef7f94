// modes_pool.cpp — many receivers on one GPU: "batch across receivers instead of across time"
// (SURVEY.md §8(f) item 4).
//
// One dump1090 process serves one RTL-SDR: rtlsdrCallback (dump1090.c:442-456) hands it 131072
// samples at a time, each buffer is prefixed with the last 238 samples of the previous one (:481),
// and detectModeS keeps its ICAO address cache, skip state and statistics for that one stream.
// A GPU decodes far more than one such 2 MHz stream in real time (the limit is the PCIe link), but a single
// stream only fills it with seconds of data at a time.  The pool takes ONE buffer from each of many
// receivers and decodes them in one batch, with everything per stream kept per receiver.
//
// The kernels are untouched: they see a batch as consecutive buffers of ONE stream, each buffer's
// carry being the tail of the buffer before it.  The batch is therefore laid out as pairs
//     [pad buffer of receiver i: no signal, its last 238 samples = receiver i's carry][receiver i's buffer]
// resident in HBM (twice: two batches may be in flight, one being uploaded and scanned while the one
// before it is resolved); per call only the data buffers and the 476-byte carries cross PCIe.  A position
// of a data buffer never looks beyond that buffer and its 238 carried samples (dump1090.c:1593:
// j < 131070, window j..j+239 of a 131310-sample array), so its candidates are exactly those of the
// receiver's own stream; whatever the scan finds inside the pad buffers is dropped.  The price is a
// second scan over constant buffers (the scan runs at 2 T samples/s; the link delivers 25 G samples/s).
//
// The order-dependent half is the host resolve, one resolve state per receiver: the records of a data
// buffer are judged where they lie in the batch's record array, at that receiver's own stream position
// and with its own address cache.  Built on the public C ABI (modes_detect_device, modes_recover_device,
// modes_levels_device) and three internal calls: the host resolve itself, detect_shard, which brings a
// batch's records to the host with one wait, and weak_device_strided, the weak scan over the data buffers.
//
// A receiver at 2.4 MS/s (modes_pool_set_input_rate) brings 131072 input samples per call, and its 2 MHz
// buffers complete at their own pace (157286.4 input samples each): at most one per call, none in the
// first and in about one call in six after it.  A call that names such a receiver uploads every buffer
// once to a staging area; one launch (K9's pool form) then resamples the buffer each 2.4 MS/s receiver
// completes into its pair (carry into the pad tail, buffer into the data buffer), reading the receiver's
// device-resident input history and the staging area, and moves the 2 MHz receivers' buffers into
// theirs; a second launch appends the call's bytes to each 2.4 MS/s receiver's history.  Only the
// receivers that complete a buffer get a pair, so the scan and every pass after it see 2 MHz bytes only.
//
// A 16-bit receiver (modes_pool_set_input_format) brings 131072 int16 I/Q samples per call, twice a UC8
// buffer's bytes.  Its call also goes the staged way: the 16-bit buffers cross PCIe into a second staging
// area, and one launch ahead of the others (K10's pool form) converts each to its UC8 buffer, straight into
// the pair's data buffer at 2 MHz, into the receiver's slot of the UC8 staging area at 2.4 MS/s.  From there
// on the receiver is a UC8 receiver at its rate; its carry (2 MHz) is converted on the host.
//
// A device-fed call (modes_pool_submit_device) reads the callers' buffers where they are: the conversion
// reads its 16-bit buffers in place, and the resampling and history launches read the 2.4 MS/s UC8
// receivers' buffers in place.  The 2 MHz receivers' carries stay on the device, in ping-pong halves of
// one array: one more launch (gather_pool_kernel), after the conversion, moves each 2 MHz buffer into its
// pair, its receiver's carry into the pad tail (no signal for a stream's first buffer) and the buffer's
// last 476 bytes into the other half.  Only the 16-bit 2.4 MS/s receivers still use a staging area, the
// UC8 one they are converted into.
//
// A finite capture ends with modes_pool_finish: each listed receiver's tail is staged as a whole buffer padded
// with 127 and goes through the same submit path as at most two internal batches (the whole buffer the tail
// completes, then the EOF buffer), with a few memsets that set what lies past the stream's end to no signal.
#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <condition_variable>
#include <cstdlib>
#include <functional>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>
#include <cuda_runtime.h>
#include "modes_b200.h"
#include "modes_internal.h"
#include "modes_input_core.cuh"
#include "modes_resample_core.cuh"
#include "modes_spectrum_core.cuh"

namespace {

constexpr size_t kBuf = MODES_BUFFER_BYTES;
constexpr int64_t kBufSamples = MODES_BUFFER_SAMPLES;
constexpr int64_t kCarrySamples = MODES_CARRY_BYTES / 2;
constexpr uint32_t kRate2M = 2000000, kRate24 = 2400000;
// 2.4 MS/s: the most one half of a receiver's input history holds: the input of one 2 MHz buffer and of
// the carry before it, with the filter's reach and 16-byte alignment (as modes_api.cpp's hold), plus one
// call's bytes.
constexpr size_t kHistBytes = 2 * ((size_t)6 * (kBufSamples + kCarrySamples) / 5 + 2 * modes::resample::kTaps + 16) + kBuf;

struct Receiver {
    modes::ResolveState rs;                    // its address cache, skip state and statistics
    int64_t buffers = 0;                       // buffers of this receiver decoded so far
    int64_t submitted = 0;                     // buffers of this receiver submitted so far (2 MHz buffers)
    uint8_t carry[MODES_CARRY_BYTES];
    modes::LevelQueue levels;
    modes::SpectrumQueue spectra;
    uint32_t rate = kRate2M;                   // modes_pool_set_input_rate
    uint32_t format = modes::input::kUC8;      // modes_pool_set_input_format, the shift resolved
    int shift = 0;
    // 2.4 MS/s: input bytes of the stream so far, and its device input history: stream bytes
    // [hist0, in_total) at hist[cur], hist0 a multiple of 16; the other half is where the next call's
    // history step writes (no launch reads what it writes)
    int64_t in_total = 0, hist0 = 0;
    modes::DevBuf<uint8_t> hist[2];            // kHistBytes each, made on the receiver's first 2.4 MS/s call
    int cur = 0;
    // which memory its stream is fed from (modes_pool_submit or modes_pool_submit_device), fixed by its
    // first call until modes_pool_reset
    enum class Feed : uint8_t { none, host, device } feed = Feed::none;
    bool finished = false;                     // modes_pool_finish ended its stream (until modes_pool_reset)
};

// 2.4 MS/s: what a call of one buffer's bytes does to receiver r: whether it completes the 2 MHz buffer
// r.submitted (its last sample with the filter's lookahead has arrived; never more than one), and
// the first stream byte later buffers read.
struct RatePlan {
    bool completes;
    int64_t keep;
};
RatePlan rate_plan(const Receiver &r) {
    const int64_t avail = (r.in_total + (int64_t)kBuf) / 2;
    RatePlan pl;
    pl.completes = modes::resample::in_hi((r.submitted + 1) * kBufSamples - 1) <= avail;
    const int64_t next = r.submitted + (pl.completes ? 1 : 0);
    int64_t keep = 2 * modes::resample::in_lo(next * kBufSamples - kCarrySamples);
    keep = keep < 0 ? 0 : keep & ~(int64_t)15;
    pl.keep = keep < r.hist0 ? r.hist0 : keep;
    return pl;
}

// A pair of a finish batch (modes_pool_finish): the receiver's tail, staged as a whole buffer padded with 127,
// makes 2 MHz buffer `buffer`.  A 2.4 MS/s receiver's pair is resampled from its history and the staged tail
// (no history step: a finish runs at most two batches, both reading the same history); a 2 MHz one is the
// staged tail itself.  Bytes past real8 of the staged buffer's UC8 bytes (a 16-bit tail's, once converted)
// and past out_real of the pair's data buffer (2.4 MS/s) are set to 127: input past the stream's end and
// output past N_out are no signal, as modes_finish pads them.  buffer < 0: an ordinary buffer of the call.
struct EofPair {
    int64_t buffer = -1;
    size_t real8 = kBuf, out_real = kBuf;
    uint32_t samples = (uint32_t)kBufSamples;  // the real samples of the buffer, for its level record
};

// The job arrays of a slot's resampling and history launches (pinned or device): PoolResampleJob[n], then
// PoolHistoryJob[n], in one allocation, so that one copy uploads both.
template <bool Pinned>
class RateJobs {
public:
    cudaError_t ensure(size_t n) {
        const cudaError_t e = mem_.ensure(n * (sizeof(modes::PoolResampleJob) + sizeof(modes::PoolHistoryJob)));
        if (e == cudaSuccess) n_ = n;
        return e;
    }
    modes::PoolResampleJob *resample() const { return reinterpret_cast<modes::PoolResampleJob *>(mem_.get()); }
    modes::PoolHistoryJob *history() const {
        return reinterpret_cast<modes::PoolHistoryJob *>(mem_.get() + n_ * sizeof(modes::PoolResampleJob));
    }
    size_t bytes() const { return n_ * (sizeof(modes::PoolResampleJob) + sizeof(modes::PoolHistoryJob)); }
private:
    modes::CudaBuf<uint8_t, Pinned> mem_;
    size_t n_ = 0;
};

// A few persistent helper threads: run(n, f) executes f(0..n-1), f(0) on the calling thread.
class Crew {
public:
    explicit Crew(size_t helpers) {
        for (size_t w = 0; w < helpers; w++) threads_.emplace_back([this, w] { loop(w + 1); });
    }
    ~Crew() {
        { std::lock_guard<std::mutex> g(m_); stop_ = true; gen_++; }
        cv_.notify_all();
        for (std::thread &t : threads_) t.join();
    }
    size_t size() const { return threads_.size() + 1; }
    void run(size_t n, const std::function<void(size_t)> &f) {
        if (n > size()) n = size();
        { std::lock_guard<std::mutex> g(m_); f_ = &f; n_ = n; pending_ = n ? n - 1 : 0; gen_++; }
        cv_.notify_all();
        if (n) f(0);
        std::unique_lock<std::mutex> g(m_);
        done_.wait(g, [this] { return pending_ == 0; });
        f_ = nullptr;
    }
private:
    void loop(size_t me) {
        uint64_t seen = 0;
        for (;;) {
            const std::function<void(size_t)> *f;
            {
                std::unique_lock<std::mutex> g(m_);
                cv_.wait(g, [&] { return gen_ != seen; });
                seen = gen_;
                if (stop_) return;
                if (me >= n_) continue;
                f = f_;
            }
            (*f)(me);
            { std::lock_guard<std::mutex> g(m_); pending_--; }
            done_.notify_one();
        }
    }
    std::vector<std::thread> threads_;
    std::mutex m_;
    std::condition_variable cv_, done_;
    const std::function<void(size_t)> *f_ = nullptr;
    size_t n_ = 0, pending_ = 0;
    uint64_t gen_ = 0;
    bool stop_ = false;
};

}  // namespace

struct modes_pool {
    modes_config cfg;
    std::vector<Receiver> rx;
    size_t max_batch = 0;
    // signal, arrival and carrier are measured by the slot contexts' own passes and reach them at once;
    // recovery, weak preambles and levels are run by the pool per batch, as they were at submit
    modes::Features feat;
    std::string err;
    // device half (created on the first modes_pool_submit / _ingest): two batches may be in flight, so
    // that one is uploaded and scanned while the one before it is resolved on the host.  Each buffer is
    // made the first time a call needs it and released after the slot context, which drains the stream.
    struct Slot {
        modes_ctx *ctx = nullptr;
        modes::DevBuf<uint8_t> d_batch;        // [2 * max_batch] buffers: pad, data, pad, data, ...
        modes::PinnedBuf<uint8_t> h_carry;     // [max_batch][MODES_CARRY_BYTES]
        std::vector<uint32_t> ids;             // the receivers of the batch in flight
        std::vector<int64_t> buf_index;        // with levels: each one's own index of its buffer
        std::vector<uint32_t> samples;         // with levels: the real samples of each one's buffer
        std::vector<modes_level> level_out;
        modes::Features feat;                  // the switches as they were at submit
        bool busy = false;
        // staged calls (a 2.4 MS/s or a 16-bit receiver): the call's UC8 buffers [max_batch], the jobs of
        // the resampling and history launches (pinned and device), and an event after the launches, which
        // the other slot's next staged call waits for (a receiver in both batches).  A device-fed call
        // records it too, after its gather launch, and waits for it first: its carries are the other slot's.
        modes::DevBuf<uint8_t> d_stage;
        RateJobs<true> h_jobs;
        RateJobs<false> d_jobs;
        cudaEvent_t rate_done = nullptr;
        bool rate_recorded = false;
        // calls that name a 16-bit receiver: their 16-bit buffers [max_batch], and the conversion jobs
        modes::DevBuf<uint8_t> d_stage16;
        modes::PinnedBuf<modes::PoolConvertJob> h_cjobs;
        modes::DevBuf<modes::PoolConvertJob> d_cjobs;
        std::vector<const uint8_t *> iq8, iq16;   // the call's UC8 and 16-bit buffers, each group in call order
        // device-fed calls: the gather jobs of their 2 MHz pairs
        modes::PinnedBuf<modes::PoolGatherJob> h_gjobs;
        modes::DevBuf<modes::PoolGatherJob> d_gjobs;
        // with spectra: one job and one record per pair
        modes::PinnedBuf<modes::PoolSpectrumJob> h_sjobs;
        modes::DevBuf<modes::PoolSpectrumJob> d_sjobs;
        modes::PinnedBuf<modes_spectrum> h_spectra;
        modes::DevBuf<modes_spectrum> d_spectra;
    } slot[2];
    unsigned submitted = 0, collected = 0;     // batches so far: slot = number & 1
    // device-fed 2 MHz receivers' carries: [2][n_receivers][MODES_CARRY_BYTES], made on the first device-fed
    // call; the call of a receiver's buffer k reads half k & 1 and writes half (k + 1) & 1
    modes::DevBuf<uint8_t> d_carries;
    // modes_pool_finish: the listed receivers' tails, each staged as a whole buffer of its format padded with
    // 127 (pinned for host tails, device memory for device tails), made on the first finish
    modes::PinnedBuf<uint8_t> h_tails;
    modes::DevBuf<uint8_t> d_tails;
    // the per-receiver resolve: one block of the receiver list per host thread
    struct Block {
        std::unique_ptr<modes::ResolveScratch, void (*)(modes::ResolveScratch *)> scratch{nullptr, modes::scratch_destroy};
        std::vector<modes_message> msgs;       // the block's messages, receiver by receiver
        std::vector<size_t> counts;            // messages of each receiver of the block
        size_t used = 0, at = 0;               // messages of the block; where they start in the call's sequence
        int64_t failed = -1;
    };
    std::vector<Block> blocks;
    std::unique_ptr<Crew> crew;
    // optional caller-owned output array (modes_pool_set_output)
    modes_message *out = nullptr; uint32_t *out_rx = nullptr; size_t out_cap = 0, out_count = 0;
};

namespace {

int fail(modes_pool *p, const char *fmt, ...) {
    char buf[256];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
    p->err = buf;
    return -1;
}

int check_ids(modes_pool *p, const uint32_t *receivers, size_t n) {
    if (!receivers && n) return fail(p, "no receiver list");
    if (n > p->max_batch) return fail(p, "%zu receivers in one call, the pool was created for %zu", n, p->max_batch);
    for (size_t i = 0; i < n; i++) {
        if (receivers[i] >= p->rx.size()) return fail(p, "receiver %u out of range (%zu receivers)", receivers[i], p->rx.size());
        for (size_t k = 0; k < i; k++)
            if (receivers[k] == receivers[i]) return fail(p, "receiver %u listed twice: one buffer per receiver and call", receivers[i]);
    }
    return 0;
}

// Host threads of the per-receiver resolve: MODES_POOL_THREADS, else 4 (receivers are independent; one
// block of 16 or more receivers per thread).
size_t pool_threads() {
    static const size_t n = [] {
        const char *e = std::getenv("MODES_POOL_THREADS");
        long v = e ? std::strtol(e, nullptr, 10) : 4;
        return (size_t)(v < 1 ? 1 : v > 64 ? 64 : v);
    }();
    return n;
}

// The switches a slot context measures itself.
void share_features(const modes_pool *p, modes_ctx *ctx) {
    modes_set_signal(ctx, p->feat.signal);
    modes_set_arrival(ctx, p->feat.arrival);
    modes_set_carrier(ctx, p->feat.carrier);
}

// One switch of the pool.
int set_feature(modes_pool *p, bool modes::Features::*f, int on) {
    if (!p) return -1;
    p->feat.*f = on != 0;
    for (modes_pool::Slot &sl : p->slot)
        if (sl.ctx) share_features(p, sl.ctx);
    return 0;
}

// A buffer of the pool could not be made: its error is cleared, so that a later call can try again.
int out_of_memory(modes_pool *p) {
    cudaGetLastError();
    return fail(p, "out of memory for %zu receivers per batch", p->max_batch);
}

// The slot contexts that are missing and the batches' buffers, with the pool's device current; the
// carries' pinned staging only for host-fed calls.
int ensure_device(modes_pool *p, bool host_fed) {
    if (cudaSetDevice(p->cfg.device) != cudaSuccess) return fail(p, "cudaSetDevice failed: %s", cudaGetErrorString(cudaGetLastError()));
    modes_config c = p->cfg;
    c.n_gpus = 1; c.gpu_resolve = 0;
    const size_t bytes = 2 * p->max_batch * kBuf;
    for (modes_pool::Slot &sl : p->slot) {
        if (!sl.ctx) {
            sl.ctx = modes_create(&c);
            if (!sl.ctx) return fail(p, "%s", modes_last_error(nullptr));
            share_features(p, sl.ctx);
        }
        if (sl.d_batch.capacity() < bytes) {
            if (sl.d_batch.ensure(bytes)) return out_of_memory(p);
            if (modes_device_memset(sl.d_batch.get(), 127, bytes)) {    // dump1090.c:344 no signal
                sl.d_batch = modes::DevBuf<uint8_t>();                  // made again with its fill by the next call
                return fail(p, "device memset failed");
            }
        }
        if (host_fed && sl.h_carry.ensure(p->max_batch * MODES_CARRY_BYTES)) return out_of_memory(p);
    }
    return 0;
}

// The callers' buffers of `bytes` bytes each to dst + i * pitch.  Buffers at a constant distance of at
// least their size in host memory (one staging block): one strided copy instead of n calls (2-3 us of host
// time each: at 256 receivers more than the copy itself takes).
int upload_buffers(modes_pool *p, cudaStream_t st, const uint8_t *const *iq, size_t n, uint8_t *dst, size_t pitch,
                   size_t bytes) {
    bool strided = n > 1 && iq[1] > iq[0];
    const size_t stride = strided ? (size_t)(iq[1] - iq[0]) : 0;
    for (size_t i = 1; strided && i + 1 < n; i++) strided = iq[i + 1] > iq[i] && (size_t)(iq[i + 1] - iq[i]) == stride;
    if (strided && stride >= bytes && stride < ((size_t)1 << 30)) {
        if (cudaMemcpy2DAsync(dst, pitch, iq[0], stride, bytes, n, cudaMemcpyHostToDevice, st) != cudaSuccess)
            return fail(p, "buffer upload failed: %s", cudaGetErrorString(cudaGetLastError()));
    } else {
        for (size_t i = 0; i < n; i++)
            if (cudaMemcpyAsync(dst + i * pitch, iq[i], bytes, cudaMemcpyHostToDevice, st) != cudaSuccess)
                return fail(p, "buffer upload failed: %s", cudaGetErrorString(cudaGetLastError()));
    }
    return 0;
}

// The carries of the slot's first n pairs, gathered in h_carry, into the tails of their pad buffers.
int upload_carries(modes_pool *p, modes_pool::Slot &sl, cudaStream_t st, size_t n) {
    if (cudaMemcpy2DAsync(sl.d_batch.get() + kBuf - MODES_CARRY_BYTES, 2 * kBuf, sl.h_carry.get(), MODES_CARRY_BYTES,
                          MODES_CARRY_BYTES, n, cudaMemcpyHostToDevice, st) != cudaSuccess)
        return fail(p, "carry upload failed: %s", cudaGetErrorString(cudaGetLastError()));
    return 0;
}

// A pair's spectrum job: receiver buffer `buffer` of a stream at 2 MHz (its bytes, data, in the pair) or 2.4 MS/s
// (read from the history and the call's staging area as the resampling job reads it).
modes::PoolSpectrumJob spectrum_job(const Receiver &r, int64_t buffer, const uint8_t *data, const uint8_t *stage) {
    namespace SP = modes::spectrum;
    if (r.rate == kRate2M)
        return modes::PoolSpectrumJob{nullptr, data, 2 * buffer * kBufSamples, 2 * buffer * kBufSamples, buffer,
                                      buffer * kBufSamples, SP::frames(1, 1, buffer), 0};
    return modes::PoolSpectrumJob{r.hist[r.cur].get(), stage, r.hist0, r.in_total, buffer, SP::first_sample(5, 6, buffer),
                                  SP::frames(5, 6, buffer), 0};
}

// The spectrum launch over the slot's n pairs (their jobs at sl.h_sjobs), the records zeroed first and copied
// back behind it, all on the slot's stream.
int launch_pool_spectra(modes_pool *p, modes_pool::Slot &sl, cudaStream_t st, size_t n) {
    uint32_t most = 0;
    for (size_t i = 0; i < n; i++) most = sl.h_sjobs[i].frames > most ? sl.h_sjobs[i].frames : most;
    if (cudaMemcpyAsync(sl.d_sjobs.get(), sl.h_sjobs.get(), n * sizeof(modes::PoolSpectrumJob), cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemsetAsync(sl.d_spectra.get(), 0, n * sizeof(modes_spectrum), st) != cudaSuccess)
        return fail(p, "spectrum job upload failed: %s", cudaGetErrorString(cudaGetLastError()));
    modes::launch_spectrum_pool(sl.d_sjobs.get(), (uint32_t)n, most, sl.d_spectra.get(), st);
    if (cudaGetLastError() != cudaSuccess ||
        cudaMemcpyAsync(sl.h_spectra.get(), sl.d_spectra.get(), n * sizeof(modes_spectrum), cudaMemcpyDeviceToHost, st) != cudaSuccess)
        return fail(p, "spectrum launch failed: %s", cudaGetErrorString(cudaGetLastError()));
    return 0;
}

// The scan and the passes of the switches over the slot's n pairs, already in place.
int detect_pairs(modes_pool *p, modes_pool::Slot &sl, size_t n) {
    if (modes_detect_device(sl.ctx, sl.d_batch.get(), 2 * n, nullptr, nullptr, 0, nullptr)) return fail(p, "%s", modes_last_error(sl.ctx));
    sl.feat = p->feat;
    sl.feat.weak &= sl.feat.recover;
    if (sl.feat.recover && modes_recover_device(sl.ctx, nullptr, 0)) return fail(p, "%s", modes_last_error(sl.ctx));
    // the data buffers only (every second buffer), like the level pass
    if (sl.feat.weak && modes::weak_device_strided(sl.ctx, nullptr, nullptr, 0, 1, 2)) return fail(p, "%s", modes_last_error(sl.ctx));
    // the data buffers only (every second buffer), on the same stream: no wait before the collect
    if (sl.feat.levels && modes_levels_device(sl.ctx, sl.d_batch.get() + kBuf, n, 2 * kBuf)) return fail(p, "%s", modes_last_error(sl.ctx));
    return 0;
}

// A finish batch's padding: every span set to 127 on the slot's stream.
using Spans = std::vector<std::pair<uint8_t *, size_t>>;
int fill_no_signal(modes_pool *p, const Spans &spans, cudaStream_t st) {
    for (const auto &sp : spans)
        if (cudaMemsetAsync(sp.first, 127, sp.second, st) != cudaSuccess)
            return fail(p, "EOF padding failed: %s", cudaGetErrorString(cudaGetLastError()));
    return 0;
}

}  // namespace

extern "C" {

modes_pool *modes_pool_create(const modes_config *cfg, size_t n_receivers, size_t max_batch_receivers) {
    if (!cfg || !n_receivers) return nullptr;
    modes_pool *p = new modes_pool();
    p->cfg = *cfg;
    p->max_batch = max_batch_receivers && max_batch_receivers < n_receivers ? max_batch_receivers : n_receivers;
    p->rx.resize(n_receivers);
    for (Receiver &r : p->rx) {
        r.rs.reset();
        memset(r.carry, 127, sizeof r.carry);
    }
    return p;
}

void modes_pool_destroy(modes_pool *p) {
    if (!p) return;
    for (modes_pool::Slot &sl : p->slot) {
        if (sl.rate_done) cudaEventDestroy(sl.rate_done);
        if (sl.ctx) modes_destroy(sl.ctx);     // waits for the slot's stream
    }
    delete p;                                  // and with it the buffers, which nothing queued uses any more
}

const char *modes_pool_last_error(const modes_pool *p) { return p ? p->err.c_str() : "no pool"; }

// The per-receiver resolve of a batch of n pairs (its records, recovery records, weak positions and carrier
// records); recovered messages carry their record's signal only when the batch measured signals.
static int pool_resolve(modes_pool *p, const uint32_t *receivers, size_t n, const modes::Shard &batch, bool signal,
                        modes_pool_sink_fn sink, void *user) {
    if (!p) return -1;
    if (check_ids(p, receivers, n)) return -1;
    if (!n) return 0;
    if (!batch.tiles) return fail(p, "no tile table");
    const modes_tile *tiles = batch.tiles;
    const uint32_t *weak_t = batch.weak.t;
    const size_t n_tiles = modes_tile_count(2 * n), n_weak = batch.weak.n;
    const modes::ResolveConfig rc{p->cfg.fix_errors, p->cfg.aggressive, p->cfg.check_crc, signal ? 1 : 0};
    // Receivers are independent: the list is cut into blocks, one host thread each; a block's messages
    // land in its own array and are moved to the caller's array / handed to the sink in list order.
    size_t n_blocks = pool_threads();
    if (n_blocks > (n + 15) / 16) n_blocks = (n + 15) / 16;
    if (n_blocks < 1) n_blocks = 1;
    if (p->blocks.size() < n_blocks) p->blocks.resize(n_blocks);
    auto tile_range = [&](size_t i, size_t &g0, size_t &g1) {
        // the data buffer of pair i is buffer 2i+1 of the batch; a position t belongs to the tile
        // that holds virtual position t + 2
        const int64_t t0 = kBufSamples * (int64_t)(2 * i + 1), t1 = t0 + kBufSamples;
        g0 = (size_t)((t0 + 2) / MODES_TILE_SAMPLES); g1 = (size_t)((t1 + 1) / MODES_TILE_SAMPLES);
        if (g1 >= n_tiles) g1 = n_tiles - 1;
    };
    auto work = [&](size_t b) {
        modes_pool::Block &bl = p->blocks[b];
        const size_t i0 = n * b / n_blocks, i1 = n * (b + 1) / n_blocks;
        bl.failed = -1;
        bl.counts.assign(i1 - i0, 0);
        size_t room = 0, ga, gb, gc, gd;
        tile_range(i0, ga, gb); tile_range(i1 - 1, gc, gd);
        // a candidate delivers at most two messages of the reference (both attempts without --check-crc,
        // dump1090.c:1803) and, with recovery, one recovered message after them; a weak position one
        const size_t per_candidate = batch.recovered ? 3 : 2;
        for (size_t g = ga; g <= gd; g++) room += per_candidate * (size_t)tiles[g].count;
        const uint32_t *wlo = std::lower_bound(weak_t, weak_t + n_weak, (uint32_t)(kBufSamples * (2 * i0 + 1)));
        const uint32_t *whi = std::lower_bound(weak_t, weak_t + n_weak, (uint32_t)(kBufSamples * (2 * i1)));
        room += (size_t)(whi - wlo);
        if (bl.msgs.size() < room) bl.msgs.resize(room);
        if (!bl.scratch) bl.scratch.reset(modes::scratch_create());
        if (!bl.scratch) { bl.failed = (int64_t)i0; return; }
        size_t used = 0;
        for (size_t i = i0; i < i1; i++) {
            Receiver &r = p->rx[receivers[i]];
            // the receiver's data buffer, batch buffer 2i+1, judged in place as its own buffer r.buffers
            modes::Shard s = batch;
            size_t g0, g1;
            tile_range(i, g0, g1);
            s.tiles = tiles + g0;
            s.n_tiles = g1 - g0 + 1;
            s.buffer_base = r.buffers - (int64_t)(2 * i + 1);
            s.b_lo = (uint32_t)(2 * i + 1);
            s.b_hi = s.b_lo + 1;
            modes::MessageOut out;
            out.array = bl.msgs.data() + used;
            out.capacity = room - used;
            modes::resolve_candidates(r.rs, rc, s, out, bl.scratch.get());
            const size_t k = out.count;
            if (k > room - used) { bl.failed = (int64_t)i; return; }   // the bound above is exact: never reached
            bl.counts[i - i0] = k;
            used += k;
            r.buffers++;
        }
        bl.used = used;
    };
    if (!p->crew) p->crew.reset(new Crew(pool_threads() - 1));
    p->crew->run(n_blocks, work);
    for (size_t b = 0; b < n_blocks; b++)
        if (p->blocks[b].failed >= 0) return fail(p, "resolve of receiver %u failed", receivers[p->blocks[b].failed]);
    // in list order into the caller's array (the count keeps running past its capacity): every block
    // moves its own messages
    size_t total = 0;
    for (size_t b = 0; b < n_blocks; b++) { p->blocks[b].at = total; total += p->blocks[b].used; }
    if (p->out) {
        const size_t base = p->out_count, cap = p->out_cap;
        auto move = [&](size_t b) {
            const modes_pool::Block &bl = p->blocks[b];
            const size_t i0 = n * b / n_blocks, first = base + bl.at;
            const size_t fit = first >= cap ? 0 : (bl.used < cap - first ? bl.used : cap - first);
            if (fit) memcpy(p->out + first, bl.msgs.data(), fit * sizeof(modes_message));
            size_t at = 0;
            for (size_t j = 0; j < bl.counts.size(); j++)
                for (size_t m = 0; m < bl.counts[j]; m++, at++)
                    if (at < fit) p->out_rx[first + at] = receivers[i0 + j];
        };
        p->crew->run(n_blocks, move);
        p->out_count += total;
    }
    if (sink)
        for (size_t b = 0; b < n_blocks; b++) {
            const modes_pool::Block &bl = p->blocks[b];
            const size_t i0 = n * b / n_blocks;
            size_t at = 0;
            for (size_t j = 0; j < bl.counts.size(); j++)
                for (size_t m = 0; m < bl.counts[j]; m++, at++) sink(user, receivers[i0 + j], &bl.msgs[at]);
        }
    return 0;
}

int modes_pool_resolve(modes_pool *p, const uint32_t *receivers, size_t n, const modes_candidate *candidates,
                       const modes_tile *tiles, modes_pool_sink_fn sink, void *user) {
    return pool_resolve(p, receivers, n, modes::Shard{candidates, tiles}, false, sink, user);
}

// One buffer of each listed receiver.  A receiver gets a pair when it decodes a buffer in this call: a 2 MHz
// receiver always, a 2.4 MS/s one when the call completes one.  A call that names only 2 MHz UC8 receivers
// uploads its buffers straight into the pairs' data buffers.  Any other call is staged: every UC8 buffer
// goes to the staging area and every 16-bit buffer to the 16-bit one; launches then convert the 16-bit
// buffers (into their pairs at 2 MHz, into the staging area at 2.4 MS/s), resample the completing
// receivers / move the 2 MHz ones into their pairs, and advance the histories.  Staging slots: the UC8
// buffers in call order, then the 16-bit 2.4 MS/s receivers'.
//
// device: the buffers are device memory of cfg.device (modes_pool_submit_device), read in place by the same
// launches, and the 2 MHz pairs are filled by the gather launch; the staging area holds only the 16-bit
// 2.4 MS/s receivers' converted bytes.
//
// eof (modes_pool_finish's batches, else nullptr): per listed receiver, the pair its staged tail makes.
static int submit(modes_pool *p, const uint32_t *receivers, const uint8_t *const *iq, size_t n, bool device,
                  const EofPair *eof = nullptr) {
    namespace input = modes::input;
    using Feed = Receiver::Feed;
    if (!p) return -1;
    if (check_ids(p, receivers, n)) return -1;
    if (!n) return fail(p, "an empty batch");
    if (!iq) return fail(p, "no buffers");
    if (device)
        for (size_t i = 0; i < n; i++) {
            if (!iq[i]) return fail(p, "modes_pool_submit_device: receiver %u: null pointer", receivers[i]);
            if (reinterpret_cast<uintptr_t>(iq[i]) & 15)
                return fail(p, "modes_pool_submit_device: receiver %u: the buffer at %p is not 16-byte aligned", receivers[i],
                            static_cast<const void *>(iq[i]));
            const std::string no = modes::device_input_refusal(iq[i], p->cfg.device, "pool", "modes_pool_submit");
            if (!no.empty()) return fail(p, "modes_pool_submit_device: receiver %u: %s", receivers[i], no.c_str());
        }
    const char *call = device ? "modes_pool_submit_device" : "modes_pool_submit";
    for (size_t i = 0; i < n; i++)
        if (p->rx[receivers[i]].finished)
            return fail(p, "%s: receiver %u after modes_pool_finish; call modes_pool_reset first", call, receivers[i]);
    for (size_t i = 0; i < n; i++)
        if (p->rx[receivers[i]].feed == (device ? Feed::host : Feed::device))
            return fail(p, "%s: receiver %u has a stream fed from %s memory in progress; call modes_pool_reset first",
                        call, receivers[i], device ? "host" : "device");
    if (ensure_device(p, !device)) return -1;
    modes_pool::Slot &sl = p->slot[p->submitted & 1];
    if (sl.busy) return fail(p, "two batches are in flight: modes_pool_collect first");
    bool staged = false, wide = false, two_mhz = false, rated = false, wide24 = false;
    for (size_t i = 0; i < n; i++) {
        if (!iq[i]) return fail(p, "receiver %u: no buffer", receivers[i]);
        const Receiver &r = p->rx[receivers[i]];
        wide |= r.format != input::kUC8;
        staged |= wide || r.rate != kRate2M;
        two_mhz |= r.rate == kRate2M;
        rated |= r.rate != kRate2M;
        wide24 |= r.format != input::kUC8 && r.rate != kRate2M;
    }
    if (device) staged = false;                // a device-fed call stages only wide24's conversions
    const size_t mb = p->max_batch;
    const bool spectra = p->feat.spectrum;
    if (staged && (sl.d_stage.ensure(mb * kBuf) || sl.h_jobs.ensure(mb) || sl.d_jobs.ensure(mb))) return out_of_memory(p);
    if (wide && !device && (sl.d_stage16.ensure(mb * 2 * kBuf) || sl.h_cjobs.ensure(mb) || sl.d_cjobs.ensure(mb)))
        return out_of_memory(p);
    if (device) {
        if ((two_mhz && (p->d_carries.ensure(2 * p->rx.size() * MODES_CARRY_BYTES) || sl.h_gjobs.ensure(mb) || sl.d_gjobs.ensure(mb))) ||
            (rated && (sl.h_jobs.ensure(mb) || sl.d_jobs.ensure(mb))) || (wide24 && sl.d_stage.ensure(mb * kBuf)) ||
            (wide && (sl.h_cjobs.ensure(mb) || sl.d_cjobs.ensure(mb))))
            return out_of_memory(p);
    }
    if (spectra && (sl.h_sjobs.ensure(mb) || sl.d_sjobs.ensure(mb) || sl.h_spectra.ensure(mb) || sl.d_spectra.ensure(mb)))
        return out_of_memory(p);
    if ((staged || device) && !sl.rate_done && cudaEventCreateWithFlags(&sl.rate_done, cudaEventDisableTiming) != cudaSuccess)
        return fail(p, "event creation failed: %s", cudaGetErrorString(cudaGetLastError()));

    modes::PoolResampleJob *rj = sl.h_jobs.resample();
    modes::PoolHistoryJob *hj = sl.h_jobs.history();
    // a device-fed receiver's carry: half k & 1 holds what its buffer k - 1 left
    auto device_carry = [p](uint32_t id, int64_t k) {
        return p->d_carries.get() + ((size_t)(k & 1) * p->rx.size() + id) * MODES_CARRY_BYTES;
    };
    size_t n_pairs = 0, n_rj = 0, n_hist = 0, n_conv = 0, n_gather = 0;
    uint64_t hist_max = 0;
    bool carries = false;
    Spans fill_in, fill_out;                   // a finish batch's padding after the conversion / the resampling
    sl.iq8.clear();
    sl.iq16.clear();
    if (!device)
        for (size_t i = 0; i < n; i++) (p->rx[receivers[i]].format == input::kUC8 ? sl.iq8 : sl.iq16).push_back(iq[i]);
    size_t n_stage = sl.iq8.size();
    sl.ids.clear();
    sl.buf_index.clear();
    sl.samples.clear();
    for (size_t i = 0, k8 = 0; i < n; i++) {
        Receiver &r = p->rx[receivers[i]];
        const bool uc8 = r.format == input::kUC8;
        const EofPair *e = eof && eof[i].buffer >= 0 ? &eof[i] : nullptr;
        const int64_t buffer = e ? e->buffer : r.submitted;   // the 2 MHz buffer of its pair, if it gets one
        uint8_t *data = sl.d_batch.get() + (2 * n_pairs + 1) * kBuf;    // the data buffer of its pair, if it gets one
        // staged: where its call's UC8 bytes are staged (none for a 16-bit 2 MHz receiver, converted into its pair);
        // device-fed: only a 16-bit 2.4 MS/s receiver's
        const bool staging = device ? !uc8 && r.rate != kRate2M : staged && (uc8 || r.rate != kRate2M);
        uint8_t *stage = staging ? sl.d_stage.get() + (uc8 ? k8++ : n_stage++) * kBuf : nullptr;
        // the UC8 bytes the resampling reads: a device-fed UC8 receiver's own buffer
        const uint8_t *in8 = device && uc8 ? iq[i] : stage;
        if (!uc8) {
            const uint8_t *in16 = device ? iq[i] : sl.d_stage16.get() + n_conv * 2 * kBuf;
            sl.h_cjobs[n_conv] = modes::PoolConvertJob{in16, stage ? stage : data, r.shift};
            n_conv++;
            if (e && e->real8 < kBuf) fill_in.emplace_back((stage ? stage : data) + e->real8, kBuf - e->real8);
        }
        bool pair = true;
        if (r.rate == kRate2M && device) {
            sl.h_gjobs[n_gather++] = modes::PoolGatherJob{uc8 ? iq[i] : nullptr, data,
                                                          r.submitted ? device_carry(receivers[i], r.submitted) : nullptr,
                                                          device_carry(receivers[i], r.submitted + 1), data - MODES_CARRY_BYTES};
        } else if (r.rate == kRate2M) {
            memcpy(sl.h_carry.get() + n_pairs * MODES_CARRY_BYTES, r.carry, MODES_CARRY_BYTES);
            carries = true;
            if (stage) rj[n_rj++] = modes::PoolResampleJob{nullptr, stage, 0, 0, -1, nullptr, data};
        } else {
            for (modes::DevBuf<uint8_t> &h : r.hist)
                if (h.ensure(kHistBytes)) {
                    cudaGetLastError();
                    return fail(p, "out of memory for the input history of receiver %u", receivers[i]);
                }
            // a finish batch's pair reads the history as it is and leaves it so: no history step
            const RatePlan pl = e ? RatePlan{true, r.hist0} : rate_plan(r);
            pair = pl.completes;
            if (pair)
                rj[n_rj++] = modes::PoolResampleJob{r.hist[r.cur].get(), in8, r.hist0, r.in_total, buffer * kBufSamples,
                                                    data - MODES_CARRY_BYTES, data};
            if (e && e->out_real < kBuf) fill_out.emplace_back(data + e->out_real, kBuf - e->out_real);
            if (!e) {
                const uint64_t bytes = (uint64_t)(r.in_total + (int64_t)kBuf - pl.keep);
                if (bytes > kHistBytes)
                    return fail(p, "internal: 2.4 MS/s input history of %llu bytes for receiver %u", (unsigned long long)bytes, receivers[i]);
                hj[n_hist++] = modes::PoolHistoryJob{r.hist[r.cur].get(), in8, r.hist0, r.in_total, pl.keep, r.hist[r.cur ^ 1].get()};
                if (bytes > hist_max) hist_max = bytes;
            }
        }
        if (!pair) continue;
        if (spectra) sl.h_sjobs[n_pairs] = spectrum_job(r, buffer, data, in8);
        n_pairs++;
        sl.ids.push_back(receivers[i]);
        sl.buf_index.push_back(buffer);
        sl.samples.push_back(e ? e->samples : (uint32_t)kBufSamples);
    }

    cudaStream_t st = static_cast<cudaStream_t>(modes_stream(sl.ctx));
    const modes_pool::Slot &other = p->slot[(p->submitted & 1) ^ 1];
    if (device) {
        if ((n_gather && cudaMemcpyAsync(sl.d_gjobs.get(), sl.h_gjobs.get(), n_gather * sizeof(modes::PoolGatherJob),
                                         cudaMemcpyHostToDevice, st) != cudaSuccess) ||
            (rated && cudaMemcpyAsync(sl.d_jobs.resample(), rj, sl.h_jobs.bytes(), cudaMemcpyHostToDevice, st) != cudaSuccess) ||
            (n_conv && cudaMemcpyAsync(sl.d_cjobs.get(), sl.h_cjobs.get(), n_conv * sizeof(modes::PoolConvertJob),
                                       cudaMemcpyHostToDevice, st) != cudaSuccess))
            return fail(p, "job upload failed: %s", cudaGetErrorString(cudaGetLastError()));
        modes::launch_convert_pool(sl.d_cjobs.get(), (uint32_t)n_conv, st);
        if (fill_no_signal(p, fill_in, st)) return -1;
        // the other batch in flight may name the same receivers: its carries, reads and history step first
        if (other.rate_recorded && cudaStreamWaitEvent(st, other.rate_done, 0) != cudaSuccess)
            return fail(p, "stream wait failed: %s", cudaGetErrorString(cudaGetLastError()));
        modes::launch_gather_pool(sl.d_gjobs.get(), (uint32_t)n_gather, st);
        modes::launch_resample_pool(sl.d_jobs.resample(), (uint32_t)n_rj, st);
        if (fill_no_signal(p, fill_out, st)) return -1;
        modes::launch_history_pool(sl.d_jobs.history(), (uint32_t)n_hist, hist_max, st);
    } else if (!staged) {
        if (upload_carries(p, sl, st, n_pairs) || upload_buffers(p, st, iq, n, sl.d_batch.get() + kBuf, 2 * kBuf, kBuf)) return -1;
    } else {
        if (!sl.iq8.empty() && upload_buffers(p, st, sl.iq8.data(), sl.iq8.size(), sl.d_stage.get(), kBuf, kBuf)) return -1;
        if (!sl.iq16.empty() && upload_buffers(p, st, sl.iq16.data(), sl.iq16.size(), sl.d_stage16.get(), 2 * kBuf, 2 * kBuf))
            return -1;
        // the 2.4 MS/s pairs' tails are then overwritten by the resampler
        if (carries && upload_carries(p, sl, st, n_pairs)) return -1;
        if (cudaMemcpyAsync(sl.d_jobs.resample(), rj, sl.h_jobs.bytes(), cudaMemcpyHostToDevice, st) != cudaSuccess ||
            (n_conv && cudaMemcpyAsync(sl.d_cjobs.get(), sl.h_cjobs.get(), n_conv * sizeof(modes::PoolConvertJob),
                                       cudaMemcpyHostToDevice, st) != cudaSuccess))
            return fail(p, "job upload failed: %s", cudaGetErrorString(cudaGetLastError()));
        // the conversion writes only this slot's pairs and staging area: it need not wait for the other slot
        modes::launch_convert_pool(sl.d_cjobs.get(), (uint32_t)n_conv, st);
        if (fill_no_signal(p, fill_in, st)) return -1;
        // the other batch in flight may name the same receivers: its reads and its history step first
        if (other.rate_recorded && cudaStreamWaitEvent(st, other.rate_done, 0) != cudaSuccess)
            return fail(p, "stream wait failed: %s", cudaGetErrorString(cudaGetLastError()));
        modes::launch_resample_pool(sl.d_jobs.resample(), (uint32_t)n_rj, st);
        if (fill_no_signal(p, fill_out, st)) return -1;
        modes::launch_history_pool(sl.d_jobs.history(), (uint32_t)n_hist, hist_max, st);
    }
    // the spectra read the histories too: before rate_done, after which the other slot's history step may
    // overwrite them
    if (spectra && n_pairs && launch_pool_spectra(p, sl, st, n_pairs)) return -1;
    if (staged || device) {
        if (cudaGetLastError() != cudaSuccess || cudaEventRecord(sl.rate_done, st) != cudaSuccess)
            return fail(p, "resampling launch failed: %s", cudaGetErrorString(cudaGetLastError()));
        sl.rate_recorded = true;
    }
    if (n_pairs && detect_pairs(p, sl, n_pairs)) return -1;

    for (size_t i = 0; i < n; i++) {
        Receiver &r = p->rx[receivers[i]];
        r.feed = device ? Feed::device : Feed::host;
        if (eof && eof[i].buffer >= 0) {       // a finish batch: the stream ends after it
            r.submitted = eof[i].buffer + 1;
            continue;
        }
        if (r.rate == kRate2M) {
            r.submitted++;
            if (device) continue;              // its carry is on the device
            // what it carries into its next buffer (dump1090.c:481)
            if (r.format == input::kUC8) memcpy(r.carry, iq[i] + kBuf - MODES_CARRY_BYTES, MODES_CARRY_BYTES);
            else input::convert_samples(iq[i] + 2 * (kBuf - MODES_CARRY_BYTES), MODES_CARRY_BYTES / 2, r.shift, r.carry);
            continue;
        }
        const RatePlan pl = rate_plan(r);
        r.submitted += pl.completes ? 1 : 0;
        r.in_total += (int64_t)kBuf;
        r.hist0 = pl.keep;
        r.cur ^= 1;
    }
    sl.busy = true;
    p->submitted++;
    return 0;
}

int modes_pool_submit(modes_pool *p, const uint32_t *receivers, const uint8_t *const *iq, size_t n) {
    return submit(p, receivers, iq, n, false);
}

int modes_pool_submit_device(modes_pool *p, const uint32_t *receivers, const void *const *d_iq, size_t n) {
    return submit(p, receivers, reinterpret_cast<const uint8_t *const *>(d_iq), n, true);
}

int modes_pool_collect(modes_pool *p, modes_pool_sink_fn sink, void *user) {
    if (!p) return -1;
    if (p->collected == p->submitted) return fail(p, "no batch in flight");
    modes_pool::Slot &sl = p->slot[p->collected & 1];
    if (sl.ids.empty()) {
        // a call in which no receiver completed a buffer: nothing was scanned; its copies done, the
        // callers' buffers are free again
        if (cudaStreamSynchronize(static_cast<cudaStream_t>(modes_stream(sl.ctx))) != cudaSuccess)
            return fail(p, "%s", cudaGetErrorString(cudaGetLastError()));
        sl.busy = false;
        p->collected++;
        return 0;
    }
    modes::Shard batch;
    if (modes::detect_shard(sl.ctx, batch)) return fail(p, "%s", modes_last_error(sl.ctx));
    const size_t n = sl.ids.size();
    if (sl.feat.levels) {
        sl.level_out.resize(n);
        if (modes_levels_fetch(sl.ctx, sl.level_out.data())) return fail(p, "%s", modes_last_error(sl.ctx));
        for (size_t i = 0; i < n; i++) {
            modes_level r = sl.level_out[i];
            r.buffer = sl.buf_index[i];
            r.n_samples = sl.samples[i];
            p->rx[sl.ids[i]].levels.push(r);
        }
    }
    if (sl.feat.spectrum) {
        if (cudaStreamSynchronize(static_cast<cudaStream_t>(modes_stream(sl.ctx))) != cudaSuccess)
            return fail(p, "%s", cudaGetErrorString(cudaGetLastError()));
        for (size_t i = 0; i < n; i++) p->rx[sl.ids[i]].spectra.push(sl.h_spectra[i]);
    }
    sl.busy = false;
    p->collected++;
    return pool_resolve(p, sl.ids.data(), n, batch, sl.feat.signal, sink, user);
}

int modes_pool_ingest(modes_pool *p, const uint32_t *receivers, const uint8_t *const *iq, size_t n,
                      modes_pool_sink_fn sink, void *user) {
    if (!p) return -1;
    if (p->collected != p->submitted) return fail(p, "a submitted batch is in flight: modes_pool_collect first");
    if (!n) return check_ids(p, receivers, n);
    if (modes_pool_submit(p, receivers, iq, n)) return -1;
    return modes_pool_collect(p, sink, user);
}

int modes_pool_ingest_device(modes_pool *p, const uint32_t *receivers, const void *const *d_iq, size_t n,
                             modes_pool_sink_fn sink, void *user) {
    if (!p) return -1;
    if (p->collected != p->submitted) return fail(p, "a submitted batch is in flight: modes_pool_collect first");
    if (!n) return check_ids(p, receivers, n);
    if (modes_pool_submit_device(p, receivers, d_iq, n)) return -1;
    return modes_pool_collect(p, sink, user);
}

}  // extern "C"

namespace {

// The end of a receiver's stream (modes_pool_finish), tests/pool_finish_model.py.  At 2 MHz as modes_finish ends
// one: a tail of a whole buffer is an ordinary buffer (batch 1), the rest of it the EOF buffer, r.submitted or the
// one after.  At 2.4 MS/s by finish_held's rule: the whole stream has n_in = in_total / 2 + the tail's samples
// (ceil(bytes / 2) UC8, floor(bytes / 4) 16-bit) and N_out = ceil(5 n_in / 6), so buffer N_out / B is the EOF
// buffer and the buffers before it from r.submitted are whole: at most one, the buffer whose filter lookahead
// had not arrived.
struct FinishPlan {
    bool whole;                                // batch 1: buffer r.submitted, whole
    bool eof;                                  // batch 2: the EOF buffer (not with drop_eof_buffer)
    EofPair pair;                              // batch 2's pair
    size_t staged;                             // the tail bytes staged (at 2 MHz a whole tail goes to batch 1 as it is)
};
FinishPlan finish_plan(const Receiver &r, size_t tail, bool drop) {
    const bool uc8 = r.format == modes::input::kUC8;
    auto samples_of = [uc8](size_t bytes) { return uc8 ? ((int64_t)bytes + 1) / 2 : (int64_t)bytes / 4; };
    FinishPlan f;
    f.eof = !drop;
    if (r.rate == kRate2M) {
        f.whole = tail == (uc8 ? kBuf : 2 * kBuf);
        f.staged = f.whole ? 0 : tail;
        f.pair.buffer = r.submitted + (f.whole ? 1 : 0);
        f.pair.samples = (uint32_t)samples_of(f.staged);
    } else {
        const int64_t n_out = modes::resample::n_out(r.in_total / 2 + samples_of(tail));
        f.pair.buffer = n_out / kBufSamples;
        f.whole = f.pair.buffer > r.submitted;
        f.staged = tail;
        f.pair.samples = (uint32_t)(n_out - f.pair.buffer * kBufSamples);
    }
    // the staged buffer's real UC8 bytes (a 16-bit tail's once converted; a trailing odd UC8 byte is an I whose Q,
    // the padding, is 127) and the EOF pair's real output bytes
    f.pair.real8 = 2 * (size_t)samples_of(f.staged);
    f.pair.out_real = 2 * (size_t)f.pair.samples;
    return f;
}

}  // namespace

static int finish_batches(modes_pool *p, const uint32_t *receivers, const uint8_t *const *tails, const size_t *tail_bytes,
                          size_t n, bool device, modes_pool_sink_fn sink, void *user);

static int finish(modes_pool *p, const uint32_t *receivers, const uint8_t *const *tails, const size_t *tail_bytes,
                  size_t n, bool device, modes_pool_sink_fn sink, void *user) {
    using Feed = Receiver::Feed;
    const char *call = device ? "modes_pool_finish_device" : "modes_pool_finish";
    if (!p) return -1;
    if (p->collected != p->submitted) return fail(p, "%s: a submitted batch is in flight: modes_pool_collect first", call);
    if (check_ids(p, receivers, n)) return -1;
    if (!n) return 0;
    if (!tails || !tail_bytes) return fail(p, "%s: no tails", call);
    size_t staging = 0;
    for (size_t i = 0; i < n; i++) {
        const Receiver &r = p->rx[receivers[i]];
        const size_t full = r.format == modes::input::kUC8 ? kBuf : 2 * kBuf;
        if (r.finished) return fail(p, "%s: receiver %u after modes_pool_finish; call modes_pool_reset first", call, receivers[i]);
        if (tail_bytes[i] > full)
            return fail(p, "%s: receiver %u: a tail of %zu bytes, more than its buffer of %zu", call, receivers[i], tail_bytes[i], full);
        if (r.feed == (device ? Feed::host : Feed::device))
            return fail(p, "%s: receiver %u has a stream fed from %s memory in progress; call modes_pool_reset first", call,
                        receivers[i], device ? "host" : "device");
        if (!tail_bytes[i]) continue;
        if (!tails[i]) return fail(p, "%s: receiver %u: null pointer with %zu bytes", call, receivers[i], tail_bytes[i]);
        if (!device) continue;
        if (reinterpret_cast<uintptr_t>(tails[i]) & 15)
            return fail(p, "%s: receiver %u: the tail at %p is not 16-byte aligned", call, receivers[i],
                        static_cast<const void *>(tails[i]));
        const std::string no = modes::device_input_refusal(tails[i], p->cfg.device, "pool", "modes_pool_finish");
        if (!no.empty()) return fail(p, "%s: receiver %u: %s", call, receivers[i], no.c_str());
    }
    for (size_t i = 0; i < n; i++) staging += p->rx[receivers[i]].format == modes::input::kUC8 ? kBuf : 2 * kBuf;
    if (ensure_device(p, !device)) return -1;
    if (device ? p->d_tails.ensure(staging) != cudaSuccess : p->h_tails.ensure(staging) != cudaSuccess) return out_of_memory(p);

    const int rc = finish_batches(p, receivers, tails, tail_bytes, n, device, sink, user);
    // every listed receiver's stream has ended, whether or not its last buffers could be decoded
    for (size_t i = 0; i < n; i++) p->rx[receivers[i]].finished = true;
    return rc;
}

// The tails staged and decoded (checked by finish).
static int finish_batches(modes_pool *p, const uint32_t *receivers, const uint8_t *const *tails, const size_t *tail_bytes,
                          size_t n, bool device, modes_pool_sink_fn sink, void *user) {
    const char *call = device ? "modes_pool_finish_device" : "modes_pool_finish";
    std::vector<FinishPlan> plan(n);
    std::vector<const uint8_t *> staged(n);
    for (size_t i = 0; i < n; i++) {
        const Receiver &r = p->rx[receivers[i]];
        plan[i] = finish_plan(r, tail_bytes[i], p->cfg.drop_eof_buffer != 0);
        if (plan[i].pair.buffer > r.submitted + 1)
            return fail(p, "internal: receiver %u: a finish of buffers %lld to %lld", receivers[i], (long long)r.submitted,
                        (long long)plan[i].pair.buffer);
    }
    // Each tail into a whole buffer of its format, padded with 127: the pool's launches load whole buffers.
    cudaStream_t st = static_cast<cudaStream_t>(modes_stream(p->slot[p->submitted & 1].ctx));
    for (size_t i = 0, at = 0; i < n; i++) {
        const size_t full = p->rx[receivers[i]].format == modes::input::kUC8 ? kBuf : 2 * kBuf, t = plan[i].staged;
        if (device) {
            uint8_t *d = p->d_tails.get() + at;
            if ((t && cudaMemcpyAsync(d, tails[i], t, cudaMemcpyDeviceToDevice, st) != cudaSuccess) ||
                cudaMemsetAsync(d + t, 127, full - t, st) != cudaSuccess)
                return fail(p, "%s: staging the tails failed: %s", call, cudaGetErrorString(cudaGetLastError()));
            staged[i] = d;
        } else {
            uint8_t *h = p->h_tails.get() + at;
            if (t) memcpy(h, tails[i], t);
            memset(h + t, 127, full - t);
            staged[i] = h;
        }
        at += full;
    }
    if (device && cudaStreamSynchronize(st) != cudaSuccess)
        return fail(p, "%s: staging the tails failed: %s", call, cudaGetErrorString(cudaGetLastError()));

    // Batch 1, the whole buffers: a 2 MHz receiver's tail as an ordinary buffer, a 2.4 MS/s receiver's buffer
    // r.submitted from its staged tail.  Batch 2, the EOF buffers.  Each keeps one pair per receiver and batch.
    std::vector<uint32_t> ids;
    std::vector<const uint8_t *> iq;
    std::vector<EofPair> pairs;
    for (int batch = 1; batch <= 2; batch++) {
        ids.clear(); iq.clear(); pairs.clear();
        for (size_t i = 0; i < n; i++) {
            const Receiver &r = p->rx[receivers[i]];
            const FinishPlan &f = plan[i];
            if (batch == 1 ? !f.whole : !f.eof) continue;
            ids.push_back(receivers[i]);
            if (batch == 2) {
                iq.push_back(staged[i]);
                pairs.push_back(f.pair);
            } else if (r.rate == kRate2M) {
                iq.push_back(tails[i]);
                pairs.push_back(EofPair());
            } else {
                EofPair e = f.pair;
                e.buffer = r.submitted;
                e.out_real = kBuf;
                e.samples = (uint32_t)kBufSamples;
                iq.push_back(staged[i]);
                pairs.push_back(e);
            }
        }
        if (ids.empty()) continue;
        if (submit(p, ids.data(), iq.data(), ids.size(), device, pairs.data())) return -1;
        if (modes_pool_collect(p, sink, user)) return -1;
    }
    return 0;
}

extern "C" {

int modes_pool_finish(modes_pool *p, const uint32_t *receivers, const uint8_t *const *tails, const size_t *tail_bytes,
                      size_t n, modes_pool_sink_fn sink, void *user) {
    return finish(p, receivers, tails, tail_bytes, n, false, sink, user);
}

int modes_pool_finish_device(modes_pool *p, const uint32_t *receivers, const void *const *d_tails,
                             const size_t *tail_bytes, size_t n, modes_pool_sink_fn sink, void *user) {
    return finish(p, receivers, reinterpret_cast<const uint8_t *const *>(d_tails), tail_bytes, n, true, sink, user);
}

int modes_pool_stats(const modes_pool *p, uint32_t receiver, modes_stats *out) {
    if (!p || receiver >= p->rx.size() || !out) return -1;
    memcpy(out->v, p->rx[receiver].rs.stats, sizeof(out->v));
    return 0;
}

int modes_pool_reset(modes_pool *p, uint32_t receiver) {
    if (!p || receiver >= p->rx.size()) return -1;
    Receiver &r = p->rx[receiver];
    r.buffers = 0;
    r.submitted = 0;
    r.in_total = 0;
    r.hist0 = 0;
    r.levels.clear();
    r.spectra.clear();
    memset(r.carry, 127, sizeof r.carry);
    r.feed = Receiver::Feed::none;             // its device carry is not read again: the next buffer is a first
    r.finished = false;
    r.rs.reset();
    return 0;
}

int modes_pool_set_input_rate(modes_pool *p, uint32_t receiver, uint32_t hz) {
    if (!p) return -1;
    if (hz != kRate2M && hz != kRate24)
        return fail(p, "modes_pool_set_input_rate: %u samples/s is not supported (2000000 or 2400000)", hz);
    if (receiver >= p->rx.size()) return fail(p, "receiver %u out of range (%zu receivers)", receiver, p->rx.size());
    Receiver &r = p->rx[receiver];
    if (r.submitted || r.in_total || r.finished)
        return fail(p, "modes_pool_set_input_rate: receiver %u has a stream in progress; call modes_pool_reset first", receiver);
    r.rate = hz;
    return 0;
}

int modes_pool_set_input_format(modes_pool *p, uint32_t receiver, uint32_t format, int32_t shift) {
    namespace input = modes::input;
    if (!p) return -1;
    if (!input::known(format))
        return fail(p, "modes_pool_set_input_format: format %u is not supported (MODES_INPUT_UC8, MODES_INPUT_SC16 or "
                       "MODES_INPUT_SC16Q11)", format);
    if (shift > input::kMaxShift)
        return fail(p, "modes_pool_set_input_format: shift %d is not supported (0 to %d, or negative for the format's default)",
                    (int)shift, input::kMaxShift);
    if (format == input::kUC8 && shift > 0)
        return fail(p, "modes_pool_set_input_format: shift %d is not supported with UC8 (0, or negative)", (int)shift);
    if (receiver >= p->rx.size()) return fail(p, "receiver %u out of range (%zu receivers)", receiver, p->rx.size());
    Receiver &r = p->rx[receiver];
    if (r.submitted || r.in_total || r.finished)
        return fail(p, "modes_pool_set_input_format: receiver %u has a stream in progress; call modes_pool_reset first", receiver);
    r.format = format;
    r.shift = shift < 0 ? input::default_shift(format) : (int)shift;
    return 0;
}

int modes_pool_set_output(modes_pool *p, modes_message *out, uint32_t *receiver_of, size_t capacity) {
    if (!p || ((out == nullptr) != (receiver_of == nullptr))) return -1;
    p->out = out; p->out_rx = receiver_of; p->out_cap = out ? capacity : 0; p->out_count = 0;
    return 0;
}

size_t modes_pool_output_count(const modes_pool *p) { return p ? p->out_count : 0; }

int modes_pool_set_arrival(modes_pool *p, int on) { return set_feature(p, &modes::Features::arrival, on); }

int modes_pool_set_carrier(modes_pool *p, int on) { return set_feature(p, &modes::Features::carrier, on); }

int modes_pool_set_signal(modes_pool *p, int on) { return set_feature(p, &modes::Features::signal, on); }

int modes_pool_set_recovery(modes_pool *p, int on) { return set_feature(p, &modes::Features::recover, on); }

int modes_pool_recovery_stats(const modes_pool *p, uint32_t receiver, modes_recovery_stats *out) {
    if (!p || receiver >= p->rx.size() || !out) return -1;
    *out = p->rx[receiver].rs.rstats;
    return 0;
}

int modes_pool_set_weak_preambles(modes_pool *p, int on) { return set_feature(p, &modes::Features::weak, on); }

int modes_pool_weak_stats(const modes_pool *p, uint32_t receiver, modes_recovery_stats *out) {
    if (!p || receiver >= p->rx.size() || !out) return -1;
    *out = p->rx[receiver].rs.wstats;
    return 0;
}

int modes_pool_set_levels(modes_pool *p, int on) { return set_feature(p, &modes::Features::levels, on); }

size_t modes_pool_take_levels(modes_pool *p, uint32_t receiver, modes_level *out, size_t cap) {
    if (!p || receiver >= p->rx.size()) return 0;
    return p->rx[receiver].levels.take(out, cap);
}

int modes_pool_set_spectrum(modes_pool *p, int on) { return set_feature(p, &modes::Features::spectrum, on); }

size_t modes_pool_take_spectra(modes_pool *p, uint32_t receiver, modes_spectrum *out, size_t cap) {
    if (!p || receiver >= p->rx.size()) return 0;
    return p->rx[receiver].spectra.take(out, cap);
}

int64_t modes_pool_buffers(const modes_pool *p, uint32_t receiver) {
    if (!p || receiver >= p->rx.size()) return -1;
    return p->rx[receiver].buffers;
}

}  // extern "C"
