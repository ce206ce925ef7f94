// modes_resolve.cpp — the sequential half of detectModeS(), on the host.
//
// The device evaluates every preamble position independently; what is left is
// the reference's order-dependent control flow, replayed over the candidates in
// stream order (SURVEY.md §8 rows a9, a13-a15, a17):
//   * retry with phase correction when the first attempt is not a good message,
//     skip past a good one (dump1090.c:1769-1791); state restarts at every
//     131072-sample buffer (:1593, :2986)
//   * ICAO address cache: filled by clean DF11/17/18, consulted by the
//     address/parity formats and by DF11 with a small residual
//     (dump1090.c:898-983, :1183-1210)
//   * statistics (dump1090.c:1651, :1662, :1738-1753, :1122-1126)
//   * the sink gate (dump1090.c:1803) and struct modesMessage field decode
//     (:1133-1179, :1212-1308) for delivered messages
#include <atomic>
#include <chrono>
#include <cmath>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <functional>
#include <mutex>
#include <new>
#include <thread>
#include <sched.h>
#include <vector>
#include "modes_internal.h"
#include "modes_carrier_core.cuh"
#include "modes_resolve_core.cuh"

namespace modes {

void ResolveState::reset() {
    std::memset(icao, 0, sizeof(icao));
    std::memset(stats, 0, sizeof(stats));
    cur_buffer = -1;
    next_j = 0;
    next_j_recovered = 0;
    std::memset(&rstats, 0, sizeof(rstats));
    std::memset(&wstats, 0, sizeof(wstats));
}

void ResolveState::start_part(const ResolveState &from, bool at_buffer) {
    *this = from;
    std::memset(stats, 0, sizeof(stats));
    std::memset(&rstats, 0, sizeof(rstats));
    std::memset(&wstats, 0, sizeof(wstats));
    if (at_buffer) { cur_buffer = -1; next_j = 0; next_j_recovered = 0; }
}

static void add_recovery_stats(modes_recovery_stats &to, const modes_recovery_stats &from) {
    to.considered += from.considered; to.found += from.found; to.ambiguous += from.ambiguous;
    to.unknown_address += from.unknown_address; to.dropped += from.dropped; to.delivered += from.delivered;
}

void ResolveState::fold_part(const ResolveState &part) {
    for (int i = 0; i < 8; i++) stats[i] += part.stats[i];
    add_recovery_stats(rstats, part.rstats);
    add_recovery_stats(wstats, part.wstats);
    std::memcpy(icao, part.icao, sizeof(icao));
}

// The host's address cache, for the rules of modes_resolve_core.cuh.
struct IcaoCache {
    uint32_t *slots;
    uint32_t read(uint32_t s) const { return slots[s]; }
    void write(uint32_t s, uint32_t a) { slots[s] = a; }
};

// struct modesMessage fields that are pure functions of the frame bytes.
static void decode_fields(modes_message *o) {
    static const char ais[] = "?ABCDEFGHIJKLMNOPQRSTUVWXYZ????? ???????????????0123456789??????";
    const uint8_t *m = o->msg;
    o->ca = m[0] & 7;
    o->aa1 = m[1]; o->aa2 = m[2]; o->aa3 = m[3];
    o->metype = m[4] >> 3; o->mesub = m[4] & 7;
    o->fs = m[0] & 7;
    o->dr = (m[1] >> 3) & 31;
    o->um = ((m[1] & 7) << 3) | (m[2] >> 5);
    // squawk: C1 A1 C2 A2 C4 A4 0 B1 D1 B2 D2 B4 D4, four octal digits read as decimal
    {
        int A = ((m[3] & 0x80) >> 5) | (m[2] & 0x02) | ((m[2] & 0x08) >> 3);
        int B = ((m[3] & 0x02) << 1) | ((m[3] & 0x08) >> 2) | ((m[3] & 0x20) >> 5);
        int C = ((m[2] & 0x01) << 2) | ((m[2] & 0x04) >> 1) | ((m[2] & 0x10) >> 4);
        int D = ((m[3] & 0x01) << 2) | ((m[3] & 0x04) >> 1) | ((m[3] & 0x10) >> 4);
        o->identity = A * 1000 + B * 100 + C * 10 + D;
    }
    const int df = o->msgtype;
    if (df == 0 || df == 4 || df == 16 || df == 20) {     // 13-bit altitude code
        o->altitude = 0;
        if (m[3] & 0x40) {
            o->unit = 1;                                   // metres: not decoded by the reference
        } else {
            o->unit = 0;
            if (m[3] & 0x10) {
                int n = ((m[2] & 31) << 6) | ((m[3] & 0x80) >> 2) | ((m[3] & 0x20) >> 1) | (m[3] & 15);
                o->altitude = n * 25 - 1000;
            }
        }
    }
    if (df != 17 && df != 18) return;
    const int tc = o->metype, sub = o->mesub;
    if (tc >= 1 && tc <= 4) {
        o->aircraft_type = tc - 1;
        const uint32_t hi = ((uint32_t)m[5] << 16) | ((uint32_t)m[6] << 8) | m[7];
        const uint32_t lo = ((uint32_t)m[8] << 16) | ((uint32_t)m[9] << 8) | m[10];
        for (int k = 0; k < 4; k++) {
            o->flight[k] = ais[(hi >> (18 - 6 * k)) & 63];
            o->flight[4 + k] = ais[(lo >> (18 - 6 * k)) & 63];
        }
        o->flight[8] = 0;
    } else if (tc >= 5 && tc <= 8) {
        o->movement = ((m[4] & 7) << 4) | (m[5] >> 4);
        o->movement_valid = o->movement != 0;
        o->ground_track_valid = (m[5] >> 3) & 1;
        o->ground_track = (((m[5] & 7) << 4) | (m[6] >> 4)) * 360 / 128;
        o->fflag = (m[6] >> 2) & 1;
        o->tflag = (m[6] >> 3) & 1;
        o->raw_latitude = ((m[6] & 3) << 15) | (m[7] << 7) | (m[8] >> 1);
        o->raw_longitude = ((m[8] & 1) << 16) | (m[9] << 8) | m[10];
    } else if (tc >= 9 && tc <= 18) {
        o->fflag = m[6] & 4;                               // the reference keeps the mask value here
        o->tflag = m[6] & 8;
        o->altitude = 0;
        if (m[5] & 1) {
            o->unit = 0;
            o->altitude = (((m[5] >> 1) << 4) | (m[6] >> 4)) * 25 - 1000;
        }
        o->raw_latitude = ((m[6] & 3) << 15) | (m[7] << 7) | (m[8] >> 1);
        o->raw_longitude = ((m[8] & 1) << 16) | (m[9] << 8) | m[10];
    } else if (tc == 19 && sub >= 1 && sub <= 4) {
        if (sub <= 2) {
            o->ew_dir = (m[5] >> 2) & 1;
            o->ew_velocity = ((m[5] & 3) << 8) | m[6];
            o->ns_dir = m[7] >> 7;
            o->ns_velocity = ((m[7] & 0x7f) << 3) | (m[8] >> 5);
            o->vert_rate_source = (m[8] >> 4) & 1;
            o->vert_rate_sign = (m[8] >> 3) & 1;
            o->vert_rate = ((m[8] & 7) << 6) | (m[9] >> 2);
            o->velocity = (int)std::sqrt((double)(o->ns_velocity * o->ns_velocity + o->ew_velocity * o->ew_velocity));
            o->heading = 0;
            if (o->velocity) {
                int ewv = o->ew_dir ? -o->ew_velocity : o->ew_velocity;
                int nsv = o->ns_dir ? -o->ns_velocity : o->ns_velocity;
                double h = std::atan2((double)ewv, (double)nsv);
                o->heading = (int)(h * 360 / (M_PI * 2));
                if (o->heading < 0) o->heading += 360;
            }
        } else {
            o->heading_is_valid = m[5] & 4;
            o->heading = (int)((360.0 / 128) * (((m[5] & 3) << 5) | (m[6] >> 3)));
        }
    }
}

static void build_message(const modes_frame_eval &p, int crcok, uint32_t iid, uint32_t ap_addr, modes_message *o) {
    std::memset(o, 0, sizeof(*o));
    std::memcpy(o->msg, p.msg, 14);
    o->msgtype = p.msgtype;
    o->msgbits = (int32_t)rcore::bits_by_type(p.msgtype);
    o->crc = p.crc;
    o->nfixed = p.nfixed;
    o->signal = p.signal;
    o->arrival = (uint8_t)(p.flags >> MODES_EVAL_ARRIVAL_SHIFT);
    o->errorbit = p.nfixed ? (int)p.errorbit : -1;
    o->crcok = crcok;
    o->iid = (int32_t)iid;
    decode_fields(o);
    if (ap_addr) { o->aa1 = (ap_addr >> 16) & 0xff; o->aa2 = (ap_addr >> 8) & 0xff; o->aa3 = ap_addr & 0xff; }
}

// A judged attempt's message fields: the DF11 interrogator id, the address of an address/parity format.
static inline uint32_t iid_of(const rcore::Decision &d) { return d.extra_is_ap ? 0u : d.extra; }
static inline uint32_t ap_addr_of(const rcore::Decision &d) { return d.extra_is_ap ? d.extra : 0u; }

int finish_message(ResolveState &st, const modes_frame_eval &p, modes_message *o) {
    IcaoCache cache{st.icao};
    rcore::Decision d{};
    const int crcok = (int)rcore::judge(st, cache, p, d);
    build_message(p, crcok, iid_of(d), ap_addr_of(d), o);
    return crcok;
}

// ---- delivered messages: verdicts first (sequential), structs second (parallel)

// What the sequential pass decides about one delivered message; the 200-byte
// struct is built from it afterwards, in parallel for array output.
struct Delivery {
    modes_frame_eval eval;       // copied while the verdict pass has the record's line: the struct-building pass then
                                 // streams through the list instead of chasing 425 744 pointers into the record array
    int64_t sample_pos;
    uint32_t iid, ap_addr;
    uint8_t crcok, phase_corrected;
    uint8_t recovered;           // eval is a recovery record's frame (1: at a candidate, 2: at a weak preamble): crc 0, nfixed = its flips
    int16_t carrier;             // the attempt's carrier code (0: not measured)
};

// Cores this process may actually keep busy: the CPUs it is allowed on, cut down to the CPU-time
// quota of its control group (a container that sees 128 CPUs but is granted 16 CPUs' worth of time
// is throttled as a whole when its threads exceed the quota: more threads then means stalls).
unsigned host_cpu_budget() {
    unsigned n = std::thread::hardware_concurrency();
    if (n == 0) n = 1;
    cpu_set_t set;
    if (sched_getaffinity(0, sizeof(set), &set) == 0) {
        const unsigned a = (unsigned)CPU_COUNT(&set);
        if (a >= 1 && a < n) n = a;
    }
    long long quota = -1, period = 0;
    if (FILE *f = std::fopen("/sys/fs/cgroup/cpu.max", "r")) {                       // cgroup v2: "<quota|max> <period>"
        char q[32];
        if (std::fscanf(f, "%31s %lld", q, &period) == 2 && std::strcmp(q, "max") != 0) quota = std::atoll(q);
        std::fclose(f);
    } else {                                                                         // cgroup v1
        FILE *fq = std::fopen("/sys/fs/cgroup/cpu/cpu.cfs_quota_us", "r"), *fp = std::fopen("/sys/fs/cgroup/cpu/cpu.cfs_period_us", "r");
        if (fq && fp && std::fscanf(fq, "%lld", &quota) == 1 && std::fscanf(fp, "%lld", &period) == 1) {} else quota = -1;
        if (fq) std::fclose(fq);
        if (fp) std::fclose(fp);
    }
    if (quota > 0 && period > 0) {
        const unsigned c = (unsigned)((quota + period - 1) / period);
        if (c >= 1 && c < n) n = c;
    }
    return n;
}

// A few helper threads for building message structs; created on first use.
class BuildPool {
  public:
    static BuildPool &get() { static BuildPool *p = new BuildPool();  /* never destroyed: workers are detached */ return *p; }
    // One job at a time: the job state below (fn_, n_, next_, pending_) belongs to whoever holds
    // job_mu_ for the whole job.  A second context on another thread that finds the pool busy
    // builds its structs itself instead of waiting (distinct contexts are independent).
    void run(size_t n, const std::function<void(size_t, size_t)> &fn) {
        if (workers_.empty() || n < 2048) { fn(0, n); return; }
        std::unique_lock<std::mutex> job(job_mu_, std::try_to_lock);
        if (!job.owns_lock()) { fn(0, n); return; }
        std::unique_lock<std::mutex> lk(mu_);
        fn_ = &fn; n_ = n; next_ = 0; pending_ = workers_.size(); gen_++;
        cv_.notify_all();
        lk.unlock();
        work();                                            // the caller helps
        lk.lock();
        done_.wait(lk, [&] { return pending_ == 0; });
    }
  private:
    BuildPool() {
        // message structs are ~200 B of stores each: a handful of threads saturates one socket's
        // write bandwidth.  MODES_BUILD_THREADS overrides (total threads, including the caller).
        unsigned hw = host_cpu_budget();
        unsigned nw = hw > 32 ? 15 : (hw > 16 ? 7 : (hw > 2 ? hw / 2 - 1 : 0));
        if (const char *e = std::getenv("MODES_BUILD_THREADS")) { int v = std::atoi(e); if (v >= 1 && v <= 256) nw = (unsigned)v - 1; }
        for (unsigned i = 0; i < nw; i++) workers_.emplace_back([this] { loop(); });
        for (auto &t : workers_) t.detach();
    }
    void work() {
        for (;;) {
            size_t b = next_.fetch_add(1024);
            if (b >= n_) break;
            (*fn_)(b, b + 1024 < n_ ? b + 1024 : n_);
        }
    }
    void loop() {
        uint64_t seen = 0;
        for (;;) {
            std::unique_lock<std::mutex> lk(mu_);
            cv_.wait(lk, [&] { return gen_ != seen; });
            seen = gen_;
            lk.unlock();
            work();
            lk.lock();
            if (--pending_ == 0) done_.notify_all();
        }
    }
    std::vector<std::thread> workers_;
    std::mutex job_mu_;
    std::mutex mu_;
    std::condition_variable cv_, done_;
    const std::function<void(size_t, size_t)> *fn_ = nullptr;
    size_t n_ = 0, pending_ = 0;
    std::atomic<size_t> next_{0};
    uint64_t gen_ = 0;
};

// With recovery records (rec[k] belongs to cands[k]; include/modes_b200.h rules 1-6), a candidate the
// walk visits where neither attempt was good may add a recovered message.  It goes into the list at
// once, in stream order, and is taken out again if the reference delivers a good message within its
// span (rule 6): only deliveries of the same buffer at later positions can follow it by then.
constexpr uint32_t kRecoveredSpan = 241;                  // (8 + 112) * 2 + 1: the skip of a long message

struct RecoveryPending {                                  // the recovered message rule 6 may still drop
    size_t index = SIZE_MAX;                              // in the delivery list
    int64_t buffer = -1;
    uint32_t end = 0;                                     // first position of the buffer outside its span
    modes_recovery_stats *stats = nullptr;                // the statistics it was counted in
};

// The recovery rules at one visited candidate, after the reference's attempts there (good: one of
// them was judged crcok), or at a visited weak position (good = false, stats = st.wstats, marker 2).
static inline void recovery_step(ResolveState &st, const ResolveConfig &cfg, const modes_recovered &r, bool good,
                                 int64_t buffer, uint32_t j, int64_t pos, std::vector<Delivery> &deliveries,
                                 RecoveryPending &pend, modes_recovery_stats &stats, uint8_t marker) {
    if (good) {                                                            // rule 6
        if (pend.index != SIZE_MAX && pend.buffer == buffer && j < pend.end) {
            // what follows it in the list lies in this buffer within its span: a few entries move
            deliveries.erase(deliveries.begin() + (ptrdiff_t)pend.index);
            pend.stats->dropped++;
            pend.stats->delivered--;
            pend.index = SIZE_MAX;
        }
        return;
    }
    if (r.status == MODES_RECOVER_INELIGIBLE) return;                      // rule 2 holds
    stats.considered++;
    if (j < st.next_j_recovered) return;                                   // rule 3
    if (r.status == MODES_RECOVER_AMBIGUOUS) stats.ambiguous++;
    if (r.status != MODES_RECOVER_FOUND) return;                           // rule 4
    stats.found++;
    const uint32_t addr = ((uint32_t)r.msg[1] << 16) | ((uint32_t)r.msg[2] << 8) | (uint32_t)r.msg[3];
    IcaoCache cache{st.icao};
    if (!rcore::seen(cache, addr)) { stats.unknown_address++; return; }    // rule 5
    modes_frame_eval e{};
    std::memcpy(e.msg, r.msg, 14);
    e.msgtype = (uint8_t)(r.msg[0] >> 3);
    e.nfixed = r.nflips;
    e.errorbit = 0xFF;
    e.signal = cfg.recover_signal ? r.signal : 0;
    e.crc = 0;
    pend.index = deliveries.size();
    pend.buffer = buffer;
    pend.end = j + kRecoveredSpan;
    pend.stats = &stats;
    st.next_j_recovered = j + kRecoveredSpan;
    deliveries.push_back(Delivery{e, pos, 0u, 0u, (uint8_t)1, (uint8_t)0, marker, (int16_t)0});
    stats.delivered++;
}

// The weak positions of the buffers [b_lo, b_hi) of a record array, merged into the walk: `next` is
// the first one not visited yet.
struct WeakCursor {
    const WeakList *w = nullptr;
    size_t next = 0;
};

// Visit the weak positions before record position `until` (and before buffer b_hi).
static inline void weak_steps(ResolveState &st, const ResolveConfig &cfg, WeakCursor &wc, uint64_t until, uint32_t b_hi,
                              int64_t buffer_base, std::vector<Delivery> &deliveries, RecoveryPending &pend) {
    for (; wc.next < wc.w->n && wc.w->t[wc.next] < until; wc.next++) {
        const uint32_t t = wc.w->t[wc.next];
        if ((t >> 17) >= b_hi) { wc.next = wc.w->n; return; }
        const int64_t buffer = buffer_base + (t >> 17);
        const uint32_t j = t & (kBufSamples - 1);
        if (buffer != st.cur_buffer) { st.cur_buffer = buffer; st.next_j = 0; st.next_j_recovered = 0; }
        if (j < st.next_j) continue;                       // inside a message the reference took (rule 1)
        const int64_t pos = buffer * (int64_t)kBufSamples + j - MODES_CARRY_SAMPLES;
        recovery_step(st, cfg, wc.w->rec[wc.next], false, buffer, j, pos, deliveries, pend, st.wstats, 2);
    }
}

// A run of a shard's record array judged in one sequence (see "parts" below).
struct Part {
    const Shard *shard;
    size_t tile_lo;              // first tile that can hold one of its candidates
    uint32_t b_lo, b_hi;         // its buffers, as numbered in the records (t >> 17)
    bool first_of_shard;         // the tail pass for a shard's first part walks the previous SHARD's array
};

// The verdict pass over the tiles of a part from tile_lo on: everything order-dependent, no message
// structs yet.  Only the candidates of the part's buffers [b_lo, b_hi) are judged; the walk ends at the
// first candidate of buffer b_hi or later (records are in stream order).  kRecover: apply the recovery
// rules with the shard's recovery records and merge its weak positions into the walk (the walk without
// them has no trace of them).
template <bool kRecover>
static void walk_tiles(ResolveState &st, const ResolveConfig &cfg, const Part &p, std::vector<Delivery> &deliveries) {
    const Shard &s = *p.shard;
    const modes_candidate *cands = s.cands;
    const modes_tile *tiles = s.tiles + p.tile_lo;
    const size_t n_tiles = s.n_tiles - p.tile_lo;
    const uint32_t b_lo = p.b_lo, b_hi = p.b_hi;
    const int64_t buffer_base = s.buffer_base;
    const modes_carrier *car = s.carrier;
    RecoveryPending pend;
    WeakCursor wc;
    const bool merge = kRecover && s.weak.n;
    if (merge) {                                           // the first weak position of buffer b_lo or later
        wc.w = &s.weak;
        const uint64_t lo = (uint64_t)b_lo << 17;
        size_t a = 0, b = s.weak.n;
        while (a < b) { const size_t m = (a + b) / 2; if (s.weak.t[m] < lo) a = m + 1; else b = m; }
        wc.next = a;
    }
    // The kernels append a tile's records wherever the global cursor stands when the tile finishes:
    // records are contiguous per tile but the tiles lie scattered through the array, so walking them
    // in stream order is a chain of cache misses (the records were just written by DMA).  Request
    // the lines of a tile well before it is reached.
    constexpr size_t kAhead = 24;
    IcaoCache cache{st.icao};
    for (size_t ti = 0; ti < n_tiles; ti++) {
        if (ti + kAhead < n_tiles && tiles[ti + kAhead].count) {
            const char *p = reinterpret_cast<const char *>(cands + tiles[ti + kAhead].offset);
            const size_t bytes = (size_t)tiles[ti + kAhead].count * sizeof(modes_candidate);
            for (size_t o = 0; o < bytes && o < 512; o += 64) __builtin_prefetch(p + o, 0, 1);
        }
        const size_t k0 = tiles[ti].offset;
        for (uint32_t k = 0; k < tiles[ti].count; k++) {
            const modes_candidate *c = cands + k0 + k;
            const uint32_t rb = (uint32_t)(c->t >> 17);
            if (rb < b_lo) continue;                       // the part before this one takes it
            if (rb >= b_hi) {                              // the next part's
                if (merge) weak_steps(st, cfg, wc, UINT64_MAX, b_hi, buffer_base, deliveries, pend);
                return;
            }
            if (merge) weak_steps(st, cfg, wc, (uint64_t)c->t, b_hi, buffer_base, deliveries, pend);
            const int64_t buffer = buffer_base + rb;
            const uint32_t j = (uint32_t)(c->t & (kBufSamples - 1));
            if (buffer != st.cur_buffer) { st.cur_buffer = buffer; st.next_j = 0; st.next_j_recovered = 0; }
            rcore::Decision d[2] = {};
            const int visit = rcore::candidate(st, cache, j, c->pass[0], c->pass[1], cfg.check_crc, d);
            if (visit < 0) continue;                       // inside a message already taken (rule 1)
            const int64_t pos = buffer * (int64_t)kBufSamples + j - MODES_CARRY_SAMPLES;
            for (int a = 0; a < 2; a++)
                if (d[a].deliver)
                    deliveries.push_back(Delivery{c->pass[a], pos, iid_of(d[a]), ap_addr_of(d[a]), (uint8_t)d[a].crcok,
                                                  (uint8_t)d[a].phase_corrected, (uint8_t)0,
                                                  car ? carrier::code_of(car[k0 + k].re[a], car[k0 + k].im[a]) : (int16_t)0});
            if constexpr (kRecover)
                recovery_step(st, cfg, s.recovered[k0 + k], visit > 0, buffer, j, pos, deliveries, pend, st.rstats, 1);
        }
    }
    if (merge) weak_steps(st, cfg, wc, UINT64_MAX, b_hi, buffer_base, deliveries, pend);
}

static void judge_tiles(ResolveState &st, const ResolveConfig &cfg, const Part &p, std::vector<Delivery> &deliveries) {
    if (p.shard->recovered) walk_tiles<true>(st, cfg, p, deliveries);
    else walk_tiles<false>(st, cfg, p, deliveries);
}

// Build n delivered structs with build(i, struct): in place and in parallel for array output, then
// the callback (if any) sequentially in stream order.
template <class Build>
static void deliver_each(size_t n, MessageOut &out, const Build &build) {
    size_t in_array = 0;
    if (out.array && out.count < out.capacity) {
        in_array = out.capacity - out.count < n ? out.capacity - out.count : n;
        modes_message *base = out.array + out.count;
        BuildPool::get().run(in_array, [&](size_t b, size_t e) { for (size_t i = b; i < e; i++) build(i, base + i); });
    }
    if (out.sink) {
        for (size_t i = 0; i < n; i++) {
            if (i < in_array) { out.sink(out.user, out.array + out.count + i); continue; }
            modes_message tmp;
            build(i, &tmp);
            out.sink(out.user, &tmp);
        }
    }
    out.count += n;
}

static void deliver(const std::vector<Delivery> &deliveries, MessageOut &out) {
    deliver_each(deliveries.size(), out, [d = deliveries.data()](size_t i, modes_message *mm) {
        build_message(d[i].eval, d[i].crcok, d[i].iid, d[i].ap_addr, mm);
        mm->sample_pos = d[i].sample_pos;
        mm->phase_corrected = d[i].phase_corrected;
        if (d[i].recovered) { mm->recovered = d[i].recovered; mm->errorbit = -1; }
        mm->carrier = d[i].carrier;
    });
}

void deliver_gpu(const modes_delivery *d, size_t n, int64_t buffer_base, MessageOut &out) {
    deliver_each(n, out, [=](size_t i, modes_message *mm) {
        const bool is_ap = (d[i].bits >> 16) & 1u;
        build_message(d[i].eval, (int)(d[i].bits & 1u), is_ap ? 0u : d[i].extra, is_ap ? d[i].extra : 0u, mm);
        mm->sample_pos = (buffer_base << 17) + d[i].t - MODES_CARRY_SAMPLES;
        mm->phase_corrected = (int)((d[i].bits >> 8) & 1u);
    });
}

// ---- parts of a stream judged concurrently, exactly
//
// The only state that crosses a buffer boundary is the ICAO address cache (the skip state restarts
// at every reference buffer, dump1090.c:1593).  A stream is therefore cut into PARTS of whole
// buffers — the shards of a multi-GPU decode, and each long shard once more into a few parts for
// this host's threads — and part k is judged from a GUESS of the cache at its start: first the
// cache the call started with, overwritten by what the tail of part k-1 writes; in later rounds the
// cache part k-1 ended with in the previous round.  The guess is verified afterwards against the
// cache part k-1 really ended with, and a part whose guess was wrong is simply judged again.  One
// round normally suffices; in the worst case the loop degenerates to the sequential order, never
// to a wrong result.
struct PartRun { ResolveState start, end; std::vector<Delivery> deliveries; };
struct ResolveScratch {
    std::vector<Part> parts;
    std::vector<PartRun> runs;   // kept between calls: delivery lists keep their capacity (growing them from nothing
                                 // in every call costs more in page faults, taken concurrently, than the verdicts)
    size_t n_runs_held = 0;      // the last resolve's deliveries are in runs[0 .. n_runs_held) until delivered
};
ResolveScratch *scratch_create() { return new (std::nothrow) ResolveScratch(); }
void scratch_destroy(ResolveScratch *s) { delete s; }

// How many parts a record array of n_tiles tiles is worth on this host: a part should be long
// enough (default 4096 tiles = 32 M samples) to repay its thread and its tail pass, and there is no
// point in more parts than threads.  MODES_RESOLVE_PARTS = 1 keeps the sequential pass;
// MODES_RESOLVE_PART_TILES sets the minimum part length (tests use small values).
static size_t parts_for(size_t n_tiles) {
    static const unsigned budget = host_cpu_budget();
    auto env_num = [](const char *name) { const char *e = std::getenv(name); return e ? std::atol(e) : 0L; };
    const long env_parts = env_num("MODES_RESOLVE_PARTS"), env_tiles = env_num("MODES_RESOLVE_PART_TILES");
    size_t max_parts = budget >= 16 ? 8 : (budget >= 4 ? budget / 2 : 1);
    const long share = env_num("MODES_BUILD_THREADS");                   // the caller's share of a host it shares with other ranks
    if (share >= 1 && (size_t)share < max_parts) max_parts = (size_t)share;
    if (env_parts > 0) max_parts = (size_t)env_parts;
    const size_t min_tiles = env_tiles > 0 ? (size_t)env_tiles : 4096;
    size_t p = n_tiles / min_tiles;
    if (p > max_parts) p = max_parts;
    return p < 1 ? 1 : p;
}

// Cut a shard's buffers [b_lo, b_hi) into up to `want` parts at buffer boundaries.  The boundary of
// part k is read from the records themselves: the buffer after the one the first candidate at or behind
// tile k * n_tiles / want lies in (tiles do not line up with buffers; records are in stream order).
static void cut_parts(const Shard &s, size_t want, std::vector<Part> &parts) {
    Part p{&s, 0, s.b_lo, s.b_hi, true};
    for (size_t k = 1; k < want; k++) {
        size_t ti = k * s.n_tiles / want;
        while (ti < s.n_tiles && s.tiles[ti].count == 0) ti++;
        if (ti >= s.n_tiles) break;
        const uint32_t b = (uint32_t)(s.cands[s.tiles[ti].offset].t >> 17) + 1;  // first buffer of the next part
        if (b <= p.b_lo) continue;                                                 // (a gap longer than a part)
        if (b >= s.b_hi) break;
        p.b_hi = b;
        parts.push_back(p);
        p.tile_lo = ti; p.b_lo = b; p.b_hi = s.b_hi; p.first_of_shard = false;
    }
    parts.push_back(p);
}

// Judge the parts (rounds of guess and verify, see above); runs[k] receives part k's deliveries
// and statistics, `st` the state after the last part.  A single part is judged in place on `st`.
static int judge_parts(ResolveState &st, const ResolveConfig &cfg, const std::vector<Part> &parts, PartRun *runs) {
    const size_t n = parts.size();
    if (n == 1) {
        runs[0].deliveries.clear();
        judge_tiles(st, cfg, parts[0], runs[0].deliveries);
        return 1;
    }
    ResolveState blank;
    blank.reset();
    auto run_part = [&](size_t k, const ResolveState &from) {
        PartRun &r = runs[k];
        r.start.start_part(from, k != 0);                  // a later part starts a buffer
        r.end = r.start;
        r.deliveries.clear();
        judge_tiles(r.end, cfg, parts[k], r.deliveries);
    };
    int rounds = 0;
    size_t done = 0;                                       // parts [0, done) are final
    for (int round = 0; done < n; round++, rounds++) {
        // fix every guess before any thread of this round starts rewriting runs[*].end
        std::vector<ResolveState> guess(n);
        std::vector<char> rerun(n, 0);
        for (size_t k = done; k < n; k++) {
            guess[k] = (k == done) ? (done ? runs[done - 1].end : st) : (round ? runs[k - 1].end : blank);
            rerun[k] = round == 0 || k == done || std::memcmp(guess[k].icao, runs[k].start.icao, sizeof(blank.icao)) != 0;
        }
        auto job = [&](size_t k) {
            if (!(round == 0 && k > done)) { run_part(k, guess[k]); return; }
            // First guess: the cache this call started with, overwritten by what the LAST SIXTEENTH of
            // part k-1 writes (addresses are re-confirmed every second or so, so the tail of a long
            // part has normally written every slot the whole part leaves changed).
            Part q = parts[k - 1];
            ResolveState g;
            g.start_part(st, true);
            const size_t n_tiles = q.shard->n_tiles;
            const size_t end_tile = parts[k].first_of_shard ? n_tiles : (parts[k].tile_lo + 1 < n_tiles ? parts[k].tile_lo + 1 : n_tiles);
            const size_t len = end_tile - q.tile_lo;
            size_t tail = len / 16 > 128 ? len / 16 : 128;             // at least ~1 M samples (half a second of stream)
            if (tail > len) tail = len;
            q.tile_lo = end_tile - tail;
            runs[k].deliveries.clear();
            walk_tiles<false>(g, cfg, q, runs[k].deliveries);          // recovery never writes the cache: the guess skips it
            run_part(k, g);
        };
        std::vector<std::thread> th;
        size_t mine = n;                                   // the caller judges one part itself
        for (size_t k = done; k < n; k++) {
            if (!rerun[k]) continue;
            if (mine == n) { mine = k; continue; }
            th.emplace_back(job, k);
        }
        if (mine < n) job(mine);
        for (auto &t : th) t.join();
        // accept the longest verified prefix
        for (; done < n; done++) {
            const ResolveState &truth = done ? runs[done - 1].end : st;
            if (std::memcmp(truth.icao, runs[done].start.icao, sizeof(truth.icao)) != 0) break;
        }
    }
    for (size_t k = 0; k < n; k++) st.fold_part(runs[k].end);
    // the skip state is that of the last part that saw a candidate (an empty part leaves none)
    for (size_t k = n; k-- > 0;)
        if (runs[k].end.cur_buffer != -1 || k == 0) {
            st.cur_buffer = runs[k].end.cur_buffer; st.next_j = runs[k].end.next_j;
            st.next_j_recovered = runs[k].end.next_j_recovered;
            break;
        }
    return rounds;
}

// Judge several shards of one stream (e.g. one per GPU) concurrently and exactly: every shard is a
// part, long shards are cut once more (see judge_parts).  The deliveries are held in the scratch
// until resolve_commit.  Returns the rounds judge_parts took.
static int judge_shards(ResolveState &st, const ResolveConfig &cfg, const Shard *shards, size_t n_shards, ResolveScratch *scratch) {
    std::vector<Part> &parts = scratch->parts;
    parts.clear();
    size_t threads_left = parts_for((size_t)-1);
    for (size_t k = 0; k < n_shards; k++) {
        size_t want = parts_for(shards[k].n_tiles);
        const size_t share = threads_left / (n_shards - k) > 0 ? threads_left / (n_shards - k) : 1;
        if (want > share) want = share;
        cut_parts(shards[k], want, parts);
        threads_left = threads_left > want ? threads_left - want : 0;
    }
    if (scratch->runs.size() < parts.size()) scratch->runs.resize(parts.size());
    const int rounds = judge_parts(st, cfg, parts, scratch->runs.data());
    scratch->n_runs_held = parts.size();
    return rounds;
}

void resolve_commit(MessageOut &out, ResolveScratch *scratch) {
    for (size_t k = 0; k < scratch->n_runs_held; k++) { deliver(scratch->runs[k].deliveries, out); scratch->runs[k].deliveries.clear(); }
    scratch->n_runs_held = 0;
}

void resolve_shards(ResolveState &st, const ResolveConfig &cfg, const Shard *shards, size_t n_shards, MessageOut &out,
                    ResolveScratch *scratch) {
    const bool timing = std::getenv("MODES_RESOLVE_TIMING") != nullptr;
    auto now = [] { return std::chrono::steady_clock::now(); };
    const auto t_start = now();
    const int rounds = judge_shards(st, cfg, shards, n_shards, scratch);
    const size_t n_parts = scratch->n_runs_held;
    const auto t_judged = now();
    resolve_commit(out, scratch);
    if (timing)
        std::fprintf(stderr, "resolve: %zu shards in %zu parts, %d rounds, verdicts %.2f ms, structs %.2f ms\n", n_shards, n_parts,
                     rounds, std::chrono::duration<double, std::milli>(t_judged - t_start).count(),
                     std::chrono::duration<double, std::milli>(now() - t_judged).count());
}

void resolve_candidates(ResolveState &st, const ResolveConfig &cfg, const Shard &shard, MessageOut &out, ResolveScratch *scratch) {
    resolve_shards(st, cfg, &shard, 1, out, scratch);
}

void resolve_tentative(ResolveState &st, const ResolveConfig &cfg, const Shard &shard, ResolveScratch *scratch) {
    judge_shards(st, cfg, &shard, 1, scratch);
}

}  // namespace modes
