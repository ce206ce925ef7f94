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

static inline uint32_t icao_slot(uint32_t a) {           // dump1090.c:898-905
    a = ((a >> 16) ^ a) * 0x45d9f3bu;
    a = ((a >> 16) ^ a) * 0x45d9f3bu;
    a = (a >> 16) ^ a;
    return a & 1023u;
}

static inline bool icao_seen(const ResolveState &st, uint32_t a) {
    return a != 0 && st.icao[icao_slot(a)] == a;         // dump1090.c:919-925, TTL not modelled
}

static inline int bits_by_type(int df) { return (df >= 16 && df <= 21) ? 112 : 56; }

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

// Order-dependent verdict of decodeModesMessage for one evaluated frame
// (dump1090.c:1108-1128 statistics, :1183-1210 ICAO logic) without building the
// message: returns crcok; *iid and *ap_addr receive the DF11 interrogator id and
// the recovered address of an address/parity format (0 when not applicable).
static inline int judge(ResolveState &st, const modes_frame_eval &p, uint32_t *iid, uint32_t *ap_addr) {
    *iid = 0; *ap_addr = 0;
    if (p.nfixed == 1) st.stats[6]++;                      // dump1090.c:1122-1126
    else if (p.nfixed == 2) st.stats[7]++;
    const int df = p.msgtype;
    int crcok = p.crc == 0;
    if (df == 11 || df == 17 || df == 18) {
        const uint32_t addr = ((uint32_t)p.msg[1] << 16) | ((uint32_t)p.msg[2] << 8) | (uint32_t)p.msg[3];
        if (crcok && p.nfixed == 0) st.icao[icao_slot(addr)] = addr;          // :1198-1200
        if (df == 11 && !crcok && p.crc < 80 && icao_seen(st, addr)) {         // :1204-1209
            *iid = p.crc;
            crcok = 1;
        }
        return crcok;
    }
    // parity field = CRC ^ address, so the syndrome is the sender's address (:962-974)
    if ((df == 0 || df == 4 || df == 5 || df == 16 || df == 20 || df == 21 || df == 24) && icao_seen(st, p.crc)) {
        *ap_addr = p.crc;
        return 1;
    }
    return 0;
}

static void build_message(const modes_frame_eval &p, int crcok, uint32_t iid, uint32_t ap_addr, modes_message *o) {
    std::memset(o, 0, sizeof(*o));
    std::memcpy(o->msg, p.msg, 14);
    o->msgtype = p.msgtype;
    o->msgbits = bits_by_type(p.msgtype);
    o->crc = p.crc;
    o->nfixed = p.nfixed;
    o->signal = p.signal;
    o->errorbit = p.nfixed ? (int)p.errorbit : -1;
    o->crcok = crcok;
    o->iid = (int32_t)iid;
    decode_fields(o);
    if (ap_addr) { o->aa1 = (ap_addr >> 16) & 0xff; o->aa2 = (ap_addr >> 8) & 0xff; o->aa3 = ap_addr & 0xff; }
}

int finish_message(ResolveState &st, const modes_frame_eval &p, modes_message *o) {
    uint32_t iid, ap;
    const int crcok = judge(st, p, &iid, &ap);
    build_message(p, crcok, iid, ap, o);
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
};

static inline void materialise(const Delivery &d, modes_message *mm) {
    build_message(d.eval, d.crcok, d.iid, d.ap_addr, mm);
    mm->sample_pos = d.sample_pos;
    mm->phase_corrected = d.phase_corrected;
    if (d.recovered) { mm->recovered = d.recovered; mm->errorbit = -1; }
}

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

// One evaluated attempt, as detectModeS handles it after the delta gate.
// Returns true when the message is good (the scan skips past it).
static inline bool attempt(ResolveState &st, const ResolveConfig &cfg, const modes_frame_eval &p, bool retry,
                           int64_t sample_pos, std::vector<Delivery> &deliveries) {
    if (!(p.flags & MODES_EVAL_DECODED)) return false;
    uint32_t iid, ap;
    const int crcok = judge(st, p, &iid, &ap);
    if (crcok || retry) {                                  // dump1090.c:1738-1753
        if (!(p.flags & MODES_EVAL_ERRORS)) st.stats[2]++;
        if (p.nfixed == 0) st.stats[crcok ? 3 : 4]++;
        else { st.stats[4]++; st.stats[5]++; st.stats[6]++; }
    }
    if (cfg.check_crc == 0 || crcok)                       // dump1090.c:1803; :1772-1773
        deliveries.push_back(Delivery{p, sample_pos, iid, ap, (uint8_t)crcok, (uint8_t)(crcok && retry), (uint8_t)0});
    return crcok != 0;
}

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
    if (!icao_seen(st, addr)) { stats.unknown_address++; return; }         // rule 5
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
    deliveries.push_back(Delivery{e, pos, 0u, 0u, (uint8_t)1, (uint8_t)0, marker});
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

// The verdict pass over one run of tiles: everything order-dependent, no message structs yet.
// `b_lo`, `b_hi`: only the candidates of the buffers [b_lo, b_hi) of this record array are judged (buffer
// numbers as in the records: t >> 17); the walk ends at the first candidate of buffer b_hi or later
// (records are in stream order).  The whole array: 0, UINT32_MAX.  kRecover: apply the recovery rules
// with `rec` and merge the weak positions `weak` (may be nullptr) into the walk (the walk without
// them has no trace of them).
template <bool kRecover>
static void walk_tiles(ResolveState &st, const ResolveConfig &cfg, const modes_candidate *cands, const modes_tile *tiles,
                       size_t n_tiles, int64_t buffer_base, std::vector<Delivery> &deliveries, uint32_t b_lo, uint32_t b_hi,
                       const modes_recovered *rec, const WeakList *weak) {
    RecoveryPending pend;
    WeakCursor wc;
    const bool merge = kRecover && weak && weak->n;
    if (merge) {                                           // the first weak position of buffer b_lo or later
        wc.w = weak;
        const uint64_t lo = (uint64_t)b_lo << 17;
        size_t a = 0, b = weak->n;
        while (a < b) { const size_t m = (a + b) / 2; if (weak->t[m] < lo) a = m + 1; else b = m; }
        wc.next = a;
    }
    // The kernels append a tile's records wherever the global cursor stands when the tile finishes:
    // records are contiguous per tile but the tiles lie scattered through the array, so walking them
    // in stream order is a chain of cache misses (the records were just written by DMA).  Request
    // the lines of a tile well before it is reached.
    constexpr size_t kAhead = 24;
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
            if (j < st.next_j) continue;                   // inside a message already taken (rule 1)
            st.stats[0]++;                                 // dump1090.c:1651
            const int64_t pos = buffer * (int64_t)kBufSamples + j - MODES_CARRY_SAMPLES;
            bool good = false;
            const modes_frame_eval &p1 = c->pass[0];
            if (p1.flags & MODES_EVAL_GATE_OK) {           // dump1090.c:1723-1726
                const uint32_t skip = (uint32_t)(8 + bits_by_type(p1.msgtype)) * 2 + 1;
                if (attempt(st, cfg, p1, false, pos, deliveries)) {
                    st.next_j = j + skip;
                    good = true;
                } else {
                    if (j) st.stats[1]++;                  // dump1090.c:1660-1663
                    const modes_frame_eval &p2 = c->pass[1];
                    if (p2.flags & MODES_EVAL_GATE_OK) {
                        const uint32_t skip2 = (uint32_t)(8 + bits_by_type(p2.msgtype)) * 2 + 1;
                        if (attempt(st, cfg, p2, true, pos, deliveries)) { st.next_j = j + skip2; good = true; }
                    }
                }
            }
            if constexpr (kRecover) recovery_step(st, cfg, rec[k0 + k], good, buffer, j, pos, deliveries, pend, st.rstats, 1);
            (void)good;
        }
    }
    if (merge) weak_steps(st, cfg, wc, UINT64_MAX, b_hi, buffer_base, deliveries, pend);
}

static void judge_tiles(ResolveState &st, const ResolveConfig &cfg, const modes_candidate *cands, const modes_tile *tiles,
                        size_t n_tiles, int64_t buffer_base, std::vector<Delivery> &deliveries,
                        uint32_t b_lo = 0, uint32_t b_hi = UINT32_MAX, const modes_recovered *rec = nullptr,
                        const WeakList *weak = nullptr) {
    if (rec) walk_tiles<true>(st, cfg, cands, tiles, n_tiles, buffer_base, deliveries, b_lo, b_hi, rec, weak);
    else walk_tiles<false>(st, cfg, cands, tiles, n_tiles, buffer_base, deliveries, b_lo, b_hi, nullptr, nullptr);
}

// Build the delivered structs: in place and in parallel for array output, then the callback
// (if any) sequentially in stream order.
static void deliver(const std::vector<Delivery> &deliveries, MessageOut &out) {
    const size_t n = deliveries.size();
    size_t in_array = 0;
    if (out.array && out.count < out.capacity) {
        in_array = out.capacity - out.count < n ? out.capacity - out.count : n;
        modes_message *base = out.array + out.count;
        const Delivery *d = deliveries.data();
        BuildPool::get().run(in_array, [=](size_t b, size_t e) {
            for (size_t i = b; i < e; i++) {
                materialise(d[i], base + i);
            }
        });
    }
    if (out.sink) {
        for (size_t i = 0; i < n; i++) {
            if (i < in_array) { out.sink(out.user, out.array + out.count + i); continue; }
            modes_message tmp;
            materialise(deliveries[i], &tmp);
            out.sink(out.user, &tmp);
        }
    }
    out.count += n;
}

void deliver_gpu(const modes_delivery *d, size_t n, int64_t buffer_base, MessageOut &out) {
    auto build = [=](const modes_delivery &x, modes_message *mm) {
        const bool is_ap = (x.bits >> 16) & 1u;
        build_message(x.eval, (int)(x.bits & 1u), is_ap ? 0u : x.extra, is_ap ? x.extra : 0u, mm);
        mm->sample_pos = (buffer_base << 17) + x.t - MODES_CARRY_SAMPLES;
        mm->phase_corrected = (int)((x.bits >> 8) & 1u);
    };
    size_t in_array = 0;
    if (out.array && out.count < out.capacity) {
        in_array = out.capacity - out.count < n ? out.capacity - out.count : n;
        modes_message *base = out.array + out.count;
        BuildPool::get().run(in_array, [=](size_t b, size_t e) { for (size_t i = b; i < e; i++) build(d[i], base + i); });
    }
    if (out.sink) {
        for (size_t i = 0; i < n; i++) {
            if (i < in_array) { out.sink(out.user, out.array + out.count + i); continue; }
            modes_message tmp;
            build(d[i], &tmp);
            out.sink(out.user, &tmp);
        }
    }
    out.count += n;
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
struct Part {
    const modes_candidate *cands; const modes_tile *tiles; size_t n_tiles;   // the record array the part lies in
    size_t tile_lo;              // first tile that can hold one of its candidates
    uint32_t b_lo, b_hi;         // its buffers, as numbered in the records (t >> 17)
    int64_t buffer_base;
    bool first_of_shard;         // the tail pass for a shard's first part walks the previous SHARD's array
    const modes_recovered *rec;  // the array's recovery records, or nullptr
    const WeakList *weak;        // the array's weak positions, or nullptr
};
struct PartRun { ResolveState start, end; std::vector<Delivery> deliveries; };
struct ResolveScratch {
    std::vector<Delivery> deliveries;
    std::vector<PartRun> runs;   // kept between calls: delivery lists keep their capacity (growing them from nothing
                                 // in every call costs more in page faults, taken concurrently, than the verdicts)
    size_t n_runs_held = 0;      // > 0: a tentative resolve left its deliveries in runs[0 .. n_runs_held)
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

// Cut one record array into up to `want` parts at buffer boundaries.  The boundary of part k is
// read from the records themselves: the buffer after the one the first candidate at or behind tile
// k * n_tiles / want lies in (tiles do not line up with buffers; records are in stream order).
static void cut_parts(const modes_candidate *cands, const modes_tile *tiles, size_t n_tiles, int64_t buffer_base, size_t want,
                      std::vector<Part> &parts, const modes_recovered *rec = nullptr, const WeakList *weak = nullptr) {
    Part p{cands, tiles, n_tiles, 0, 0, UINT32_MAX, buffer_base, true, rec, weak};
    for (size_t k = 1; k < want; k++) {
        size_t ti = k * n_tiles / want;
        while (ti < n_tiles && tiles[ti].count == 0) ti++;
        if (ti >= n_tiles) break;
        const uint32_t b = (uint32_t)(cands[tiles[ti].offset].t >> 17) + 1;      // first buffer of the next part
        if (b <= p.b_lo) continue;                                                 // (a gap longer than a part)
        p.b_hi = b;
        parts.push_back(p);
        p.tile_lo = ti; p.b_lo = b; p.b_hi = UINT32_MAX; p.first_of_shard = false;
    }
    parts.push_back(p);
}

void add_recovery_stats(modes_recovery_stats &to, const modes_recovery_stats &from) {
    to.considered += from.considered; to.found += from.found; to.ambiguous += from.ambiguous;
    to.unknown_address += from.unknown_address; to.dropped += from.dropped; to.delivered += from.delivered;
}

// Judge the parts (rounds of guess and verify, see above); runs[k] receives part k's deliveries
// and statistics, `st` the state after the last part.
static int judge_parts(ResolveState &st, const ResolveConfig &cfg, const std::vector<Part> &parts, PartRun *runs) {
    const size_t n = parts.size();
    ResolveState blank;
    blank.reset();
    auto run_part = [&](size_t k, const ResolveState &from) {
        PartRun &r = runs[k];
        const Part &p = parts[k];
        r.start = from;
        std::memset(r.start.stats, 0, sizeof(r.start.stats));
        std::memset(&r.start.rstats, 0, sizeof(r.start.rstats));
        std::memset(&r.start.wstats, 0, sizeof(r.start.wstats));
        if (k) { r.start.cur_buffer = -1; r.start.next_j = 0; r.start.next_j_recovered = 0; }   // a part starts a buffer
        r.end = r.start;
        r.deliveries.clear();
        judge_tiles(r.end, cfg, p.cands, p.tiles + p.tile_lo, p.n_tiles - p.tile_lo, p.buffer_base, r.deliveries, p.b_lo, p.b_hi,
                    p.rec, p.weak);
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
            const Part &q = parts[k - 1];
            ResolveState g = st;
            g.cur_buffer = -1; g.next_j = 0; g.next_j_recovered = 0;   // (recovery never writes the cache: the guess skips it)
            const size_t end_tile = parts[k].first_of_shard ? q.n_tiles : (parts[k].tile_lo + 1 < q.n_tiles ? parts[k].tile_lo + 1 : q.n_tiles);
            const size_t len = end_tile - q.tile_lo;
            size_t tail = len / 16 > 128 ? len / 16 : 128;             // at least ~1 M samples (half a second of stream)
            if (tail > len) tail = len;
            runs[k].deliveries.clear();
            judge_tiles(g, cfg, q.cands, q.tiles + (end_tile - tail), q.n_tiles - (end_tile - tail), q.buffer_base, runs[k].deliveries,
                        q.b_lo, q.b_hi);
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
    for (size_t k = 0; k < n; k++) {
        for (int i = 0; i < 8; i++) st.stats[i] += runs[k].end.stats[i];
        add_recovery_stats(st.rstats, runs[k].end.rstats);
        add_recovery_stats(st.wstats, runs[k].end.wstats);
    }
    if (n) {
        std::memcpy(st.icao, runs[n - 1].end.icao, sizeof(st.icao));
        // the skip state is that of the last part that saw a candidate (an empty part leaves none)
        for (size_t k = n; k-- > 0;)
            if (runs[k].end.cur_buffer != -1 || k == 0) {
                st.cur_buffer = runs[k].end.cur_buffer; st.next_j = runs[k].end.next_j;
                st.next_j_recovered = runs[k].end.next_j_recovered;
                break;
            }
    }
    return rounds;
}

static PartRun *runs_for(ResolveScratch *scratch, size_t n) {
    if (scratch->runs.size() < n) scratch->runs.resize(n);
    return scratch->runs.data();
}

void resolve_candidates(ResolveState &st, const ResolveConfig &cfg, const modes_candidate *cands,
                        const modes_tile *tiles, size_t n_tiles, int64_t buffer_base, MessageOut &out,
                        ResolveScratch *scratch, const modes_recovered *recovered, const WeakList &weak) {
    const bool timing = std::getenv("MODES_RESOLVE_TIMING") != nullptr;
    auto now = [] { return std::chrono::steady_clock::now(); };
    auto ms = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) {
        return std::chrono::duration<double, std::milli>(b - a).count(); };
    const auto t0 = now();
    scratch->n_runs_held = 0;
    const size_t want = parts_for(n_tiles);
    if (want <= 1) {
        std::vector<Delivery> &deliveries = scratch->deliveries;
        deliveries.clear();
        judge_tiles(st, cfg, cands, tiles, n_tiles, buffer_base, deliveries, 0, UINT32_MAX, recovered, &weak);
        const auto t1 = now();
        deliver(deliveries, out);
        if (timing) std::fprintf(stderr, "resolve_candidates: %zu tiles, verdicts %.2f ms, structs %.2f ms\n", n_tiles, ms(t0, t1), ms(t1, now()));
        return;
    }
    std::vector<Part> parts;
    cut_parts(cands, tiles, n_tiles, buffer_base, want, parts, recovered, &weak);
    PartRun *runs = runs_for(scratch, parts.size());
    const int rounds = judge_parts(st, cfg, parts, runs);
    const auto t1 = now();
    for (size_t k = 0; k < parts.size(); k++) deliver(runs[k].deliveries, out);
    if (timing)
        std::fprintf(stderr, "resolve_candidates: %zu tiles in %zu parts, %d rounds, verdicts %.2f ms, structs %.2f ms\n", n_tiles,
                     parts.size(), rounds, ms(t0, t1), ms(t1, now()));
}

void resolve_tentative(ResolveState &st, const ResolveConfig &cfg, const modes_candidate *cands, const modes_tile *tiles,
                       size_t n_tiles, int64_t buffer_base, ResolveScratch *scratch) {
    scratch->deliveries.clear();
    scratch->n_runs_held = 0;
    const size_t want = parts_for(n_tiles);
    if (want <= 1) {
        judge_tiles(st, cfg, cands, tiles, n_tiles, buffer_base, scratch->deliveries);
        return;
    }
    std::vector<Part> parts;
    cut_parts(cands, tiles, n_tiles, buffer_base, want, parts);
    judge_parts(st, cfg, parts, runs_for(scratch, parts.size()));
    scratch->n_runs_held = parts.size();
}

void resolve_commit(MessageOut &out, ResolveScratch *scratch) {
    if (scratch->n_runs_held) {
        for (size_t k = 0; k < scratch->n_runs_held; k++) { deliver(scratch->runs[k].deliveries, out); scratch->runs[k].deliveries.clear(); }
        scratch->n_runs_held = 0;
        return;
    }
    deliver(scratch->deliveries, out);
    scratch->deliveries.clear();
}

// Several shards of one stream (e.g. one per GPU), resolved concurrently and exactly: every shard
// is a part, long shards are cut once more (see judge_parts).
void resolve_shards(ResolveState &st, const ResolveConfig &cfg, size_t n_shards, const modes_candidate *const *cands,
                    const modes_tile *const *tiles, const size_t *n_tiles, const int64_t *buffer_base,
                    MessageOut &out, ResolveScratch *scratch, const modes_recovered *const *recovered, const WeakList *weak) {
    const bool timing = std::getenv("MODES_RESOLVE_TIMING") != nullptr;
    auto now = [] { return std::chrono::steady_clock::now(); };
    auto t_start = now();
    scratch->n_runs_held = 0;
    std::vector<Part> parts;
    size_t threads_left = parts_for((size_t)-1);
    for (size_t k = 0; k < n_shards; k++) {
        size_t want = parts_for(n_tiles[k]);
        const size_t share = threads_left / (n_shards - k) > 0 ? threads_left / (n_shards - k) : 1;
        if (want > share) want = share;
        cut_parts(cands[k], tiles[k], n_tiles[k], buffer_base[k], want, parts, recovered ? recovered[k] : nullptr,
                  recovered && weak ? weak + k : nullptr);
        threads_left = threads_left > want ? threads_left - want : 0;
    }
    PartRun *runs = runs_for(scratch, parts.size());
    const int rounds = judge_parts(st, cfg, parts, runs);
    auto t_judged = now();
    for (size_t k = 0; k < parts.size(); k++) deliver(runs[k].deliveries, out);
    if (timing)
        std::fprintf(stderr, "resolve_shards: %zu shards in %zu parts, %d rounds, verdicts %.2f ms, structs %.2f ms\n", n_shards,
                     parts.size(), rounds, std::chrono::duration<double, std::milli>(t_judged - t_start).count(),
                     std::chrono::duration<double, std::milli>(now() - t_judged).count());
}

}  // namespace modes
