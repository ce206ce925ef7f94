// TEST INFRASTRUCTURE — not part of the product.
// Host run of the algorithm the device resolve executes (dump1090_b200/csrc/modes_resolve_gpu.cu):
// every reference buffer is replayed on its own from a guessed address cache
// (modes_resolve_core.cuh), the caches are handed from buffer to buffer (last writer of a slot
// wins), and a buffer whose guess was wrong in a slot it read before writing is replayed again.
// With max_rounds > 0 that is done at most max_rounds times, as on the device; if the caches have
// not settled by then, every buffer is replayed once more in stream order from the starting cache
// (the device's fallback) and a last hand-over checks that nothing changes.  max_rounds <= 0
// repeats until nothing changes.  The CPU tests compare the outcome with the host resolver.
#include <cstring>
#include <vector>
#include "modes_resolve_core.cuh"

namespace {
struct TrackCache {
    uint32_t *c; uint32_t written[32], readfirst[32];
    uint32_t read(uint32_t s) { if (!((written[s >> 5] >> (s & 31)) & 1u)) readfirst[s >> 5] |= 1u << (s & 31); return c[s]; }
    void write(uint32_t s, uint32_t a) { c[s] = a; written[s >> 5] |= 1u << (s & 31); }
};
struct Out { int64_t t; int pass; modes::rcore::Decision d; };
}

struct shim_delivery { int64_t t; int32_t pass, crcok, phase_corrected, extra, extra_is_ap, pad; };

// Returns the number of deliveries; -2: the rounds did not settle within the number of buffers
// (+2), -3: the hand-over after the fallback still found a wrong cache.  *rounds_out = the guessed
// rounds run, *fallback_out = 1 when the in-order replay was needed.
extern "C" long shim_resolve_buffers(const modes_candidate *cands, const modes_tile *tiles, size_t n_tiles, size_t n_buffers,
                                     int check_crc, const uint32_t *start_cache, shim_delivery *out, size_t cap,
                                     int64_t stats[8], uint32_t *end_cache, int *rounds_out, int tile_samples,
                                     int max_rounds, int *fallback_out) {
    using namespace modes::rcore;
    const size_t B = n_buffers;
    std::vector<std::vector<uint32_t>> C(B, std::vector<uint32_t>(start_cache, start_cache + 1024)), E(B, std::vector<uint32_t>(1024));
    std::vector<std::vector<Out>> deliv(B);
    std::vector<BufferState> st(B);
    std::vector<TrackCache> tc(B);
    std::vector<char> rerun(B, 1);

    auto replay = [&](size_t b) {                     // buffer b from the cache C[b]; its end cache in E[b]
        E[b] = C[b];
        TrackCache &k = tc[b];
        k.c = E[b].data(); std::memset(k.written, 0, sizeof(k.written)); std::memset(k.readfirst, 0, sizeof(k.readfirst));
        std::memset(&st[b], 0, sizeof(st[b]));
        deliv[b].clear();
        const uint64_t v_lo = (uint64_t)b * 131072 + 2, v_hi = (uint64_t)(b + 1) * 131072 + 1;
        size_t t_lo = v_lo / tile_samples, t_hi = v_hi / tile_samples;
        if (t_hi >= n_tiles) t_hi = n_tiles - 1;
        for (size_t ti = t_lo; ti <= t_hi && ti < n_tiles; ti++)
            for (uint32_t i = 0; i < tiles[ti].count; i++) {
                const modes_candidate &c = cands[tiles[ti].offset + i];
                if ((uint64_t)(c.t >> 17) != b) continue;
                Decision d[2];
                candidate(st[b], k, (uint32_t)(c.t & 131071), attempt_of(c.pass[0]), attempt_of(c.pass[1]), check_crc, d);
                for (int p = 0; p < 2; p++) if (d[p].deliver) deliv[b].push_back(Out{c.t, p, d[p]});
            }
        rerun[b] = 0;
    };
    // hand the caches on: slot by slot, the last writer among the earlier buffers; true if a
    // buffer's guess was wrong in a slot it read before writing
    auto handover = [&]() {
        std::vector<uint32_t> cur(start_cache, start_cache + 1024);
        bool more = false;
        for (size_t b = 0; b < B; b++) {
            bool again = false;
            for (uint32_t s = 0; s < 1024; s++) {
                if (cur[s] != C[b][s] && ((tc[b].readfirst[s >> 5] >> (s & 31)) & 1u)) again = true;
                C[b][s] = cur[s];
            }
            rerun[b] = again;
            more |= again;
            for (uint32_t s = 0; s < 1024; s++)
                if ((tc[b].written[s >> 5] >> (s & 31)) & 1u) cur[s] = E[b][s];
        }
        std::memcpy(end_cache, cur.data(), 4096);
        return more;
    };

    int rounds = 0;
    bool more = B > 0;
    if (B == 0) std::memcpy(end_cache, start_cache, 4096);
    while (more && (max_rounds <= 0 || rounds < max_rounds)) {
        for (size_t b = 0; b < B; b++)
            if (rerun[b]) replay(b);
        rounds++;
        more = handover();
        if (rounds > (int)B + 2) return -2;
    }
    *fallback_out = more;
    if (more) {                                       // the fallback: stream order from the starting cache
        std::vector<uint32_t> cur(start_cache, start_cache + 1024);
        for (size_t b = 0; b < B; b++) {
            C[b] = cur;
            replay(b);
            cur = E[b];
        }
        if (handover()) return -3;
    }
    std::memset(stats, 0, 8 * sizeof(int64_t));
    size_t n = 0;
    for (size_t b = 0; b < B; b++) {
        for (int i = 0; i < 8; i++) stats[i] += st[b].stats[i];
        for (const Out &o : deliv[b]) {
            if (n < cap) out[n] = shim_delivery{o.t, o.pass, (int32_t)o.d.crcok, (int32_t)o.d.phase_corrected, (int32_t)o.d.extra, (int32_t)o.d.extra_is_ap, 0};
            n++;
        }
    }
    *rounds_out = rounds;
    return (long)n;
}
