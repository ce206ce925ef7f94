// TEST INFRASTRUCTURE — not part of the product.
// Host build of dump1090_b200/csrc/modes_recover_core.cuh: the recovery record of a window computed
// with the same per-bit keys, per-part search and record packing as modes_recover.cu, the warp's
// ballots and reductions replaced by loops, so that the CPU test suite can check the arithmetic
// against a numpy restatement of the definition.
#include <algorithm>
#include <cstring>
#include <vector>
#include "modes_internal.h"
#include "modes_recover_core.cuh"
#include "modes_signal_core.cuh"

namespace {
struct Tables {
    std::vector<uint16_t> lutn;
    uint32_t bit_syn[112];
    Tables() : lutn(modes::kNLutEntries) {
        modes::build_lutn(lutn.data());
        modes::build_bit_syndromes(bit_syn);
    }
};
const Tables &tables() {
    static const Tables t;
    return t;
}

void recover_window(const uint8_t *iq, uint8_t rec[20]) {
    using namespace modes;
    const Tables &T = tables();
    uint32_t frame[4] = {0, 0, 0, 0}, syn = 0;
    uint64_t sq = 0;
    std::vector<uint32_t> keys;
    for (uint32_t i = 0; i < 112; i++) {
        uint32_t pair, a, c;
        std::memcpy(&pair, iq + 4 * i, 4);
        signal::pair_mags(pair, T.lutn.data(), a, c);
        if (a > c) { frame[i >> 5] |= 0x80000000u >> (i & 31); syn ^= T.bit_syn[i]; }
        const uint32_t k = recover::bit_key(a, c, i);
        if (k != recover::kNoKey) keys.push_back(k);
        const uint32_t p = a > c ? a : c;
        sq += (uint64_t)p * p;
    }
    uint32_t status = MODES_RECOVER_INELIGIBLE, nflips = 0;
    const uint32_t df = frame[0] >> 27;
    if (df == 17 || df == 18) {
        std::sort(keys.begin(), keys.end());
        uint32_t pos[recover::kBits], s[recover::kBits];
        for (int k = 0; k < recover::kBits; k++) { pos[k] = keys[k] & 127u; s[k] = T.bit_syn[pos[k]]; }
        uint32_t minw = recover::kNoSolution, count = 0, mask = 0;
        for (uint32_t hi = 0; hi < 32; hi++) {
            const recover::Part p = recover::search_part(hi, s, syn);
            if (p.minw < minw) { minw = p.minw; count = p.count; mask = p.mask; }
            else if (p.minw == minw && p.minw != recover::kNoSolution) count += p.count;
        }
        status = recover::status_of(minw, count);
        if (status == MODES_RECOVER_FOUND) {
            for (int k = 0; k < recover::kBits; k++)
                if ((mask >> k) & 1u) frame[pos[k] >> 5] ^= 0x80000000u >> (pos[k] & 31u);
            nflips = (uint32_t)__builtin_popcount(mask);
        } else if (status == MODES_RECOVER_AMBIGUOUS) {
            nflips = minw;
        }
    }
    uint32_t w[5];
    recover::record_words(frame, status, nflips, signal::signal_of(sq, 112), w);
    std::memcpy(rec, w, 20);
}
}  // namespace

// iq: n windows of 112 sample pairs (448 bytes each: the samples m[j+16 .. j+239] of a candidate);
// out: n records of 20 bytes.
extern "C" int shim_recover(const uint8_t *iq, size_t n, uint8_t *out) {
    for (size_t k = 0; k < n; k++) recover_window(iq + 448 * k, out + 20 * k);
    return 0;
}
