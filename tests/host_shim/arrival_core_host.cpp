// TEST INFRASTRUCTURE — not part of the product.
// Host build of dump1090_b200/csrc/modes_arrival_core.cuh (frame bits -> class masks -> class sums and
// counts -> code, as the arrival pass computes them), so that the CPU test suite can check it against
// a plain restatement of the definition.
#include <cstring>
#include <vector>
#include "modes_internal.h"
#include "modes_signal_core.cuh"
#include "modes_arrival_core.cuh"

namespace {
const std::vector<uint16_t> &lutn() {
    static const std::vector<uint16_t> t = [] {
        std::vector<uint16_t> v(modes::kNLutEntries);
        modes::build_lutn(v.data());
        return v;
    }();
    return t;
}
}  // namespace

// iq: window samples 0 .. 16+2b as I/Q bytes; msg16: the attempt's 14 frame bytes and the two bytes
// that follow them in its record (msgtype, flags); bits: 56 or 112.
extern "C" uint32_t shim_arrival_window(const uint8_t *iq, const uint8_t *msg16, uint32_t bits) {
    using namespace modes::arrival;
    uint32_t m[17 + 2 * 112];
    for (uint32_t s = 0; s < 17 + 2 * bits; s++) {
        uint16_t sample;
        std::memcpy(&sample, iq + 2 * s, 2);
        uint32_t second;
        modes::signal::pair_mags(sample | 0x7f7f0000u, lutn().data(), m[s], second);
    }
    uint32_t mw[4], B[4];
    std::memcpy(mw, msg16, 16);
    bit_words(mw, bits, B);
    uint32_t S[4] = {0, 0, 0, 0};
    for (int r = 0; r < 4; r++) {
        const PairClasses c = pair_classes(B, r, bits);
        for (int l = 0; l < 32; l++) {
            const uint32_t i = 32 * r + l;
            if (i >= bits) break;
            if ((c.main1 >> l) & 1u) S[kMain] += m[16 + 2 * i];
            if ((c.early1 >> l) & 1u) S[kEarly] += m[16 + 2 * i];
            if ((c.main2 >> l) & 1u) S[kMain] += m[17 + 2 * i];
            if ((c.late2 >> l) & 1u) S[kLate] += m[17 + 2 * i];
        }
    }
    const uint32_t bit0 = B[0] & 1u, last = (B[(bits - 1) >> 5] >> ((bits - 1) & 31)) & 1u;
    for (uint32_t s = 1; s <= 16 + 2 * bits; s = (s == 15 ? 16 + 2 * bits : s + 1)) {
        const uint32_t cls = edge_class(s, bits, bit0, last);
        if (cls < 4) S[cls] += m[s];
    }
    uint32_t n[4];
    class_counts(B, bits, n);
    return code_of(S, n);
}

extern "C" uint32_t shim_code_of(const uint32_t *S, const uint32_t *n) { return modes::arrival::code_of(S, n); }

extern "C" void shim_class_counts(const uint8_t *msg16, uint32_t bits, uint32_t *n) {
    uint32_t mw[4], B[4];
    std::memcpy(mw, msg16, 16);
    modes::arrival::bit_words(mw, bits, B);
    modes::arrival::class_counts(B, bits, n);
}
