// TEST INFRASTRUCTURE — not part of the product.
// Host build of dump1090_b200/csrc/modes_weak_core.cuh: the weak-preamble test of a window of raw I/Q
// samples with the same magnitude words and conditions as modes_weak.cu, so that the CPU test suite
// can check the arithmetic against a numpy restatement of the definition.
#include <cstring>
#include <vector>
#include "modes_internal.h"
#include "modes_weak_core.cuh"

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

// iq: n windows of weak::kWindow samples (I/Q byte pairs, the samples m[j .. j+25] of a position);
// out[k]: bit 0 = weak preamble, bit 1 = conditions 1 and 2, bit 2 = the reference's preamble test.
extern "C" int shim_weak(const uint8_t *iq, size_t n, uint8_t *out) {
    using namespace modes;
    for (size_t k = 0; k < n; k++) {
        uint16_t m[weak::kWindow];
        for (int w = 0; w < weak::kWindow / 2; w++) {
            uint32_t word;
            std::memcpy(&word, iq + 2 * weak::kWindow * k + 4 * w, 4);
            const uint32_t pair = weak::word_mags(word, lutn().data());
            m[2 * w] = (uint16_t)(pair & 0xffffu);
            m[2 * w + 1] = (uint16_t)(pair >> 16);
        }
        out[k] = (uint8_t)((weak::weak_preamble(m, 0) ? 1 : 0) | (weak::shape_and_contrast(m, 0) ? 2 : 0) |
                           (weak::reference_preamble(m, 0) ? 4 : 0));
    }
    return 0;
}
