// TEST INFRASTRUCTURE — not part of the product.
// Host build of dump1090_b200/csrc/modes_levels_core.cuh (magnitude, sums, peak and clip count of a
// buffer, as the level pass computes them), so that the CPU test suite can check it against a plain
// restatement of the definition.
#include <cstring>
#include <vector>
#include "modes_internal.h"
#include "modes_levels_core.cuh"

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

// iq: nbytes (a multiple of 16) of I/Q bytes, split over `threads` partial sums the way the kernel
// splits a buffer (thread t takes the 16-byte words t, t + threads, ...).
// out: sum_mag, sum_power, peak, clipped.
extern "C" int shim_levels(const uint8_t *iq, size_t nbytes, uint32_t threads, uint64_t out[4]) {
    if (nbytes % 16 || !threads) return -1;
    const size_t nvec = nbytes / 16;
    uint64_t mag = 0, pw = 0, peak = 0, clip = 0;
    for (uint32_t t = 0; t < threads; t++) {
        modes::levels::Acc a;
        modes::levels::acc_clear(a);
        for (size_t v = t; v < nvec; v += threads) {
            uint32_t w[4];
            std::memcpy(w, iq + 16 * v, 16);
            modes::levels::add_quad(a, w[0], w[1], w[2], w[3], lutn().data());
        }
        mag += a.sum_mag; pw += a.sum_power; clip += a.clipped;
        if (a.peak > peak) peak = a.peak;
    }
    out[0] = mag; out[1] = pw; out[2] = peak; out[3] = clip;
    return 0;
}
