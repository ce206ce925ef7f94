// TEST INFRASTRUCTURE — not part of the product.
// Host build of dump1090_b200/csrc/modes_signal_core.cuh (magnitude -> pulse -> sums -> integer square
// root, as the signal pass computes them), so that the CPU test suite can check it against a plain
// restatement of the definition.
#include <cstring>
#include <vector>
#include "modes_internal.h"
#include "modes_signal_core.cuh"

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

// iq: the window's 2 * bits samples (the pairs of bits 0 .. bits-1) as I/Q bytes.
extern "C" uint32_t shim_signal_window(const uint8_t *iq, uint32_t bits) {
    uint64_t sum = 0;
    for (uint32_t b = 0; b < bits; b++) {
        uint32_t pair;
        std::memcpy(&pair, iq + 4 * b, 4);
        sum += modes::signal::pulse_sq(pair, lutn().data());
    }
    return modes::signal::signal_of(sum, bits);
}

extern "C" uint32_t shim_signal_of(uint64_t sum_sq, uint32_t bits) { return modes::signal::signal_of(sum_sq, bits); }
