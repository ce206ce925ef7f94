// TEST INFRASTRUCTURE — not part of the product.
// Host build of dump1090_b200/csrc/modes_input_core.cuh (the 16-bit input formats' conversion to UC8),
// so that the CPU test suite can check it against the numpy model of the definition.
#include <cstddef>
#include <cstdint>
#include <cstring>
#include "modes_input_core.cuh"

namespace I = modes::input;

// n whole samples (4 bytes each) of a 16-bit stream to their 2 n UC8 bytes, a sample at a time as the
// kernels convert them.
extern "C" int shim_input_convert(const uint8_t *in, size_t n, int shift, uint8_t *out) {
    if (shift < 0 || shift > I::kMaxShift) return -1;
    for (size_t k = 0; k < n; k++) {
        uint32_t w;
        memcpy(&w, in + 4 * k, 4);
        const uint32_t y = I::convert_pair(w, shift);
        out[2 * k] = (uint8_t)y;
        out[2 * k + 1] = (uint8_t)(y >> 8);
    }
    return 0;
}

// The format's bytes per sample and default shift; -1 for an unknown format.
extern "C" int shim_input_format(uint32_t format, int *sample_bytes, int *default_shift) {
    if (!I::known(format)) return -1;
    *sample_bytes = I::sample_bytes(format);
    *default_shift = I::default_shift(format);
    return 0;
}
