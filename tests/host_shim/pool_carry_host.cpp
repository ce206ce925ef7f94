// TEST INFRASTRUCTURE — not part of the product.
// Host build of modes::input::convert_samples (dump1090_b200/csrc/modes_input_core.cuh), the conversion
// the receiver pool makes of a 2 MHz 16-bit receiver's carry on the host, so that the CPU test suite can
// check it against the numpy model of the definition (tests/test_pool_input_format.py).
#include <cstddef>
#include <cstdint>
#include "modes_input_core.cuh"

extern "C" int shim_pool_convert_samples(const uint8_t *in, size_t n, int shift, uint8_t *out) {
    if (shift < 0 || shift > modes::input::kMaxShift) return -1;
    modes::input::convert_samples(in, (int64_t)n, shift, out);
    return 0;
}
