// TEST INFRASTRUCTURE — not part of the product.
// Host build of the input spectrum arithmetic (dump1090_b200/csrc/modes_spectrum_core.cuh), so that the CPU
// test suite can check it against the numpy model of the definition (tests/spectrum_model.py).
#include <cstddef>
#include <cstdint>
#include "modes_spectrum_core.cuh"

namespace SP = modes::spectrum;

extern "C" {

// n frames of 256 UC8 pairs at iq -> their power, 256 bins each in record order, at out.
int shim_frame_power(const uint8_t *iq, size_t n, uint32_t *out) {
    for (size_t f = 0; f < n; f++) SP::frame_power(iq + 2 * SP::kN * f, out + SP::kN * f);
    return 0;
}

// s_b and F of buffer b at the ratio out : in, and the launch bound on F.
int shim_geometry(int out, int in, int64_t b, int64_t *first, uint32_t *frames, uint32_t *max_frames) {
    *first = SP::first_sample(out, in, b);
    *frames = SP::frames(out, in, b);
    *max_frames = SP::max_frames(out, in);
    return 0;
}

}
