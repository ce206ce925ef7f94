// TEST INFRASTRUCTURE — not part of the product.
// Host build of dump1090_b200/csrc/modes_resample_core.cuh (the 2.4 MS/s -> 2 MHz polyphase
// arithmetic), so that the CPU test suite can check it against the numpy model of the definition.
#include <cstddef>
#include <cstdint>
#include "modes_resample_core.cuh"

namespace R = modes::resample;

// The input byte at stream byte position p, with in[0] at stream byte 2 * in_first and in_bytes of them:
// no signal (127) outside.
static int byte_at(const uint8_t *in, size_t in_bytes, int64_t in_first, int64_t p) {
    const int64_t j = p - 2 * in_first;
    return (j >= 0 && j < (int64_t)in_bytes) ? in[j] : 127;
}

// Output samples [out_first, out_first + count) as I/Q bytes into out, one polyphase period at a time as
// the kernel computes them; samples at or past out_end are 127.
extern "C" int shim_resample(const uint8_t *in, size_t in_bytes, int64_t in_first, int64_t out_first, size_t count,
                             int64_t out_end, uint8_t *out) {
    for (size_t i = 0; i < count;) {
        const int64_t n = out_first + (int64_t)i;
        const int64_t q = R::floor_div(n, 5);
        int xi[R::kPeriodIn], xq[R::kPeriodIn];
        for (int k = 0; k < R::kPeriodIn; k++) {
            const int64_t s = 6 * q - R::kLead + k;
            xi[k] = byte_at(in, in_bytes, in_first, 2 * s) - 127;
            xq[k] = byte_at(in, in_bytes, in_first, 2 * s + 1) - 127;
        }
        uint32_t y[5];
        R::period(xi, xq, y);
        for (int r = (int)(n - 5 * q); r < 5 && i < count; r++, i++) {
            const uint32_t v = (out_first + (int64_t)i >= out_end) ? 0x7f7fu : y[r];
            out[2 * i] = (uint8_t)v;
            out[2 * i + 1] = (uint8_t)(v >> 8);
        }
    }
    return 0;
}

// The tap table, row by row.
extern "C" int shim_resample_taps(int16_t *out, int cap) {
    if (cap < 5 * R::kTaps) return -1;
    for (int r = 0; r < 5; r++)
        for (int k = 0; k < R::kTaps; k++) out[r * R::kTaps + k] = (int16_t)R::tap(r, k);
    return R::kTaps;
}
