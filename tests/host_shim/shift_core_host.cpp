// TEST INFRASTRUCTURE — not part of the product.
// Host build of the frequency shift in front of the integer decimator (shift:: in
// dump1090_b200/csrc/modes_resample_core.cuh), so that the CPU test suite can check it against the numpy
// model of the definition (tests/shift_model.py).
#include <cstddef>
#include <cstdint>
#include "modes_input_core.cuh"
#include "modes_resample_core.cuh"

namespace D = modes::decimate;
namespace S = modes::shift;

// Input sample s of the stream as its UC8 pair (decimate_core_host.cpp's rule): UC8 (shift < 0) or int16
// converted with the shift; no signal outside the span.
static uint32_t sample_at(const uint8_t *in, size_t in_bytes, int64_t in_first, int64_t s, int shift) {
    const int64_t j = s - in_first;
    if (shift < 0) {
        const int64_t b = 2 * j;
        if (b < 0 || b >= (int64_t)in_bytes) return 0x7f7fu;
        return in[b] | (uint32_t)(b + 1 < (int64_t)in_bytes ? in[b + 1] : 127) << 8;
    }
    const int64_t b = 4 * j;
    if (b < 0 || b + 4 > (int64_t)(in_bytes & ~(size_t)3)) return 0x7f7fu;
    return modes::input::convert_pair((uint32_t)in[b] | (uint32_t)in[b + 1] << 8 | (uint32_t)in[b + 2] << 16 |
                                          (uint32_t)in[b + 3] << 24, shift);
}

// The kernel's shared-memory table: rotation(C[k], S[k]) at k.
static const uint32_t *table() {
    static uint32_t tab[S::kPhases];
    static bool built = false;
    if (!built) {
        for (int k = 0; k < S::kPhases; k++) tab[k] = S::rotation(S::kCos[k], S::kSin[k]);
        built = true;
    }
    return tab;
}

template <int M>
static void run(const uint8_t *in, size_t in_bytes, int64_t in_first, int64_t out_first, size_t count,
                int64_t out_end, int shift, uint32_t step, uint8_t *out) {
    for (size_t i = 0; i < count;) {
        const int64_t n = out_first + (int64_t)i;
        const int64_t g = modes::resample::floor_div(n, 8);
        const int64_t m0 = 8 * M * g - D::extent(M);
        uint32_t w[D::group_words(M) + 1] = {};
        for (int j = 0; j < D::group_in(M); j++)
            w[j >> 1] |= sample_at(in, in_bytes, in_first, m0 + j, shift) << (16 * (j & 1));
        uint32_t y[4];
        S::shift_group<M>(w, table(), (uint32_t)m0 * step, step, y);
        for (int r = (int)(n - 8 * g); r < 8 && i < count; r++, i++) {
            const uint32_t v = (out_first + (int64_t)i >= out_end) ? 0x7f7fu : (y[r >> 1] >> (16 * (r & 1))) & 0xffffu;
            out[2 * i] = (uint8_t)v;
            out[2 * i + 1] = (uint8_t)(v >> 8);
        }
    }
}

// Output samples [out_first, out_first + count) of the shifted decimation by m with the given step, as the
// kernel computes them one group of 8 at a time; samples at or past out_end are 127.
extern "C" int shim_shift_decimate(int m, const uint8_t *in, size_t in_bytes, int64_t in_first, int64_t out_first,
                                   size_t count, int64_t out_end, int shift, uint32_t step, uint8_t *out) {
    switch (m) {
    case 2: run<2>(in, in_bytes, in_first, out_first, count, out_end, shift, step, out); return 0;
    case 3: run<3>(in, in_bytes, in_first, out_first, count, out_end, shift, step, out); return 0;
    case 4: run<4>(in, in_bytes, in_first, out_first, count, out_end, shift, step, out); return 0;
    case 5: run<5>(in, in_bytes, in_first, out_first, count, out_end, shift, step, out); return 0;
    }
    return -1;
}

// The header's C and S.
extern "C" void shim_shift_tables(int16_t *c, int16_t *s) {
    for (int k = 0; k < S::kPhases; k++) {
        c[k] = S::kCos[k];
        s[k] = S::kSin[k];
    }
}

extern "C" uint32_t shim_shift_step(int32_t offset_hz, uint32_t fs) { return S::step(offset_hz, fs); }

// The largest offset hz takes, or -1 for a rate the decoder does not take; offset_fits at offset_hz in *fits.
extern "C" int32_t shim_shift_max_offset(uint32_t hz, int32_t offset_hz, int32_t *fits) {
    const modes::InputRate *r = modes::find_input_rate(hz);
    if (!r) return -1;
    *fits = modes::offset_fits(*r, offset_hz);
    return modes::max_offset(*r);
}
