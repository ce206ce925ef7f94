// TEST INFRASTRUCTURE — not part of the product.
// Host build of the integer decimator and the input-rate descriptor of
// dump1090_b200/csrc/modes_resample_core.cuh, so that the CPU test suite can check them against the numpy
// model of the definition (tests/decimate_model.py).
#include <cstddef>
#include <cstdint>
#include "modes_input_core.cuh"
#include "modes_resample_core.cuh"

namespace D = modes::decimate;

// Input sample s of the stream as its UC8 pair, with in[0] the first byte of input sample in_first: UC8
// (shift < 0, a trailing odd byte an I whose Q is 127) or int16 converted with the shift (a trailing
// partial sample not in the span); no signal outside the span.
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

template <int M>
static void run(const uint8_t *in, size_t in_bytes, int64_t in_first, int64_t out_first, size_t count,
                int64_t out_end, int shift, uint8_t *out) {
    for (size_t i = 0; i < count;) {
        const int64_t n = out_first + (int64_t)i;
        const int64_t g = modes::resample::floor_div(n, 8);
        uint32_t w[D::group_words(M) + 1] = {};
        for (int j = 0; j < D::group_in(M); j++)
            w[j >> 1] |= sample_at(in, in_bytes, in_first, 8 * M * g - D::extent(M) + j, shift) << (16 * (j & 1));
        uint32_t y[4];
        D::group<M>(w, y);
        for (int r = (int)(n - 8 * g); r < 8 && i < count; r++, i++) {
            const uint32_t v = (out_first + (int64_t)i >= out_end) ? 0x7f7fu : (y[r >> 1] >> (16 * (r & 1))) & 0xffffu;
            out[2 * i] = (uint8_t)v;
            out[2 * i + 1] = (uint8_t)(v >> 8);
        }
    }
}

// Output samples [out_first, out_first + count) of decimation by m as I/Q bytes into out, one group of 8 at
// a time as the kernel computes them; samples at or past out_end are 127.
extern "C" int shim_decimate(int m, const uint8_t *in, size_t in_bytes, int64_t in_first, int64_t out_first,
                             size_t count, int64_t out_end, int shift, uint8_t *out) {
    switch (m) {
    case 2: run<2>(in, in_bytes, in_first, out_first, count, out_end, shift, out); return 0;
    case 3: run<3>(in, in_bytes, in_first, out_first, count, out_end, shift, out); return 0;
    case 4: run<4>(in, in_bytes, in_first, out_first, count, out_end, shift, out); return 0;
    case 5: run<5>(in, in_bytes, in_first, out_first, count, out_end, shift, out); return 0;
    }
    return -1;
}

// M's table: returns T.
extern "C" int shim_decimate_taps(int m, int16_t *out, int cap) {
    if (m < 2 || m > 5 || cap < D::taps(m)) return -1;
    for (int k = 0; k < D::taps(m); k++) out[k] = (int16_t)D::tap(m, k);
    return D::taps(m);
}

// The descriptor of hz: {out, in, lead, taps, carry, m}, or -1 for a rate the decoder does not take.
extern "C" int shim_input_rate(uint32_t hz, int32_t *out6) {
    const modes::InputRate *r = modes::find_input_rate(hz);
    if (!r) return -1;
    const int32_t v[6] = {r->out, r->in, r->lead, r->taps, r->carry, r->m};
    for (int k = 0; k < 6; k++) out6[k] = v[k];
    return 0;
}

// The input reach of output sample n and the output count of n_in input samples at hz.
extern "C" int shim_input_reach(uint32_t hz, int64_t n, int64_t n_in, int64_t *out3) {
    const modes::InputRate *r = modes::find_input_rate(hz);
    if (!r) return -1;
    out3[0] = modes::in_lo(*r, n);
    out3[1] = modes::in_hi(*r, n);
    out3[2] = modes::n_out(*r, n_in);
    return 0;
}
