// modes_spectrum_core.cuh — the arithmetic of the input spectrum pass (modes_set_spectrum; K13 in
// modes_spectrum.cu): an exact integer power spectrum of the input each reference buffer stands for.
//
// Reference buffer b (2 MHz samples [b B, (b + 1) B), B = MODES_BUFFER_SAMPLES) stands for the input samples
// [s_b, s_{b+1}), s_b = floor(in b B / out) with (out, in) the rate's ratio (InputRate: 1:1 at 2 MHz, 5:6 at
// 2.4 MS/s, 1:M at 2 M MS/s).  Its F = floor((s_{b+1} - s_b) / N) whole frames of N = 256 input samples start
// at s_b, s_b + N, ...; the remainder is not measured.  A sample is xi = I - 127, xq = Q - 127 of the UC8
// bytes (16-bit input after its conversion, modes_input_core.cuh; 0 past the stream's end), without the
// input offset.  Per frame, in int32 with arithmetic shifts:
//   window   v[n] = (x[n] w[n] + 8192) >> 14,  w[n] = (16384 - C[4 n]) >> 1   (a periodic Hann, Q14)
//   FFT      radix-2 decimation in time, in place on the bit-reversed frame, no scaling; the butterfly of
//            stage s (half = 2^s, s = 0..7) on a = X[i], b = X[i + half], j = i mod half, k = j 2^(7-s):
//                t_re = (b_re c + b_im s + 8192) >> 14,   t_im = (b_im c - b_re s + 8192) >> 14
//                X[i] = a + t,  X[i + half] = a - t
//            with c = C[4 k], s = S[4 k] (the 1024-phase Q14 tables of modes_resample_core.cuh), i.e.
//            t = b e^{-j 2 pi k / 256}
//   power    P[m] = X_re[m]^2 + X_im[m]^2 (uint32)
// and the record holds sum_frames P[(i + 128) mod 256] at bin i: natural frequency order, bin 0 at -fs/2,
// bin 128 at DC.  Bounds: |x| <= 128 and w <= 16384, so |v| <= 128 per component and |X| < 256 * 128 * sqrt(2)
// + 8 (one rounding per stage) < 46400: every product and sum fits int32 (|b c + b' s| <= |b| 16384 by
// Cauchy-Schwarz), P < 2^31.01 fits uint32 and a record's sum (F <= 2560) fits uint64 with room.
// tests/spectrum_model.py restates the definition in numpy; the CPU suite checks it against this header's
// host build (tests/host_shim/spectrum_core_host.cpp).
#pragma once
#include <cstdint>
#include "modes_b200.h"
#include "modes_resample_core.cuh"

#if defined(__CUDACC__)
#define MODES_SPECTRUM_FN __host__ __device__ __forceinline__
#else
#define MODES_SPECTRUM_FN static inline
#endif

namespace modes {
namespace spectrum {

constexpr int kN = 256;                 // samples per frame (== MODES_SPECTRUM_BINS)
constexpr int kLog2N = 8;
constexpr int kShift = 14;

// s_b: the first input sample reference buffer b stands for, at the ratio out : in.
MODES_SPECTRUM_FN int64_t first_sample(int out, int in, int64_t b) {
    return resample::floor_div((int64_t)in * b * (int64_t)MODES_BUFFER_SAMPLES, out);
}
// F: buffer b's whole frames.
MODES_SPECTRUM_FN uint32_t frames(int out, int in, int64_t b) {
    return (uint32_t)((first_sample(out, in, b + 1) - first_sample(out, in, b)) / kN);
}
// The most frames a buffer has at the ratio (F differs between buffers by at most one frame's remainder).
MODES_SPECTRUM_FN uint32_t max_frames(int out, int in) {
    return (uint32_t)(((int64_t)in * MODES_BUFFER_SAMPLES / out + 1) / kN);
}

// w[n], Q14.
MODES_SPECTRUM_FN int window(int cos4n) { return (16384 - cos4n) >> 1; }
MODES_SPECTRUM_FN int windowed(int x, int w) { return (x * w + (1 << (kShift - 1))) >> kShift; }

// The 8-bit bit reversal of n: where sample n sits in the decimation-in-time input.
MODES_SPECTRUM_FN int bitrev8(int n) {
    n = (n & 0xf0) >> 4 | (n & 0x0f) << 4;
    n = (n & 0xcc) >> 2 | (n & 0x33) << 2;
    return (n & 0xaa) >> 1 | (n & 0x55) << 1;
}

// One butterfly, c and s those of its k.
MODES_SPECTRUM_FN void butterfly(int &ar, int &ai, int &br, int &bi, int c, int s) {
    const int tr = (br * c + bi * s + (1 << (kShift - 1))) >> kShift;
    const int ti = (bi * c - br * s + (1 << (kShift - 1))) >> kShift;
    br = ar - tr;
    bi = ai - ti;
    ar += tr;
    ai += ti;
}

MODES_SPECTRUM_FN uint32_t power(int re, int im) { return (uint32_t)re * (uint32_t)re + (uint32_t)im * (uint32_t)im; }

// Record bin of FFT output m.
MODES_SPECTRUM_FN int bin_of(int m) { return (m + kN / 2) & (kN - 1); }

#if !defined(__CUDACC__)
// One frame on the host (the host build only), the definition's order: iq = the frame's 256 UC8 pairs, out[bin] its power.
inline void frame_power(const uint8_t *iq, uint32_t out[kN]) {
    int re[kN], im[kN];
    for (int n = 0; n < kN; n++) {
        const int w = window(shift::kCos[4 * n]);
        re[bitrev8(n)] = windowed((int)iq[2 * n] - 127, w);
        im[bitrev8(n)] = windowed((int)iq[2 * n + 1] - 127, w);
    }
    for (int st = 0; st < kLog2N; st++) {
        const int half = 1 << st;
        for (int i = 0; i < kN; i++) {
            if (i & half) continue;
            const int k = (i & (half - 1)) << (kLog2N - 1 - st);
            butterfly(re[i], im[i], re[i + half], im[i + half], shift::kCos[4 * k], shift::kSin[4 * k]);
        }
    }
    for (int m = 0; m < kN; m++) out[bin_of(m)] = power(re[m], im[m]);
}
#endif

}  // namespace spectrum
}  // namespace modes
