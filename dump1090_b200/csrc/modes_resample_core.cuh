// modes_resample_core.cuh — the arithmetic of the 2.4 MS/s input resampler (modes_resample.cu).
//
// The decoder's pipeline runs on 2 MHz bytes.  A 2.4 MS/s capture (what dump1090-fa and readsb record)
// is first turned into 2 MHz bytes by an exact 5:6 polyphase filter, defined bit for bit:
//   input   UC8 I/Q at 2.4 MS/s, zero at 127; n_in = ceil(bytes / 2), a trailing odd byte is an I whose
//           Q is 127, and samples outside [0, n_in) read as (127, 127)
//   output  sample n = 5q + r (r = 0..4, q = floor(n / 5), n may be negative) has base input index
//           b = 6q + r and, for I and Q separately,
//               y = clamp(127 + ((sum_k h[r][k] * (x[b + k - T/2 + 1] - 127) + 8192) >> 14), 0, 255)
//           (int32 sum, arithmetic shift); the stream has N_out = ceil(5 n_in / 6) output samples.
// Output sample n sits at input time 1.2 n exactly, so 6 * sample_pos stays the input time in 12 MHz
// ticks (an input sample is 5 ticks, an output sample 6).
//
// The taps: one symmetric Kaiser-windowed sinc prototype (beta 5, cutoff 1.1 MHz, +-T/2 input samples),
// sampled at input offset k - T/2 + 1 - 0.2 r (a whole number of 12 MHz ticks).  Each branch is scaled to
// sum 1, rounded to Q14 and its remainder put on its largest tap, so every branch sums to exactly 16384:
// a constant 127 input gives exactly 127, and a stream start needs no special case.  tests/resample_model.py
// derives the table from this formula and restates the whole definition; the CPU suite checks both
// against this header's host build (tests/host_shim/resample_core_host.cpp).
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define MODES_RESAMPLE_FN __host__ __device__ __forceinline__
#else
#define MODES_RESAMPLE_FN static inline
#endif

namespace modes {
namespace resample {

constexpr int kTaps = 6;
constexpr int kShift = 14;
// kTaps / 2 - 1: tap k of output b reads input b + k - kLead
constexpr int kLead = kTaps / 2 - 1;

// h[r][k], Q14 (DESIGN §3 K9; the sweep that chose T = 6 and 1.1 MHz is in DESIGN §6)
// (a function, so that device code folds each tap into an immediate)
MODES_RESAMPLE_FN constexpr int tap(int r, int k) {
    constexpr int16_t h[5][kTaps] = {
        {-430, 1052, 15095, 1052, -430, 45},
        {31, -929, 14091, 4131, -1073, 133},
        {229, -1737, 11457, 7853, -1643, 225},
        {225, -1643, 7853, 11457, -1737, 229},
        {133, -1073, 4131, 14091, -929, 31},
    };
    return h[r][k];
}

// floor(a / b) for b > 0 and any a.
MODES_RESAMPLE_FN int64_t floor_div(int64_t a, int64_t b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }

// The input samples [in_lo(n), in_hi(n)) that output sample n reads.
MODES_RESAMPLE_FN int64_t in_base(int64_t n) { return floor_div(6 * n, 5); }
MODES_RESAMPLE_FN int64_t in_lo(int64_t n) { return in_base(n) - kLead; }
MODES_RESAMPLE_FN int64_t in_hi(int64_t n) { return in_base(n) - kLead + kTaps; }

// Output samples of a stream of n_in input samples.
MODES_RESAMPLE_FN int64_t n_out(int64_t n_in) { return (5 * n_in + 5) / 6; }

// One output byte of branch r from its T inputs, each already minus 127.
template <int R>
MODES_RESAMPLE_FN uint32_t branch(const int *x) {
    int acc = 0;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int k = 0; k < kTaps; k++) acc += tap(R, k) * x[k];
    const int y = 127 + ((acc + (1 << (kShift - 1))) >> kShift);
    return (uint32_t)(y < 0 ? 0 : (y > 255 ? 255 : y));
}

// One polyphase period: the 5 output samples 5q .. 5q + 4 from the input samples 6q - kLead ..
// 6q - kLead + kTaps + 3 (x[0 .. kTaps + 3], I and Q each already minus 127).  out[r] = I | Q << 8.
MODES_RESAMPLE_FN void period(const int *xi, const int *xq, uint32_t out[5]) {
    out[0] = branch<0>(xi + 0) | branch<0>(xq + 0) << 8;
    out[1] = branch<1>(xi + 1) | branch<1>(xq + 1) << 8;
    out[2] = branch<2>(xi + 2) | branch<2>(xq + 2) << 8;
    out[3] = branch<3>(xi + 3) | branch<3>(xq + 3) << 8;
    out[4] = branch<4>(xi + 4) | branch<4>(xq + 4) << 8;
}

// Input samples a period reads.
constexpr int kPeriodIn = kTaps + 4;

}  // namespace resample
}  // namespace modes
