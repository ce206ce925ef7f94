// modes_resample_core.cuh — the arithmetic of the input rates other than 2 MHz (modes_resample.cu): the
// 2.4 MS/s resampler (K9), the 4-10 MS/s decimator (K11, below) and the descriptor of every rate the
// decoder takes (InputRate, at the end), which the host's streaming reads its rate decision from.
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

// ---- 4, 6, 8 and 10 MS/s: integer decimation by M = 2, 3, 4, 5 (DESIGN §3 K11)
//
//   input   as above, at 2 M MS/s
//   output  sample n stands for input samples [M n, M n + M) and, for I and Q separately,
//               y = clamp(127 + ((sum_{k<T} h_M[k] * (x[M n - E + k] - 127) + 8192) >> 14), 0, 255)
//           with T = M + 2 E (int32 sum, arithmetic shift); the stream has N_out = ceil(n_in / M) output
//           samples.  Output n starts at input sample M n exactly, so 6 * sample_pos stays the 12 MHz time.
// h_M is symmetric about input M n + (M - 1) / 2 and sums to exactly 16384 (the remainder of its Q14
// rounding is on its middle tap, or split over the two middle taps); a constant 127 gives exactly 127.
// tests/decimate_model.py derives each table and restates the definition (host build:
// tests/host_shim/decimate_core_host.cpp).
namespace decimate {

// E of M's table: the taps on each side of the output's M input samples (DESIGN §6 has the sweep).
MODES_RESAMPLE_FN constexpr int extent(int m) { return m == 3 ? 1 : 2; }
MODES_RESAMPLE_FN constexpr int taps(int m) { return m + 2 * extent(m); }

// h_M[k], Q14: a Kaiser-windowed sinc (beta 5, cutoff 0.8 MHz) over T input samples for every M (DESIGN §3
// K11).  A function, so that device code folds each tap into an immediate.
MODES_RESAMPLE_FN constexpr int tap(int m, int k) {
    constexpr int16_t h2[6] = {0, 1974, 6218, 6218, 1974, 0};
    constexpr int16_t h3[5] = {715, 4116, 6722, 4116, 715};
    constexpr int16_t h4[8] = {185, 1073, 2740, 4194, 4194, 2740, 1073, 185};
    constexpr int16_t h5[9] = {177, 828, 2016, 3266, 3810, 3266, 2016, 828, 177};
    return m == 2 ? h2[k] : m == 3 ? h3[k] : m == 4 ? h4[k] : h5[k];
}

// Input samples a group of 8 output samples reads, and the 32-bit words (2 UC8 samples each) they fill.
MODES_RESAMPLE_FN constexpr int group_in(int m) { return 8 * m + 2 * extent(m); }
MODES_RESAMPLE_FN constexpr int group_words(int m) { return (group_in(m) + 1) / 2; }

// The group of output samples 8g .. 8g + 7 from its input samples 8 M g - E ... as little-endian words of
// UC8 bytes (w[j / 2] holds sample j at bits 16 (j & 1) ..): out[i] = samples 2i and 2i + 1 as I/Q bytes.
// Every table sums to 2^14, so sum h (x - 127) = sum h x - 127 * 2^14 and the 127s cancel outside the shift.
template <int M>
MODES_RESAMPLE_FN void group(const uint32_t *w, uint32_t out[4]) {
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int i = 0; i < 8; i++) {
        int ai = 0, aq = 0;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
        for (int k = 0; k < taps(M); k++) {
            const int j = M * i + k;
            const uint32_t v = w[j >> 1] >> (16 * (j & 1));
            ai += tap(M, k) * (int)(v & 0xff);
            aq += tap(M, k) * (int)((v >> 8) & 0xff);
        }
        int yi = (ai + (1 << 13)) >> 14, yq = (aq + (1 << 13)) >> 14;
        yi = yi < 0 ? 0 : (yi > 255 ? 255 : yi);
        yq = yq < 0 ? 0 : (yq > 255 ? 255 : yq);
        const uint32_t y = (uint32_t)yi | (uint32_t)yq << 8;
        out[i >> 1] = (i & 1) ? (out[i >> 1] | y << 16) : y;
    }
}

}  // namespace decimate

// ---- the input rates the decoder takes: which input samples each 2 MHz output sample reads
struct InputRate {
    uint32_t hz;
    int out, in;       // out output samples per in input samples
    int lead, taps;    // output n reads input samples floor(in n / out) - lead ... + taps
    int carry;         // output samples before a batch that its input span covers (the carry block's 238, or the
                       // 240 of its whole 16-byte groups where a kernel writes them as such)
    int m;             // decimation factor (K11), 0 where the ratio is not an integer one
};

constexpr InputRate kInputRates[] = {
    {2000000, 1, 1, 0, 1, 240, 0},
    {2400000, 5, 6, resample::kLead, resample::kTaps, 238, 0},
    {4000000, 1, 2, decimate::extent(2), decimate::taps(2), 240, 2},
    {6000000, 1, 3, decimate::extent(3), decimate::taps(3), 240, 3},
    {8000000, 1, 4, decimate::extent(4), decimate::taps(4), 240, 4},
    {10000000, 1, 5, decimate::extent(5), decimate::taps(5), 240, 5},
};

// The descriptor of hz, or nullptr for a rate the decoder does not take.
inline const InputRate *find_input_rate(uint32_t hz) {
    for (const InputRate &r : kInputRates)
        if (r.hz == hz) return &r;
    return nullptr;
}

// The input samples [in_lo(r, n), in_hi(r, n)) that output sample n reads.
MODES_RESAMPLE_FN int64_t in_lo(const InputRate &r, int64_t n) { return resample::floor_div((int64_t)r.in * n, r.out) - r.lead; }
MODES_RESAMPLE_FN int64_t in_hi(const InputRate &r, int64_t n) { return in_lo(r, n) + r.taps; }

// Output samples of a stream of n_in input samples: ceil(out n_in / in).
MODES_RESAMPLE_FN int64_t n_out(const InputRate &r, int64_t n_in) { return ((int64_t)r.out * n_in + r.in - 1) / r.in; }

}  // namespace modes
