// modes_resample_core.cuh — the arithmetic of the input rates other than 2 MHz (modes_resample.cu): the
// 2.4 MS/s resampler (K9), the 4-10 MS/s decimator (K11, below), its frequency shift (K12, after it) and
// the descriptor of every rate the decoder takes (InputRate, at the end), which the host's streaming reads
// its rate decision from.
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

// ---- 4-10 MS/s captures tuned off 1090 MHz: an exact frequency shift in front of the decimator (DESIGN §3 K12)
//
// modes_set_input_offset: 1090 MHz sits at offset_hz in the capture's baseband.  Each input sample m (counted
// from the stream's start; int16 input after its conversion) is rotated by e^{-j 2 pi offset m / fs} before
// the decimator's filter, with xi = I - 127, xq = Q - 127 (0 outside the stream):
//   step   = round(offset_hz 2^32 / fs)                      (int64, stored as uint32)
//   theta  = (m step) mod 2^32                               (m mod 2^32 first)
//   k      = ((theta + 2^21) >> 22) & 1023                   (the nearest of 1024 phases)
//   u_i    = (xi C[k] + xq S[k] + 8192) >> 14                (int32, arithmetic shift)
//   u_q    = (xq C[k] - xi S[k] + 8192) >> 14
//   y      = clamp(127 + ((sum_{k<T} h_M[k] u[M n - E + k] + 8192) >> 14), 0, 255)   (I and Q separately)
// C and S are Q14 cos and sin, round(16384 cos(2 pi k / 1024)) and round(16384 sin(2 pi k / 1024)).  The
// shift applied is step fs / 2^32 Hz, within 0.002 Hz of offset_hz; h_M, E and T are K11's.  At offset 0
// (step 0, k 0: C = 16384, S = 0) u = x, so this is K11 exactly.  Bounds: |x| <= 128 and |C| + |S| <= 23170,
// so |u| <= 182 and |sum h_M u| <= 16384 * 182 (every tap is >= 0): all of it fits int32 with room.
// tests/shift_model.py derives C and S and restates the definition (host build:
// tests/host_shim/shift_core_host.cpp).
#if defined(__CUDACC__)
#define MODES_SHIFT_TABLE static __device__ const
#else
#define MODES_SHIFT_TABLE static const
#endif
namespace shift {

MODES_SHIFT_TABLE int16_t kCos[1024] = {
    16384, 16384, 16383, 16381, 16379, 16376, 16373, 16369, 16364, 16359, 16353, 16347, 16340, 16332, 16324, 16315,
    16305, 16295, 16284, 16273, 16261, 16248, 16235, 16221, 16207, 16192, 16176, 16160, 16143, 16125, 16107, 16088,
    16069, 16049, 16029, 16008, 15986, 15964, 15941, 15917, 15893, 15868, 15843, 15817, 15791, 15763, 15736, 15707,
    15679, 15649, 15619, 15588, 15557, 15525, 15493, 15460, 15426, 15392, 15357, 15322, 15286, 15250, 15213, 15175,
    15137, 15098, 15059, 15019, 14978, 14937, 14896, 14854, 14811, 14768, 14724, 14680, 14635, 14589, 14543, 14497,
    14449, 14402, 14354, 14305, 14256, 14206, 14155, 14104, 14053, 14001, 13949, 13896, 13842, 13788, 13733, 13678,
    13623, 13567, 13510, 13453, 13395, 13337, 13279, 13219, 13160, 13100, 13039, 12978, 12916, 12854, 12792, 12729,
    12665, 12601, 12537, 12472, 12406, 12340, 12274, 12207, 12140, 12072, 12004, 11935, 11866, 11797, 11727, 11656,
    11585, 11514, 11442, 11370, 11297, 11224, 11151, 11077, 11003, 10928, 10853, 10778, 10702, 10625, 10549, 10471,
    10394, 10316, 10238, 10159, 10080, 10001, 9921, 9841, 9760, 9679, 9598, 9516, 9434, 9352, 9269, 9186,
    9102, 9019, 8935, 8850, 8765, 8680, 8595, 8509, 8423, 8337, 8250, 8163, 8076, 7988, 7900, 7812,
    7723, 7635, 7545, 7456, 7366, 7276, 7186, 7096, 7005, 6914, 6823, 6731, 6639, 6547, 6455, 6363,
    6270, 6177, 6084, 5990, 5897, 5803, 5708, 5614, 5520, 5425, 5330, 5235, 5139, 5044, 4948, 4852,
    4756, 4660, 4563, 4467, 4370, 4273, 4176, 4078, 3981, 3883, 3786, 3688, 3590, 3492, 3393, 3295,
    3196, 3098, 2999, 2900, 2801, 2702, 2603, 2503, 2404, 2305, 2205, 2105, 2006, 1906, 1806, 1706,
    1606, 1506, 1406, 1306, 1205, 1105, 1005, 904, 804, 704, 603, 503, 402, 302, 201, 101,
    0, -101, -201, -302, -402, -503, -603, -704, -804, -904, -1005, -1105, -1205, -1306, -1406, -1506,
    -1606, -1706, -1806, -1906, -2006, -2105, -2205, -2305, -2404, -2503, -2603, -2702, -2801, -2900, -2999, -3098,
    -3196, -3295, -3393, -3492, -3590, -3688, -3786, -3883, -3981, -4078, -4176, -4273, -4370, -4467, -4563, -4660,
    -4756, -4852, -4948, -5044, -5139, -5235, -5330, -5425, -5520, -5614, -5708, -5803, -5897, -5990, -6084, -6177,
    -6270, -6363, -6455, -6547, -6639, -6731, -6823, -6914, -7005, -7096, -7186, -7276, -7366, -7456, -7545, -7635,
    -7723, -7812, -7900, -7988, -8076, -8163, -8250, -8337, -8423, -8509, -8595, -8680, -8765, -8850, -8935, -9019,
    -9102, -9186, -9269, -9352, -9434, -9516, -9598, -9679, -9760, -9841, -9921, -10001, -10080, -10159, -10238, -10316,
    -10394, -10471, -10549, -10625, -10702, -10778, -10853, -10928, -11003, -11077, -11151, -11224, -11297, -11370, -11442, -11514,
    -11585, -11656, -11727, -11797, -11866, -11935, -12004, -12072, -12140, -12207, -12274, -12340, -12406, -12472, -12537, -12601,
    -12665, -12729, -12792, -12854, -12916, -12978, -13039, -13100, -13160, -13219, -13279, -13337, -13395, -13453, -13510, -13567,
    -13623, -13678, -13733, -13788, -13842, -13896, -13949, -14001, -14053, -14104, -14155, -14206, -14256, -14305, -14354, -14402,
    -14449, -14497, -14543, -14589, -14635, -14680, -14724, -14768, -14811, -14854, -14896, -14937, -14978, -15019, -15059, -15098,
    -15137, -15175, -15213, -15250, -15286, -15322, -15357, -15392, -15426, -15460, -15493, -15525, -15557, -15588, -15619, -15649,
    -15679, -15707, -15736, -15763, -15791, -15817, -15843, -15868, -15893, -15917, -15941, -15964, -15986, -16008, -16029, -16049,
    -16069, -16088, -16107, -16125, -16143, -16160, -16176, -16192, -16207, -16221, -16235, -16248, -16261, -16273, -16284, -16295,
    -16305, -16315, -16324, -16332, -16340, -16347, -16353, -16359, -16364, -16369, -16373, -16376, -16379, -16381, -16383, -16384,
    -16384, -16384, -16383, -16381, -16379, -16376, -16373, -16369, -16364, -16359, -16353, -16347, -16340, -16332, -16324, -16315,
    -16305, -16295, -16284, -16273, -16261, -16248, -16235, -16221, -16207, -16192, -16176, -16160, -16143, -16125, -16107, -16088,
    -16069, -16049, -16029, -16008, -15986, -15964, -15941, -15917, -15893, -15868, -15843, -15817, -15791, -15763, -15736, -15707,
    -15679, -15649, -15619, -15588, -15557, -15525, -15493, -15460, -15426, -15392, -15357, -15322, -15286, -15250, -15213, -15175,
    -15137, -15098, -15059, -15019, -14978, -14937, -14896, -14854, -14811, -14768, -14724, -14680, -14635, -14589, -14543, -14497,
    -14449, -14402, -14354, -14305, -14256, -14206, -14155, -14104, -14053, -14001, -13949, -13896, -13842, -13788, -13733, -13678,
    -13623, -13567, -13510, -13453, -13395, -13337, -13279, -13219, -13160, -13100, -13039, -12978, -12916, -12854, -12792, -12729,
    -12665, -12601, -12537, -12472, -12406, -12340, -12274, -12207, -12140, -12072, -12004, -11935, -11866, -11797, -11727, -11656,
    -11585, -11514, -11442, -11370, -11297, -11224, -11151, -11077, -11003, -10928, -10853, -10778, -10702, -10625, -10549, -10471,
    -10394, -10316, -10238, -10159, -10080, -10001, -9921, -9841, -9760, -9679, -9598, -9516, -9434, -9352, -9269, -9186,
    -9102, -9019, -8935, -8850, -8765, -8680, -8595, -8509, -8423, -8337, -8250, -8163, -8076, -7988, -7900, -7812,
    -7723, -7635, -7545, -7456, -7366, -7276, -7186, -7096, -7005, -6914, -6823, -6731, -6639, -6547, -6455, -6363,
    -6270, -6177, -6084, -5990, -5897, -5803, -5708, -5614, -5520, -5425, -5330, -5235, -5139, -5044, -4948, -4852,
    -4756, -4660, -4563, -4467, -4370, -4273, -4176, -4078, -3981, -3883, -3786, -3688, -3590, -3492, -3393, -3295,
    -3196, -3098, -2999, -2900, -2801, -2702, -2603, -2503, -2404, -2305, -2205, -2105, -2006, -1906, -1806, -1706,
    -1606, -1506, -1406, -1306, -1205, -1105, -1005, -904, -804, -704, -603, -503, -402, -302, -201, -101,
    0, 101, 201, 302, 402, 503, 603, 704, 804, 904, 1005, 1105, 1205, 1306, 1406, 1506,
    1606, 1706, 1806, 1906, 2006, 2105, 2205, 2305, 2404, 2503, 2603, 2702, 2801, 2900, 2999, 3098,
    3196, 3295, 3393, 3492, 3590, 3688, 3786, 3883, 3981, 4078, 4176, 4273, 4370, 4467, 4563, 4660,
    4756, 4852, 4948, 5044, 5139, 5235, 5330, 5425, 5520, 5614, 5708, 5803, 5897, 5990, 6084, 6177,
    6270, 6363, 6455, 6547, 6639, 6731, 6823, 6914, 7005, 7096, 7186, 7276, 7366, 7456, 7545, 7635,
    7723, 7812, 7900, 7988, 8076, 8163, 8250, 8337, 8423, 8509, 8595, 8680, 8765, 8850, 8935, 9019,
    9102, 9186, 9269, 9352, 9434, 9516, 9598, 9679, 9760, 9841, 9921, 10001, 10080, 10159, 10238, 10316,
    10394, 10471, 10549, 10625, 10702, 10778, 10853, 10928, 11003, 11077, 11151, 11224, 11297, 11370, 11442, 11514,
    11585, 11656, 11727, 11797, 11866, 11935, 12004, 12072, 12140, 12207, 12274, 12340, 12406, 12472, 12537, 12601,
    12665, 12729, 12792, 12854, 12916, 12978, 13039, 13100, 13160, 13219, 13279, 13337, 13395, 13453, 13510, 13567,
    13623, 13678, 13733, 13788, 13842, 13896, 13949, 14001, 14053, 14104, 14155, 14206, 14256, 14305, 14354, 14402,
    14449, 14497, 14543, 14589, 14635, 14680, 14724, 14768, 14811, 14854, 14896, 14937, 14978, 15019, 15059, 15098,
    15137, 15175, 15213, 15250, 15286, 15322, 15357, 15392, 15426, 15460, 15493, 15525, 15557, 15588, 15619, 15649,
    15679, 15707, 15736, 15763, 15791, 15817, 15843, 15868, 15893, 15917, 15941, 15964, 15986, 16008, 16029, 16049,
    16069, 16088, 16107, 16125, 16143, 16160, 16176, 16192, 16207, 16221, 16235, 16248, 16261, 16273, 16284, 16295,
    16305, 16315, 16324, 16332, 16340, 16347, 16353, 16359, 16364, 16369, 16373, 16376, 16379, 16381, 16383, 16384,
};
MODES_SHIFT_TABLE int16_t kSin[1024] = {
    0, 101, 201, 302, 402, 503, 603, 704, 804, 904, 1005, 1105, 1205, 1306, 1406, 1506,
    1606, 1706, 1806, 1906, 2006, 2105, 2205, 2305, 2404, 2503, 2603, 2702, 2801, 2900, 2999, 3098,
    3196, 3295, 3393, 3492, 3590, 3688, 3786, 3883, 3981, 4078, 4176, 4273, 4370, 4467, 4563, 4660,
    4756, 4852, 4948, 5044, 5139, 5235, 5330, 5425, 5520, 5614, 5708, 5803, 5897, 5990, 6084, 6177,
    6270, 6363, 6455, 6547, 6639, 6731, 6823, 6914, 7005, 7096, 7186, 7276, 7366, 7456, 7545, 7635,
    7723, 7812, 7900, 7988, 8076, 8163, 8250, 8337, 8423, 8509, 8595, 8680, 8765, 8850, 8935, 9019,
    9102, 9186, 9269, 9352, 9434, 9516, 9598, 9679, 9760, 9841, 9921, 10001, 10080, 10159, 10238, 10316,
    10394, 10471, 10549, 10625, 10702, 10778, 10853, 10928, 11003, 11077, 11151, 11224, 11297, 11370, 11442, 11514,
    11585, 11656, 11727, 11797, 11866, 11935, 12004, 12072, 12140, 12207, 12274, 12340, 12406, 12472, 12537, 12601,
    12665, 12729, 12792, 12854, 12916, 12978, 13039, 13100, 13160, 13219, 13279, 13337, 13395, 13453, 13510, 13567,
    13623, 13678, 13733, 13788, 13842, 13896, 13949, 14001, 14053, 14104, 14155, 14206, 14256, 14305, 14354, 14402,
    14449, 14497, 14543, 14589, 14635, 14680, 14724, 14768, 14811, 14854, 14896, 14937, 14978, 15019, 15059, 15098,
    15137, 15175, 15213, 15250, 15286, 15322, 15357, 15392, 15426, 15460, 15493, 15525, 15557, 15588, 15619, 15649,
    15679, 15707, 15736, 15763, 15791, 15817, 15843, 15868, 15893, 15917, 15941, 15964, 15986, 16008, 16029, 16049,
    16069, 16088, 16107, 16125, 16143, 16160, 16176, 16192, 16207, 16221, 16235, 16248, 16261, 16273, 16284, 16295,
    16305, 16315, 16324, 16332, 16340, 16347, 16353, 16359, 16364, 16369, 16373, 16376, 16379, 16381, 16383, 16384,
    16384, 16384, 16383, 16381, 16379, 16376, 16373, 16369, 16364, 16359, 16353, 16347, 16340, 16332, 16324, 16315,
    16305, 16295, 16284, 16273, 16261, 16248, 16235, 16221, 16207, 16192, 16176, 16160, 16143, 16125, 16107, 16088,
    16069, 16049, 16029, 16008, 15986, 15964, 15941, 15917, 15893, 15868, 15843, 15817, 15791, 15763, 15736, 15707,
    15679, 15649, 15619, 15588, 15557, 15525, 15493, 15460, 15426, 15392, 15357, 15322, 15286, 15250, 15213, 15175,
    15137, 15098, 15059, 15019, 14978, 14937, 14896, 14854, 14811, 14768, 14724, 14680, 14635, 14589, 14543, 14497,
    14449, 14402, 14354, 14305, 14256, 14206, 14155, 14104, 14053, 14001, 13949, 13896, 13842, 13788, 13733, 13678,
    13623, 13567, 13510, 13453, 13395, 13337, 13279, 13219, 13160, 13100, 13039, 12978, 12916, 12854, 12792, 12729,
    12665, 12601, 12537, 12472, 12406, 12340, 12274, 12207, 12140, 12072, 12004, 11935, 11866, 11797, 11727, 11656,
    11585, 11514, 11442, 11370, 11297, 11224, 11151, 11077, 11003, 10928, 10853, 10778, 10702, 10625, 10549, 10471,
    10394, 10316, 10238, 10159, 10080, 10001, 9921, 9841, 9760, 9679, 9598, 9516, 9434, 9352, 9269, 9186,
    9102, 9019, 8935, 8850, 8765, 8680, 8595, 8509, 8423, 8337, 8250, 8163, 8076, 7988, 7900, 7812,
    7723, 7635, 7545, 7456, 7366, 7276, 7186, 7096, 7005, 6914, 6823, 6731, 6639, 6547, 6455, 6363,
    6270, 6177, 6084, 5990, 5897, 5803, 5708, 5614, 5520, 5425, 5330, 5235, 5139, 5044, 4948, 4852,
    4756, 4660, 4563, 4467, 4370, 4273, 4176, 4078, 3981, 3883, 3786, 3688, 3590, 3492, 3393, 3295,
    3196, 3098, 2999, 2900, 2801, 2702, 2603, 2503, 2404, 2305, 2205, 2105, 2006, 1906, 1806, 1706,
    1606, 1506, 1406, 1306, 1205, 1105, 1005, 904, 804, 704, 603, 503, 402, 302, 201, 101,
    0, -101, -201, -302, -402, -503, -603, -704, -804, -904, -1005, -1105, -1205, -1306, -1406, -1506,
    -1606, -1706, -1806, -1906, -2006, -2105, -2205, -2305, -2404, -2503, -2603, -2702, -2801, -2900, -2999, -3098,
    -3196, -3295, -3393, -3492, -3590, -3688, -3786, -3883, -3981, -4078, -4176, -4273, -4370, -4467, -4563, -4660,
    -4756, -4852, -4948, -5044, -5139, -5235, -5330, -5425, -5520, -5614, -5708, -5803, -5897, -5990, -6084, -6177,
    -6270, -6363, -6455, -6547, -6639, -6731, -6823, -6914, -7005, -7096, -7186, -7276, -7366, -7456, -7545, -7635,
    -7723, -7812, -7900, -7988, -8076, -8163, -8250, -8337, -8423, -8509, -8595, -8680, -8765, -8850, -8935, -9019,
    -9102, -9186, -9269, -9352, -9434, -9516, -9598, -9679, -9760, -9841, -9921, -10001, -10080, -10159, -10238, -10316,
    -10394, -10471, -10549, -10625, -10702, -10778, -10853, -10928, -11003, -11077, -11151, -11224, -11297, -11370, -11442, -11514,
    -11585, -11656, -11727, -11797, -11866, -11935, -12004, -12072, -12140, -12207, -12274, -12340, -12406, -12472, -12537, -12601,
    -12665, -12729, -12792, -12854, -12916, -12978, -13039, -13100, -13160, -13219, -13279, -13337, -13395, -13453, -13510, -13567,
    -13623, -13678, -13733, -13788, -13842, -13896, -13949, -14001, -14053, -14104, -14155, -14206, -14256, -14305, -14354, -14402,
    -14449, -14497, -14543, -14589, -14635, -14680, -14724, -14768, -14811, -14854, -14896, -14937, -14978, -15019, -15059, -15098,
    -15137, -15175, -15213, -15250, -15286, -15322, -15357, -15392, -15426, -15460, -15493, -15525, -15557, -15588, -15619, -15649,
    -15679, -15707, -15736, -15763, -15791, -15817, -15843, -15868, -15893, -15917, -15941, -15964, -15986, -16008, -16029, -16049,
    -16069, -16088, -16107, -16125, -16143, -16160, -16176, -16192, -16207, -16221, -16235, -16248, -16261, -16273, -16284, -16295,
    -16305, -16315, -16324, -16332, -16340, -16347, -16353, -16359, -16364, -16369, -16373, -16376, -16379, -16381, -16383, -16384,
    -16384, -16384, -16383, -16381, -16379, -16376, -16373, -16369, -16364, -16359, -16353, -16347, -16340, -16332, -16324, -16315,
    -16305, -16295, -16284, -16273, -16261, -16248, -16235, -16221, -16207, -16192, -16176, -16160, -16143, -16125, -16107, -16088,
    -16069, -16049, -16029, -16008, -15986, -15964, -15941, -15917, -15893, -15868, -15843, -15817, -15791, -15763, -15736, -15707,
    -15679, -15649, -15619, -15588, -15557, -15525, -15493, -15460, -15426, -15392, -15357, -15322, -15286, -15250, -15213, -15175,
    -15137, -15098, -15059, -15019, -14978, -14937, -14896, -14854, -14811, -14768, -14724, -14680, -14635, -14589, -14543, -14497,
    -14449, -14402, -14354, -14305, -14256, -14206, -14155, -14104, -14053, -14001, -13949, -13896, -13842, -13788, -13733, -13678,
    -13623, -13567, -13510, -13453, -13395, -13337, -13279, -13219, -13160, -13100, -13039, -12978, -12916, -12854, -12792, -12729,
    -12665, -12601, -12537, -12472, -12406, -12340, -12274, -12207, -12140, -12072, -12004, -11935, -11866, -11797, -11727, -11656,
    -11585, -11514, -11442, -11370, -11297, -11224, -11151, -11077, -11003, -10928, -10853, -10778, -10702, -10625, -10549, -10471,
    -10394, -10316, -10238, -10159, -10080, -10001, -9921, -9841, -9760, -9679, -9598, -9516, -9434, -9352, -9269, -9186,
    -9102, -9019, -8935, -8850, -8765, -8680, -8595, -8509, -8423, -8337, -8250, -8163, -8076, -7988, -7900, -7812,
    -7723, -7635, -7545, -7456, -7366, -7276, -7186, -7096, -7005, -6914, -6823, -6731, -6639, -6547, -6455, -6363,
    -6270, -6177, -6084, -5990, -5897, -5803, -5708, -5614, -5520, -5425, -5330, -5235, -5139, -5044, -4948, -4852,
    -4756, -4660, -4563, -4467, -4370, -4273, -4176, -4078, -3981, -3883, -3786, -3688, -3590, -3492, -3393, -3295,
    -3196, -3098, -2999, -2900, -2801, -2702, -2603, -2503, -2404, -2305, -2205, -2105, -2006, -1906, -1806, -1706,
    -1606, -1506, -1406, -1306, -1205, -1105, -1005, -904, -804, -704, -603, -503, -402, -302, -201, -101,
};

constexpr int kPhases = 1024;

// step for offset_hz at fs: round(offset_hz 2^32 / fs), no ties (fs / 2^k is odd at every rate).  For the
// offsets offset_fits takes (|offset_hz| <= 4 MHz, so the int64 product has room).
MODES_RESAMPLE_FN uint32_t step(int32_t offset_hz, uint32_t fs) {
    return (uint32_t)resample::floor_div((int64_t)offset_hz * ((int64_t)1 << 33) + fs, 2 * (int64_t)fs);
}

// Phase k's rotation as shift_group's table holds it: the Q14 pair (C, S) as the 16-bit halves of a word.
MODES_RESAMPLE_FN uint32_t rotation(int c, int s) { return (uint32_t)(uint16_t)c | (uint32_t)(uint16_t)s << 16; }

// a.h0 * b.byte[2 Hi] + a.h1 * b.byte[2 Hi + 1] + c: a's halves signed, b's bytes unsigned (the I/Q bytes of
// the sample in b's low (Hi = 0) or high half) or, with SignedB, signed.  One IDP.2A on the device.
template <int Hi, bool SignedB = false>
MODES_RESAMPLE_FN int dot2(uint32_t a, uint32_t b, int c) {
#if defined(__CUDA_ARCH__)
    int d;
    if (SignedB) asm("dp2a.lo.s32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    else if (Hi) asm("dp2a.hi.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    else asm("dp2a.lo.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
#else
    const uint32_t v = b >> (16 * Hi);
    const int b0 = SignedB ? (int)(int8_t)(v & 0xffu) : (int)(v & 0xffu);
    const int b1 = SignedB ? (int)(int8_t)((v >> 8) & 0xffu) : (int)((v >> 8) & 0xffu);
    return c + (int16_t)(a & 0xffffu) * b0 + (int16_t)(a >> 16) * b1;
#endif
}

// decimate::group<M> on the rotated samples: the group of output samples 8g .. 8g + 7 from its input samples
// 8 M g - E ... (w as there), the first of which is stream sample m0 with theta0 = (m0 step) mod 2^32.  tab
// holds rotation(C[k], S[k]) at tab[k].  Each sample is rotated once and added into the (at most
// ceil(T / M)) outputs whose taps reach it, so only the 8 pairs of sums stay live.  With a = (C, S):
//   u_i = (C I + S Q + b_i) >> 14,          b_i = 8192 - 127 (C + S)           (one dot product for b_i)
//   u_q = (S (255 - I) + C Q + b_q) >> 14,  b_q = 8192 - 127 C - 128 S = b_i - S
// which are the definition's (the 127s folded into the constants); 255 - I is one XOR per pair of samples
// and (S, C) one byte permutation.  The sums start at 8192 + 127 * 2^14: the output's rounding and its 127,
// outside the shift.
template <int M>
MODES_RESAMPLE_FN void shift_group(const uint32_t *w, const uint32_t *tab, uint32_t theta0, uint32_t step,
                                   uint32_t out[4]) {
    constexpr int kBias = (1 << 13) + (127 << 14);
    int ai[8], aq[8];
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int i = 0; i < 8; i++) ai[i] = aq[i] = kBias;
    uint32_t theta = theta0 + (1u << 21);
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int j = 0; j < decimate::group_in(M); j++, theta += step) {
        const uint32_t a = tab[theta >> 22];
#if defined(__CUDA_ARCH__)
        const uint32_t as = __byte_perm(a, 0, 0x1032);
#else
        const uint32_t as = a >> 16 | a << 16;
#endif
        const int bi = dot2<0, true>(a, 0x8181u, 8192);
        const int bq = bi - ((int)a >> 16);
        const uint32_t v = w[j >> 1], vf = v ^ 0x00ff00ffu;
        const int ui = ((j & 1) ? dot2<1>(a, v, bi) : dot2<0>(a, v, bi)) >> 14;
        const int uq = ((j & 1) ? dot2<1>(as, vf, bq) : dot2<0>(as, vf, bq)) >> 14;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
        for (int i = 0; i < 8; i++) {
            const int t = j - M * i;
            if (t >= 0 && t < decimate::taps(M)) {
                ai[i] += decimate::tap(M, t) * ui;
                aq[i] += decimate::tap(M, t) * uq;
            }
        }
    }
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int i = 0; i < 8; i++) {
        int yi = ai[i] >> 14, yq = aq[i] >> 14;
        yi = yi < 0 ? 0 : (yi > 255 ? 255 : yi);
        yq = yq < 0 ? 0 : (yq > 255 ? 255 : yq);
        const uint32_t y = (uint32_t)yi | (uint32_t)yq << 8;
        out[i >> 1] = (i & 1) ? (out[i >> 1] | y << 16) : y;
    }
}

}  // namespace shift

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

// The largest |offset_hz| modes_set_input_offset takes at the rate: fs / 2 - 1 MHz at the decimated rates
// (the channel's +-1 MHz stays inside the band), 0 at 2 MHz and 2.4 MS/s.
MODES_RESAMPLE_FN int32_t max_offset(const InputRate &r) { return r.m ? (int32_t)(r.hz / 2) - 1000000 : 0; }
MODES_RESAMPLE_FN bool offset_fits(const InputRate &r, int32_t offset_hz) {
    return offset_hz >= -max_offset(r) && offset_hz <= max_offset(r);
}

}  // namespace modes
