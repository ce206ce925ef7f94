// modes_input_core.cuh — the arithmetic of the 16-bit input formats (modes_set_input_format; kernels
// K10 and K9's int16 loader in modes_resample.cu).
//
// The decoder's pipeline runs on UC8 bytes (unsigned 8-bit I/Q, zero at 127).  A capture of signed
// little-endian 16-bit I/Q (SC16: SoapySDR and Airspy-class tools; SC16Q11: bladeRF, 12-bit values in
// int16) is first converted to UC8, I and Q separately, defined bit for bit:
//     q    = s ? (v + (1 << (s - 1))) >> s : v        (int32, arithmetic shift: round half up)
//     byte = clamp(127 + q, 0, 255)
// for a value v and a shift s in 0..15.  A sample is 4 bytes (I, Q); a stream of `bytes` bytes has
// n_in = floor(bytes / 4) samples, and 1-3 trailing bytes are ignored.  The converted stream is then
// decoded as a UC8 stream at the input rate (at 2.4 MS/s: convert, then resample).  SC16 and SC16Q11
// differ only in the default shift, which maps full scale to full scale; this header is the one place
// that knows it.  tests/input_format_model.py restates the definition; the CPU suite checks it against
// this header's host build (tests/host_shim/input_core_host.cpp).
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define MODES_INPUT_FN __host__ __device__ __forceinline__
#else
#define MODES_INPUT_FN static inline
#endif

namespace modes {
namespace input {

constexpr uint32_t kUC8 = 0;        // == MODES_INPUT_UC8
constexpr uint32_t kSC16 = 1;       // == MODES_INPUT_SC16
constexpr uint32_t kSC16Q11 = 2;    // == MODES_INPUT_SC16Q11
constexpr int kMaxShift = 15;

MODES_INPUT_FN constexpr bool known(uint32_t format) { return format <= kSC16Q11; }
// Bytes per I/Q sample.
MODES_INPUT_FN constexpr int sample_bytes(uint32_t format) { return format == kUC8 ? 2 : 4; }
// The shift that maps the format's full scale to UC8's: SC16 +-32768 and SC16Q11 +-2048 to +-128.
MODES_INPUT_FN constexpr int default_shift(uint32_t format) { return format == kSC16 ? 8 : format == kSC16Q11 ? 4 : 0; }

// One int16 value (I or Q) as its UC8 byte.
MODES_INPUT_FN uint32_t convert(int v, int s) {
    const int q = (v + ((1 << s) >> 1)) >> s;
    const int y = 127 + q;
    return (uint32_t)(y < 0 ? 0 : (y > 255 ? 255 : y));
}

// One 4-byte sample (I in the low half, Q in the high half, little-endian) as its UC8 pair I | Q << 8.
MODES_INPUT_FN uint32_t convert_pair(uint32_t w, int s) {
    return convert((int)(int16_t)(w & 0xffffu), s) | convert((int)(int16_t)(w >> 16), s) << 8;
}

// n whole samples of 16-bit I/Q bytes at in (4 bytes a sample, little-endian) to their 2 n UC8 bytes at out,
// on the host: the carry of a 2 MHz 16-bit receiver of the pool (modes_pool.cpp).
inline void convert_samples(const uint8_t *in, int64_t n, int s, uint8_t *out) {
    for (int64_t k = 0; k < n; k++) {
        const uint8_t *x = in + 4 * k;
        const uint32_t y = convert_pair((uint32_t)x[0] | (uint32_t)x[1] << 8 | (uint32_t)x[2] << 16 | (uint32_t)x[3] << 24, s);
        out[2 * k] = (uint8_t)y;
        out[2 * k + 1] = (uint8_t)(y >> 8);
    }
}

}  // namespace input
}  // namespace modes
