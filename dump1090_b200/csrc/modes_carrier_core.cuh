// modes_carrier_core.cuh — the arithmetic of the carrier measurement (modes_set_carrier, definition in
// include/modes_b200.h), run by the signal pass's kernel (modes_signal.cu) and converted to the message's
// code by the host resolve (modes_resolve.cpp).
//
// Window samples are numbered relative to the attempt's position j.  The pulse sample of bit i is
// 16+2i when the bit is 1 and 17+2i when it is 0, so the pulses of bits i and i+1 are exactly two
// samples (1 us) apart when the two bits are equal; the preamble's pulses give the pairs (0, 2) and
// (7, 9).  With z = (I - 127) + i (Q - 127), the record is the sum of z_later conj(z_earlier) over
// those pairs, in int32 (each term's parts are at most 2^15 in magnitude, and there are at most 113
// pairs).
//
// Like modes_arrival_core.cuh the file needs nothing from CUDA, so the test suite also compiles it for
// the host (tests/host_shim/carrier_core_host.cpp) and checks it against a plain restatement of the
// definition.  That build is test infrastructure.
#pragma once
#include <cmath>
#include <cstdint>

#if defined(__CUDACC__)
#define MODES_CARRIER_FN __host__ __device__ __forceinline__
#else
#define MODES_CARRIER_FN static inline
#endif

namespace modes {
namespace carrier {

// The code of a message not measured, and of the centre of the bytes (0 Hz).
constexpr int kNotMeasured = 0;
constexpr int kCodeZero = 16384;

// z_b conj(z_a) added to (re, im): a, b = two samples as their raw 16-bit words (I in the low byte).
MODES_CARRIER_FN void add_pair(uint32_t a, uint32_t b, int32_t &re, int32_t &im) {
    const int32_t ia = (int32_t)(a & 0xffu) - 127, qa = (int32_t)((a >> 8) & 0xffu) - 127;
    const int32_t ib = (int32_t)(b & 0xffu) - 127, qb = (int32_t)((b >> 8) & 0xffu) - 127;
    re += ia * ib + qa * qb;
    im += ia * qb - qa * ib;
}

// The pulse sample of a bit from its pair word (first sample in the low half): the first when the bit is 1.
MODES_CARRIER_FN uint32_t pulse_of(uint32_t pair, uint32_t bit) { return bit ? (pair & 0xffffu) : (pair >> 16); }

// The bits 32r + l (bit l of the mask) that pair with the next bit: 32r + l + 1 < b and both bits equal.
// B: the frame's bits as arrival::bit_words holds them (bits from b on cleared).
MODES_CARRIER_FN uint32_t equal_next(const uint32_t B[4], int r, uint32_t b) {
    const uint32_t cur = B[r];
    const uint32_t next = (cur >> 1) | (r < 3 ? B[r + 1] << 31 : 0u);
    const int left = (int)b - 1 - 32 * r;                                 // bits of this word with a successor
    const uint32_t valid = left >= 32 ? 0xffffffffu : (left <= 0 ? 0u : (1u << left) - 1u);
    return ~(cur ^ next) & valid;
}

// The code of a record: 16384 + round(f / 100 Hz), halves away from zero, with f = atan2(im, re) / (2 pi 1 us)
// in (-500 kHz, 500 kHz]; 0 (not measured) when re = im = 0.  A measured record's code is 11384 .. 21384.
MODES_CARRIER_FN int16_t code_of(int32_t re, int32_t im) {
    if (re == 0 && im == 0) return (int16_t)kNotMeasured;
    const double c = std::atan2((double)im, (double)re) * (1e4 / (2.0 * 3.14159265358979323846));   // f / 100 Hz
    const double q = c < 0 ? -std::floor(-c + 0.5) : std::floor(c + 0.5);
    return (int16_t)(kCodeZero + (int)q);
}

}  // namespace carrier
}  // namespace modes
