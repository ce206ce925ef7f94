// TEST INFRASTRUCTURE — not part of the product.
// Host build of dump1090_b200/csrc/modes_carrier_core.cuh (frame bits -> pulse samples -> pair sums -> code,
// as the carrier pass and the host resolve compute them), so that the CPU test suite can check it against
// a plain restatement of the definition.
#include <cstring>
#include "modes_arrival_core.cuh"
#include "modes_carrier_core.cuh"

// iq: window samples 0 .. 17+2b as I/Q bytes; msg16: the attempt's 14 frame bytes and the two bytes that
// follow them in its record; bits: 56 or 112.  Writes (re, im) to out[0], out[1], the way the kernel
// forms them: word by word, each lane's pulse paired with the next bit's.
extern "C" void shim_carrier_window(const uint8_t *iq, const uint8_t *msg16, uint32_t bits, int32_t *out) {
    using namespace modes;
    auto sample = [&](uint32_t s) { uint16_t v; std::memcpy(&v, iq + 2 * s, 2); return (uint32_t)v; };
    uint32_t mw[4], B[4];
    std::memcpy(mw, msg16, 16);
    arrival::bit_words(mw, bits, B);
    int32_t re = 0, im = 0;
    carrier::add_pair(sample(0), sample(2), re, im);
    carrier::add_pair(sample(7), sample(9), re, im);
    auto pulse = [&](uint32_t i) {
        const uint32_t pair = sample(16 + 2 * i) | (sample(17 + 2 * i) << 16);
        return carrier::pulse_of(pair, (B[i >> 5] >> (i & 31)) & 1u);
    };
    for (int r = 0; r < 4; r++) {
        const uint32_t eq = carrier::equal_next(B, r, bits);
        for (int l = 0; l < 32; l++)
            if ((eq >> l) & 1u) carrier::add_pair(pulse(32 * r + l), pulse(32 * r + l + 1), re, im);
    }
    out[0] = re;
    out[1] = im;
}

extern "C" int32_t shim_carrier_code(int32_t re, int32_t im) { return modes::carrier::code_of(re, im); }
