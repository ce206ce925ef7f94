// modes_tables.cpp — host-side construction of the small constant tables the
// kernels read.  Generated from their defining formulas, never copied:
//   lutn     magnitude by squared amplitude: the reference's
//            round(sqrt(i*i+q*q)*360) (dump1090.c:362) keyed by n = i*i+q*q
//   lut_iq   the same magnitude keyed by (|I-127|, |Q-127|), rows kLutIqStride apart (the
//            frame-evaluation kernel keeps it in shared memory)
//   bit_syn  syndrome of one flipped bit at frame position p of a 112-bit frame:
//            x^(111-p) mod the Mode S generator 0x1FFF409 for data bits (what
//            modes_checksum_table holds, dump1090.c:683-698), the bit itself for
//            the 24 parity bits (dump1090.c:738-741)
//   fix_hash open-addressed inverse of bit_syn over positions 5..111, the domain
//            of the reference's bitErrorTable (dump1090.c:806)
//   pair_hash open-addressed map from the syndrome of TWO flipped bits p < q (positions 5..111,
//            5671 patterns, all syndromes distinct and none equal to a single's: dump1090.c:817-841,
//            checked here) to p; q follows from
//            fix_hash(S ^ bit_syn[p]).  One or two probes replace a 107-step search per frame.
#include <cmath>
#include <cstring>
#include "modes_internal.h"

namespace modes {

void build_lutn(uint16_t *out) {
    for (int n = 0; n < kNLutEntries; n++) out[n] = (uint16_t)std::round(std::sqrt((double)n) * 360);
}

void build_lut_iq(uint16_t *out) {
    std::memset(out, 0, sizeof(uint16_t) * kLutIqEntries);
    for (int i = 0; i <= 128; i++)
        for (int q = 0; q <= 128; q++) out[i * kLutIqStride + q] = (uint16_t)std::round(std::sqrt((double)(i * i + q * q)) * 360);
}

void build_bit_syndromes(uint32_t *out) {
    uint32_t v = 0xFFF409;                       // x^24 mod G
    for (int p = 87; p >= 0; p--) {
        out[p] = v;
        v <<= 1;
        if (v & 0x1000000u) v ^= 0x1FFF409u;
    }
    for (int p = 88; p < 112; p++) out[p] = 1u << (111 - p);
}

bool build_fix_hash(const uint32_t *bit_syn, uint32_t *out) {
    std::memset(out, 0xFF, sizeof(uint32_t) * kFixHashSlots);
    for (int p = 5; p < 112; p++) {
        uint32_t s = bit_syn[p];
        uint32_t h = (s * 0x9E3779B1u) >> 24;
        int i = 0;
        for (; i < kFixHashSlots; i++) {
            uint32_t &e = out[(h + i) & (kFixHashSlots - 1)];
            if (e == 0xFFFFFFFFu) { e = (s << 8) | (uint32_t)p; break; }
            if ((e >> 8) == s) return false;     // two positions with one syndrome: impossible for this code
        }
        if (i == kFixHashSlots) return false;
    }
    return true;
}

bool build_pair_hash(const uint32_t *bit_syn, uint32_t *out) {
    std::memset(out, 0xFF, sizeof(uint32_t) * kPairHashSlots);
    for (int p = 5; p < 112; p++)
        for (int q = p + 1; q < 112; q++) {
            const uint32_t s = bit_syn[p] ^ bit_syn[q];
            if (s == 0 || s >= (1u << 24)) return false;
            // nor may a pair share a single's syndrome: the kernels go on to this table when the
            // single-bit hit lies outside a short frame, where the reference stops at the single
            for (int r = 5; r < 112; r++)
                if (s == bit_syn[r]) return false;
            const uint32_t h = (s * 0x9E3779B1u) >> (32 - kPairHashBits);
            int i = 0;
            for (; i < kPairHashMaxProbe; i++) {
                uint32_t &e = out[(h + i) & (kPairHashSlots - 1)];
                if (e == 0xFFFFFFFFu) { e = (s << 7) | (uint32_t)p; break; }
                if ((e >> 7) == s) return false;     // two patterns with one syndrome: impossible for this code
            }
            if (i == kPairHashMaxProbe) return false;    // the probe bound the kernels rely on
        }
    return true;
}

}  // namespace modes
