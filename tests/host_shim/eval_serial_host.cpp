// TEST INFRASTRUCTURE — not part of the product.
// Host build of dump1090_b200/csrc/modes_eval_serial.cuh (the per-candidate evaluation that
// eval_serial_kernel runs one thread per candidate), so that its logic can be checked against the
// oracle's candidate records in the CPU test suite.  Windows are staged exactly as the kernel
// stages them; the constant tables come from the product's own builders (modes_tables.cpp).
#include <cstring>
#include <vector>
#include "modes_eval_serial.cuh"

namespace modes {
void build_lutn(uint16_t *out);
void build_lut_iq(uint16_t *out);
void build_bit_syndromes(uint32_t *out);
bool build_fix_hash(const uint32_t *bit_syn, uint32_t *out);
bool build_pair_hash(const uint32_t *bit_syn, uint32_t *out);
}

// The constant tables, built once by the product's builders; false if a builder refused.
static bool tables(modes::serial::Tables &tab) {
    using namespace modes::serial;
    static uint32_t bit_syn[112], fix_hash[256];
    static std::vector<uint32_t> nib_syn(28 * 16);
    static std::vector<uint16_t> lut_iq(kIqLutEntries);
    static std::vector<uint32_t> pair_hash(1u << kPairHashBits);
    static int ready = 0;                        // 0 not yet, 1 built, -1 refused
    if (!ready) {
        modes::build_bit_syndromes(bit_syn);
        for (int pos = 0; pos < 28; pos++)
            for (uint32_t v = 0; v < 16; v++) nib_syn[pos * 16 + v] = nibble_syndrome(bit_syn, pos, v);
        modes::build_lut_iq(lut_iq.data());
        ready = modes::build_fix_hash(bit_syn, fix_hash) && modes::build_pair_hash(bit_syn, pair_hash.data()) ? 1 : -1;
    }
    tab = Tables{lut_iq.data(), bit_syn, nib_syn.data(), fix_hash, pair_hash.data()};
    return ready == 1;
}

// The syndrome tables as the kernels see them: bit_syn[112], fix_hash[256], pair_hash[1 << kPairHashBits].
// Returns 0, or -1 if a builder refused.
extern "C" int shim_tables(uint32_t *bit_syn, uint32_t *fix_hash, uint32_t *pair_hash) {
    using namespace modes::serial;
    Tables tab;
    const bool ok = tables(tab);
    std::memcpy(bit_syn, tab.bit_syn, 112 * sizeof(uint32_t));
    std::memcpy(fix_hash, tab.fix_hash, 256 * sizeof(uint32_t));
    std::memcpy(pair_hash, tab.pair_hash, (1u << kPairHashBits) * sizeof(uint32_t));
    return ok ? 0 : -1;
}

// The builders themselves on caller-supplied syndromes (returns what the builder returns).
extern "C" int shim_build_bit_syndromes(uint32_t *out) { modes::build_bit_syndromes(out); return 0; }
extern "C" int shim_build_fix_hash(const uint32_t *bit_syn, uint32_t *out) { return modes::build_fix_hash(bit_syn, out); }
extern "C" int shim_build_pair_hash(const uint32_t *bit_syn, uint32_t *out) { return modes::build_pair_hash(bit_syn, out); }

// The hash probes: position (or first position of a pair) with syndrome s[i], or -1.
extern "C" void shim_probe(const uint32_t *s, uint32_t n, int32_t *single, int32_t *pair_first) {
    using namespace modes::serial;
    Tables tab;
    tables(tab);
    for (uint32_t i = 0; i < n; i++) {
        single[i] = syndrome_pos(tab.fix_hash, s[i]);
        pair_first[i] = modes::serial::pair_first(tab.pair_hash, s[i]);
    }
}

// serial::crc_and_fix on n 14-byte frames (the DF field decides the length): out[i] is the
// modes_frame_eval of the frame after the repair (flags GATE_OK | DECODED).
extern "C" int shim_crc_and_fix(const uint8_t *frames, uint64_t n, int fix_errors, int aggressive, modes_frame_eval *out) {
    using namespace modes::serial;
    Tables tab;
    if (!tables(tab)) return -1;
    for (uint64_t i = 0; i < n; i++) {
        const uint8_t *m = frames + 14 * i;
        Verdict R;
        R.F[0] = R.F[1] = R.F[2] = R.F[3] = 0;
        for (int b = 0; b < 112; b++) R.F[b >> 5] |= (uint32_t)((m[b >> 3] >> (7 - (b & 7))) & 1) << (b & 31);
        R.msgtype = m[0] >> 3;
        const int msgbits = (R.msgtype >= 16 && R.msgtype <= 21) ? 112 : 56;
        R.flags = MODES_EVAL_GATE_OK | MODES_EVAL_DECODED;
        crc_and_fix(R.F, msgbits, R.msgtype, fix_errors, aggressive, tab, R.crc, R.errorbit, R.nfixed);
        uint32_t w[6];
        eval_words(R, w);
        std::memcpy(&out[i], w, sizeof(w));
    }
    return 0;
}

// virt: the virtual sample array as bytes: 480 halo bytes (2 unused samples + 238 carried) then the body.
extern "C" int shim_eval_candidates(const uint8_t *virt, uint64_t n_virtual_samples, const uint32_t *cand_v, uint32_t n,
                                    int fix_errors, int aggressive, int lean, modes_candidate *out) {
    using namespace modes::serial;
    Tables tab;
    if (!tables(tab)) return -1;
    auto s16 = [&](uint64_t idx) -> uint32_t { uint16_t w; std::memcpy(&w, virt + 2 * idx, 2); return w; };
    for (uint32_t c = 0; c < n; c++) {
        const uint32_t v = cand_v[c];
        if ((uint64_t)v + 240 > n_virtual_samples) return -2;
        uint32_t win[kWindowWords];
        uint32_t odd = 0;
        if (v > 240) {
            const uint32_t first = v - 241;                      // body sample index of m[-1]
            odd = first & 1u;
            std::memcpy(win, virt + 480 + 4 * (uint64_t)(first >> 1), sizeof(win));
        } else {
            for (int k = 0; k < kWindowWords; k++) win[k] = s16((uint64_t)v - 1 + 2 * k) | (s16((uint64_t)v + 2 * k) << 16);
        }
        const uint64_t t = (uint64_t)v - 2;
        uint32_t rec[12];
        if (lean == 3) {
            // the same walk from half windows, as eval_fused_kernel<2, ..> stages them: slots 0..56, then
            // slots 56..112 into the same 57 words
            fused::Lane L;
            fused::phase_setup(win, odd, tab.lut_iq, 1u, 0xffffffffu, (uint32_t)-16384, L);
            uint32_t part[fused::kSlots];
            fused::Walk W;
            for (int u = 0; u < fused::kSlots; u++) part[u] = 0xdeadbeefu;
            for (int u = 0; u < 57; u++) part[u] = L.fwd ? win[8 + u] : win[120 - u];
            fused::walk_begin(W, L, part[0]);
            fused::walk_blocks(W, L, part, 0, 2, fused::Lut{tab.lut_iq});
            for (int u = 0; u < 56; u++) part[u] = 0xdeadbeefu;         // the second half must not look back
            for (int u = 56; u < fused::kSlots; u++) part[u] = L.fwd ? win[8 + u] : win[120 - u];
            fused::walk_blocks(W, L, part, 2, 4, fused::Lut{tab.lut_iq});
            fused::walk_finish(W, L, (t & 131071u) == 0, fix_errors, aggressive, tab, rec);
        } else if (lean == 2) {
            // the fused single sweep: direction and factors from the preamble words, then the
            // window in walk order (the kernel stages a backwards walk's words reversed)
            fused::Lane L;
            fused::phase_setup(win, odd, tab.lut_iq, 1u, 0xffffffffu, (uint32_t)-16384, L);
            uint32_t slots[fused::kSlots];
            for (int u = 0; u < fused::kSlots; u++) slots[u] = L.fwd ? win[8 + u] : win[120 - u];
            fused::evaluate(slots, L, (t & 131071u) == 0, fix_errors, aggressive, tab, fused::Lut{tab.lut_iq}, rec);
        } else if (lean) evaluate<true>(win, odd, (t & 131071u) == 0, fix_errors, aggressive, tab, rec);
        else evaluate<false>(win, odd, (t & 131071u) == 0, fix_errors, aggressive, tab, rec);
        std::memset(&out[c], 0, sizeof(out[c]));
        out[c].t = (int64_t)t;
        std::memcpy(&out[c].pass[0], rec, 24);
        std::memcpy(&out[c].pass[1], rec + 6, 24);
    }
    return 0;
}
