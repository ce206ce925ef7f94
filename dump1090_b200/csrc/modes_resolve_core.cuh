// modes_resolve_core.cuh — the sequential half of detectModeS() for ONE candidate: the rules both the
// host resolve (modes_resolve.cpp, stream order) and the device resolve (modes_resolve_gpu.cu: one
// warp per reference buffer) run.
//
// They read the few fields of a candidate record the order-dependent logic looks at:
//   * skip past a good message, retry with phase correction otherwise (dump1090.c:1769-1791);
//     the skip state restarts at every 131072-sample buffer (:1593)
//   * ICAO address cache: filled by clean DF11/17/18, consulted by the address/parity formats and
//     by DF11 with a small residual (dump1090.c:898-983, :1183-1210)
//   * statistics (dump1090.c:1651, :1662, :1738-1753, :1122-1126) and the sink gate (:1803)
// The running state is any type with next_j and stats[8] (the host's ResolveState, the device's
// BufferState).  The cache is reached through a small accessor so that the device version can keep
// it in shared memory and record which slots a buffer read before writing them (what its result
// depends on) and which it wrote (what later buffers inherit).
//
// tests/host_shim/resolve_core_host.cpp drives the device's per-buffer replay, the cache hand-over
// between buffers and the verify-and-repeat rounds on the CPU against the host resolver.  That build
// is test infrastructure.
#pragma once
#include <cstdint>
#include "modes_b200.h"

#if defined(__CUDACC__)
#define MODES_RCORE_FN __device__ __forceinline__
#else
#define MODES_RCORE_FN static inline
#endif

namespace modes {
namespace rcore {

// The fields of one evaluated attempt (modes_frame_eval) the sequential half uses.
struct Attempt {
    uint32_t meta;     // msgtype | flags << 8 | errorbit << 16 | nfixed << 24  (bytes 14..17 of modes_frame_eval)
    uint32_t crc;      // 24-bit syndrome after the repair
    uint32_t addr;     // msg[1] << 16 | msg[2] << 8 | msg[3]
};
// The rules read an attempt's fields through these, from an Attempt (the device's words) or straight
// from a record in memory (the host), where each field is then read only when a rule needs it.
MODES_RCORE_FN uint32_t a_msgtype(const Attempt &a) { return a.meta & 0xffu; }
MODES_RCORE_FN uint32_t a_flags(const Attempt &a) { return (a.meta >> 8) & 0xffu; }
MODES_RCORE_FN uint32_t a_nfixed(const Attempt &a) { return a.meta >> 24; }
MODES_RCORE_FN uint32_t a_crc(const Attempt &a) { return a.crc; }
MODES_RCORE_FN uint32_t a_addr(const Attempt &a) { return a.addr; }
MODES_RCORE_FN uint32_t a_msgtype(const modes_frame_eval &e) { return e.msgtype; }
MODES_RCORE_FN uint32_t a_flags(const modes_frame_eval &e) { return e.flags; }
MODES_RCORE_FN uint32_t a_nfixed(const modes_frame_eval &e) { return e.nfixed; }
MODES_RCORE_FN uint32_t a_crc(const modes_frame_eval &e) { return e.crc; }
MODES_RCORE_FN uint32_t a_addr(const modes_frame_eval &e) {
    return ((uint32_t)e.msg[1] << 16) | ((uint32_t)e.msg[2] << 8) | (uint32_t)e.msg[3];
}

// What the sequential half decides about one attempt.
struct Decision {
    uint32_t deliver;          // handed to the sink (dump1090.c:1803)
    uint32_t crcok, phase_corrected;
    uint32_t extra;            // DF11 interrogator id, or the recovered address of an address/parity format (0: none)
    uint32_t extra_is_ap;
};

// The device's per-buffer running state.  stats[] in the reference's order (modes_stats).
struct BufferState {
    uint32_t next_j;
    uint32_t stats[8];
};

MODES_RCORE_FN uint32_t icao_slot(uint32_t a) {                        // dump1090.c:898-905
    a = ((a >> 16) ^ a) * 0x45d9f3bu;
    a = ((a >> 16) ^ a) * 0x45d9f3bu;
    a = (a >> 16) ^ a;
    return a & 1023u;
}

MODES_RCORE_FN uint32_t bits_by_type(uint32_t df) { return (df >= 16 && df <= 21) ? 112u : 56u; }

// Cache: any type with  uint32_t read(uint32_t slot)  and  void write(uint32_t slot, uint32_t addr).
template <class Cache>
MODES_RCORE_FN bool seen(Cache &c, uint32_t a) { return a != 0 && c.read(icao_slot(a)) == a; }   // dump1090.c:919-925, TTL not modelled

// decodeModesMessage's order-dependent verdict for one attempt (dump1090.c:1108-1128, :1183-1210).
template <class State, class Cache, class A>
MODES_RCORE_FN uint32_t judge(State &st, Cache &c, const A &p, Decision &d) {
    d.extra = 0; d.extra_is_ap = 0;
    const uint32_t nfixed = a_nfixed(p), df = a_msgtype(p), crc = a_crc(p);
    if (nfixed == 1) st.stats[6]++;                                    // dump1090.c:1122-1126
    else if (nfixed == 2) st.stats[7]++;
    uint32_t crcok = crc == 0;
    if (df == 11 || df == 17 || df == 18) {
        const uint32_t addr = a_addr(p);
        if (crcok && nfixed == 0) c.write(icao_slot(addr), addr);      // :1198-1200
        if (df == 11 && !crcok && crc < 80 && seen(c, addr)) {         // :1204-1209
            d.extra = crc;
            crcok = 1;
        }
        return crcok;
    }
    // parity field = CRC ^ address, so the syndrome is the sender's address (:962-974)
    if ((df == 0 || df == 4 || df == 5 || df == 16 || df == 20 || df == 21 || df == 24) && seen(c, crc)) {
        d.extra = crc; d.extra_is_ap = 1;
        return 1;
    }
    return 0;
}

// One evaluated attempt, as detectModeS handles it after the delta gate.  Returns "good".
template <class State, class Cache, class A>
MODES_RCORE_FN bool attempt(State &st, Cache &c, const A &p, bool retry, int check_crc, Decision &d) {
    d.deliver = 0; d.crcok = 0; d.phase_corrected = 0; d.extra = 0; d.extra_is_ap = 0;
    if (!(a_flags(p) & MODES_EVAL_DECODED)) return false;
    const uint32_t crcok = judge(st, c, p, d);
    if (crcok || retry) {                                              // dump1090.c:1738-1753
        if (!(a_flags(p) & MODES_EVAL_ERRORS)) st.stats[2]++;
        if (a_nfixed(p) == 0) st.stats[crcok ? 3 : 4]++;
        else { st.stats[4]++; st.stats[5]++; st.stats[6]++; }
    }
    if (check_crc == 0 || crcok) {                                     // dump1090.c:1803; :1772-1773
        d.deliver = 1; d.crcok = crcok; d.phase_corrected = crcok && retry;
    }
    return crcok != 0;
}

// One candidate of the buffer whose state is `st`: j = its position inside the buffer.  d[0] / d[1]
// say what happens to its first attempt / its retry.  Returns -1 when j lies inside a message already
// taken (the candidate is not visited), 1 when one of its attempts was good, 0 otherwise.
template <class State, class Cache, class A>
MODES_RCORE_FN int candidate(State &st, Cache &c, uint32_t j, const A &p1, const A &p2, int check_crc,
                             Decision d[2]) {
    d[0].deliver = 0; d[1].deliver = 0;
    if (j < st.next_j) return -1;                                      // inside a message already taken
    st.stats[0]++;                                                     // dump1090.c:1651
    if (!(a_flags(p1) & MODES_EVAL_GATE_OK)) return 0;                 // dump1090.c:1723-1726
    if (attempt(st, c, p1, false, check_crc, d[0])) {
        st.next_j = j + (8 + bits_by_type(a_msgtype(p1))) * 2 + 1;
        return 1;
    }
    if (j) st.stats[1]++;                                              // dump1090.c:1660-1663
    if (!(a_flags(p2) & MODES_EVAL_GATE_OK)) return 0;
    if (!attempt(st, c, p2, true, check_crc, d[1])) return 0;
    st.next_j = j + (8 + bits_by_type(a_msgtype(p2))) * 2 + 1;
    return 1;
}

// The fields above from a candidate record in memory (little-endian).
MODES_RCORE_FN Attempt attempt_of(const modes_frame_eval &e) {
    Attempt a;
    a.meta = (uint32_t)e.msgtype | ((uint32_t)e.flags << 8) | ((uint32_t)e.errorbit << 16) | ((uint32_t)e.nfixed << 24);
    a.crc = e.crc;
    a.addr = a_addr(e);
    return a;
}

}  // namespace rcore
}  // namespace modes
