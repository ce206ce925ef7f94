"""Soft-decision recovery (modes_set_recovery) restated in numpy, and the resolve rules 1-6 of
include/modes_b200.h restated in Python.  TEST INFRASTRUCTURE, also used by scripts/recover_gain.py.

The restatement works from the raw stream bytes: for a candidate record with position t (buffer
k = t >> 17, j = t & 131071) the window's magnitudes are m[s + 16 + 2i] and m[s + 17 + 2i], i < 112,
with s = 131072 k + j - 238 the stream sample of the candidate's m[j] (samples before the stream's
start and after its end are the reference's 127 padding: magnitude 0).  The subset syndromes are
built by doubling, syn[:, 2^k : 2^(k+1)] = syn[:, :2^k] ^ bit_syn[P[:, k]]."""
from __future__ import annotations

import math

import numpy as np

import checker as C
from dump1090_b200 import api, synth

BUF = api.BUFFER_BYTES
K = api.RECOVER_BITS
SPAN = 241                                   # (8 + 112) * 2 + 1


def _mag_table():
    i, q = np.meshgrid(np.arange(129), np.arange(129), indexing="ij")
    return np.floor(np.sqrt((i * i + q * q).astype(np.float64)) * 360 + 0.5).astype(np.int64)


MAG = _mag_table()


def magnitudes(iq) -> np.ndarray:
    a = np.abs(np.asarray(iq, dtype=np.uint8).reshape(-1, 2).astype(np.int64) - 127)
    return MAG[a[:, 0], a[:, 1]]


def _syndrome(frame: bytes) -> int:
    return synth.modes_parity(frame[:11]) ^ int.from_bytes(frame[11:14], "big")


def _bit_syndromes() -> np.ndarray:
    """Syndrome of each single set bit of a long frame, from the frame CRC itself."""
    out = np.zeros(112, dtype=np.int64)
    for i in range(112):
        f = bytearray(14)
        f[i >> 3] = 0x80 >> (i & 7)
        out[i] = _syndrome(bytes(f))
    return out


BIT_SYN = _bit_syndromes()
_SUBSET_W = np.array([bin(s).count("1") for s in range(1 << K)], dtype=np.int64)


def windows(mag: np.ndarray, t) -> tuple:
    """(a, c): (n, 112) first / second magnitudes of the candidates at record positions t."""
    t = np.asarray(t, dtype=np.int64)
    s = (t >> 17) * 131072 + (t & 131071) - 238
    idx = s[:, None] + 16 + np.arange(224)[None, :]
    ok = (idx >= 0) & (idx < mag.size)
    w = np.where(ok, mag[np.clip(idx, 0, max(mag.size - 1, 0))], 0)
    return w[:, 0::2], w[:, 1::2]


def restate(a: np.ndarray, c: np.ndarray) -> np.ndarray:
    """The recovery records (RECOVERED_DTYPE) of windows a, c."""
    n = a.shape[0]
    out = np.zeros(n, dtype=api.RECOVERED_DTYPE)
    if not n:
        return out
    bits = (a > c).astype(np.uint8)
    frames = np.packbits(bits, axis=1)                                   # (n, 14), bit 0 = MSB of byte 0
    df = frames[:, 0] >> 3
    s0 = np.bitwise_xor.reduce(np.where(bits.astype(bool), BIT_SYN[None, :], 0), axis=1)
    sq = np.maximum(a, c).astype(np.int64) ** 2
    out["signal"] = [math.isqrt(int(v) // 112) for v in sq.sum(axis=1)]
    out["msg"] = frames
    elig = np.flatnonzero((df == 17) | (df == 18))
    out["status"] = api.RECOVER_INELIGIBLE
    if elig.size:
        w = np.abs(a[elig].astype(np.int64) - c[elig])[:, 5:112]
        keys = (w << 7) | np.arange(5, 112)[None, :]
        P = np.sort(keys, axis=1)[:, :K] & 127                            # (m, 10), by (w, i)
        syn = np.zeros((elig.size, 1 << K), dtype=np.int64)
        for k in range(K):
            syn[:, 1 << k: 2 << k] = syn[:, : 1 << k] ^ BIT_SYN[P[:, k]][:, None]
        sol = syn == s0[elig][:, None]
        wsol = np.where(sol, _SUBSET_W[None, :], 99)
        minw = wsol.min(axis=1)
        count = (wsol == minw[:, None]).sum(axis=1)
        status = np.where(minw == 99, api.RECOVER_NOT_FOUND, np.where(count == 1, api.RECOVER_FOUND, api.RECOVER_AMBIGUOUS))
        out["status"][elig] = status
        out["nflips"][elig] = np.where(status == api.RECOVER_NOT_FOUND, 0, minw)
        for r in np.flatnonzero(status == api.RECOVER_FOUND):
            subset = int(np.argmax(wsol[r] == minw[r]))
            b = bits[elig[r]].copy()
            for k in range(K):
                if (subset >> k) & 1:
                    b[P[r, k]] ^= 1
            out["msg"][elig[r]] = np.packbits(b)
    return out


def restate_records(data, t) -> np.ndarray:
    a, c = windows(magnitudes(data), t)
    return restate(a, c)


# ---------------------------------------------------------------- the resolve rules


def _icao_slot(a: int) -> int:
    m = 0xFFFFFFFF
    a = (((a >> 16) ^ a) * 0x45D9F3B) & m
    a = (((a >> 16) ^ a) * 0x45D9F3B) & m
    a = (a >> 16) ^ a
    return a & 1023


def model(off_msgs, cands, recovered, check_crc=1, signal=True):
    """Rules 1-6 over candidate records in stream order (cands, recovered: parallel arrays) and the
    messages of the recovery-off resolve: (messages as (sample_pos, frame bytes, nflips, signal) for
    recovered ones and Message objects for the reference's, in delivery order; statistics)."""
    st = dict.fromkeys(api.RECOVERY_STAT_NAMES, 0)
    good = {}                                               # sample_pos -> skip of the crcok message there
    for m in off_msgs:
        if m.crcok:
            good[int(m.sample_pos)] = (8 + m.msgbits) * 2 + 1
    # the reference's messages by position, and the cache writes they make
    by_pos = {}
    for m in off_msgs:
        by_pos.setdefault(int(m.sample_pos), []).append(m)
    order = np.argsort(cands["t"], kind="stable")
    cache = [0] * 1024
    out = []
    emitted = set()
    cur_buffer, next_j, next_rec, pending = -1, 0, 0, None

    def emit_reference(pos):
        for m in by_pos.get(pos, []):
            out.append(m)
            if m.crc == 0 and m.nfixed == 0 and m.msgtype in (11, 17, 18):
                a = (m.msg[1] << 16) | (m.msg[2] << 8) | m.msg[3]
                cache[_icao_slot(a)] = a
        emitted.add(pos)

    for idx in order:
        t = int(cands["t"][idx])
        buffer, j = t >> 17, t & 131071
        pos = buffer * 131072 + j - 238
        if buffer != cur_buffer:
            cur_buffer, next_j, next_rec, pending = buffer, 0, 0, None
        if j < next_j:
            continue
        emit_reference(pos)
        if pos in good:
            next_j = j + good[pos]
            if pending is not None and pending[0] == buffer and j < pending[1]:
                out.remove(pending[2])
                st["dropped"] += 1
                st["delivered"] -= 1
                pending = None
            continue
        r = recovered[idx]
        if r["status"] == api.RECOVER_INELIGIBLE:
            continue
        st["considered"] += 1
        if j < next_rec:
            continue
        if r["status"] == api.RECOVER_AMBIGUOUS:
            st["ambiguous"] += 1
        if r["status"] != api.RECOVER_FOUND:
            continue
        st["found"] += 1
        frame = bytes(r["msg"])
        a = (frame[1] << 16) | (frame[2] << 8) | frame[3]
        if a == 0 or cache[_icao_slot(a)] != a:
            st["unknown_address"] += 1
            continue
        entry = (pos, frame, int(r["nflips"]), int(r["signal"]) if signal else 0)
        out.append(entry)
        pending = (buffer, j + SPAN, entry)
        next_rec = j + SPAN
        st["delivered"] += 1
    assert emitted >= set(by_pos), "a reference message at a position the walk never reached"
    return out, st


# ---------------------------------------------------------------- the CPU path


def flag_cfg(kw):
    return dict(fix_errors=kw.get("fix", 1), aggressive=kw.get("aggressive", 0), check_crc=kw.get("check_crc", 1))


def tiled(sel, n_buffers):
    g = (sel["t"] + 2) // api.TILE_SAMPLES
    nt = api.tiles_for(n_buffers)
    cnt = np.bincount(g, minlength=nt).astype(np.uint32)
    t = np.zeros(nt, dtype=api.TILE_DTYPE)
    t["count"] = cnt
    t["offset"] = np.concatenate([[0], np.cumsum(cnt)[:-1]])
    return t


def oracle_records(data, kw, drop_eof=0):
    recs = C.oracle_scan_candidates(data, fix=kw.get("fix", 1), aggressive=kw.get("aggressive", 0), drop_eof=drop_eof,
                                    cap=max(400000, np.asarray(data).size // 50))
    return np.frombuffer(b"".join(bytes(c) for c in recs), dtype=api.CANDIDATE_DTYPE).copy()


def cpu_decode(data, kw, drop_eof=0, signal=False):
    """The host half over the oracle's records and the restated recovery records: (messages,
    reference statistics, recovery statistics, candidate records, recovery records)."""
    data = np.asarray(data, dtype=np.uint8)
    arr = oracle_records(data, kw, drop_eof)
    nbuf = data.size // BUF + (0 if drop_eof else 1)
    rec = restate_records(data, arr["t"])
    if not signal:
        rec["signal"] = 0
    res = api.Resolver(**flag_cfg(kw))
    res.run(arr, tiled(arr, max(nbuf, 1)), recovered=rec)
    return res.take_messages(), res.stats(), res.recovery_stats(), arr, rec
