"""Weak preambles (modes_set_weak_preambles) restated in numpy, and the resolve rules with weak
positions merged into the walk restated in Python.  TEST INFRASTRUCTURE, also used by
scripts/recover_gain.py.

A batch of n_buffers reference buffers has positions t = 131072 k + j, j < 131070; the magnitude m[j+x]
of position t is stream sample t - 238 + x (recover_model's convention), 0 outside the stream (the
reference's 127 padding)."""
from __future__ import annotations

import numpy as np

import recover_model as R
from dump1090_b200 import api

BUF = api.BUFFER_BYTES
WINDOW = 26


def padded_mags(data, n_buffers: int) -> np.ndarray:
    """M with M[t + x] = m[j + x] of position t, for every position of n_buffers buffers."""
    mag = R.magnitudes(np.asarray(data, dtype=np.uint8)[: 2 * (np.asarray(data).size // 2)])
    n = n_buffers * 131072
    out = np.zeros(238 + n + WINDOW + 8, dtype=np.int64)
    k = min(mag.size, n + WINDOW)
    out[238: 238 + k] = mag[:k]
    return out


def conditions(W: np.ndarray):
    """(weak, shape and contrast, reference test) of windows W[:, 0..25] of magnitudes."""
    g = lambda x: W[:, x].astype(np.int64)
    shape = (g(0) > g(1)) & (g(2) > g(1)) & (g(7) > g(8)) & (g(9) > g(8))
    quiet = g(4) + g(5) + g(6) + g(11) + g(12) + g(13) + g(14)
    contrast = 7 * (g(0) + g(2) + g(7) + g(9)) > 8 * quiet
    df = np.zeros(W.shape[0], dtype=np.int64)
    for i in range(5):
        df = (df << 1) | (g(16 + 2 * i) > g(17 + 2 * i))
    ref = (g(0) > g(1)) & (g(1) < g(2)) & (g(2) > g(3)) & (g(3) < g(0)) & (g(4) < g(0)) & (g(5) < g(0)) & (g(6) < g(0)) \
        & (g(7) > g(8)) & (g(8) < g(9)) & (g(9) > g(6))
    high = (g(0) + g(2) + g(7) + g(9)) // 6
    for x in (4, 5, 11, 12, 13, 14):
        ref &= g(x) < high
    weak = shape & contrast & ((df == 17) | (df == 18)) & ~ref
    return weak, shape & contrast, ref


def window_mags(iq_windows: np.ndarray) -> np.ndarray:
    """(n, 52) raw windows -> (n, 26) magnitudes."""
    return R.magnitudes(np.ascontiguousarray(iq_windows, dtype=np.uint8).reshape(-1)).reshape(-1, WINDOW)


def _scan(data, n_buffers: int, which: int) -> np.ndarray:
    M = padded_mags(data, n_buffers)
    out = []
    step = 1 << 17
    for t0 in range(0, n_buffers * 131072, step):
        t = np.arange(t0, t0 + step, dtype=np.int64)
        t = t[(t & 131071) < 131070]
        W = M[t[:, None] + np.arange(WINDOW)[None, :]]
        out.append(t[conditions(W)[which]])
    return np.concatenate(out).astype(np.uint32) if out else np.zeros(0, np.uint32)


def weak_positions(data, n_buffers: int) -> np.ndarray:
    """The weak positions of a batch of n_buffers buffers, in stream order."""
    return _scan(data, n_buffers, 0)


def reference_positions(data, n_buffers: int) -> np.ndarray:
    """The positions that pass the reference's preamble test (the scan's candidates)."""
    return _scan(data, n_buffers, 2)


def weak_records(data, t) -> np.ndarray:
    return R.restate_records(np.asarray(data, dtype=np.uint8), np.asarray(t, dtype=np.int64))


# ---------------------------------------------------------------- the merged resolve rules


def model(off_msgs, cands, recovered, weak_t, weak_rec, check_crc=1, signal=True):
    """recover_model.model with the weak positions merged into the walk: (messages, candidate recovery
    statistics, weak statistics).  A recovered message is (sample_pos, frame, nflips, signal, marker)."""
    st = dict.fromkeys(api.RECOVERY_STAT_NAMES, 0)
    wst = dict.fromkeys(api.RECOVERY_STAT_NAMES, 0)
    good = {int(m.sample_pos): (8 + m.msgbits) * 2 + 1 for m in off_msgs if m.crcok}
    by_pos = {}
    for m in off_msgs:
        by_pos.setdefault(int(m.sample_pos), []).append(m)
    events = [(int(cands["t"][i]), 0, i) for i in range(cands.size)] + [(int(weak_t[i]), 1, i) for i in range(len(weak_t))]
    events.sort()
    cache = [0] * 1024
    out, emitted = [], set()
    cur_buffer, next_j, next_rec, pending = -1, 0, 0, None

    def emit_reference(pos):
        for m in by_pos.get(pos, []):
            out.append(m)
            if m.crc == 0 and m.nfixed == 0 and m.msgtype in (11, 17, 18):
                a = (m.msg[1] << 16) | (m.msg[2] << 8) | m.msg[3]
                cache[R._icao_slot(a)] = a
        emitted.add(pos)

    for t, is_weak, idx in events:
        buffer, j = t >> 17, t & 131071
        pos = buffer * 131072 + j - 238
        if buffer != cur_buffer:
            cur_buffer, next_j, next_rec, pending = buffer, 0, 0, None
        if j < next_j:
            continue
        if not is_weak:
            emit_reference(pos)
            if pos in good:
                next_j = j + good[pos]
                if pending is not None and pending[0] == buffer and j < pending[1]:
                    out.remove(pending[2])
                    pending[3]["dropped"] += 1
                    pending[3]["delivered"] -= 1
                    pending = None
                continue
        r = weak_rec[idx] if is_weak else recovered[idx]
        s = wst if is_weak else st
        if r["status"] == api.RECOVER_INELIGIBLE:
            continue
        s["considered"] += 1
        if j < next_rec:
            continue
        if r["status"] == api.RECOVER_AMBIGUOUS:
            s["ambiguous"] += 1
        if r["status"] != api.RECOVER_FOUND:
            continue
        s["found"] += 1
        frame = bytes(r["msg"])
        a = (frame[1] << 16) | (frame[2] << 8) | frame[3]
        if a == 0 or cache[R._icao_slot(a)] != a:
            s["unknown_address"] += 1
            continue
        entry = (pos, frame, int(r["nflips"]), int(r["signal"]) if signal else 0, 2 if is_weak else 1)
        out.append(entry)
        pending = (buffer, j + R.SPAN, entry, s)
        next_rec = j + R.SPAN
        s["delivered"] += 1
    assert emitted >= set(by_pos), "a reference message at a position the walk never reached"
    return out, st, wst


def as_rows(msgs):
    """Messages as model() lists them."""
    return [(int(m.sample_pos), bytes(m.msg), int(m.nfixed), int(m.signal), int(m.recovered)) if m.recovered else bytes(m)
            for m in msgs]


def model_rows(rows):
    return [w if isinstance(w, tuple) else bytes(w) for w in rows]


# ---------------------------------------------------------------- the CPU path


def cpu_decode(data, kw, drop_eof=0, signal=False):
    """The host half over the oracle's records, the restated recovery records and the restated weak
    positions and records: (messages, reference statistics, recovery statistics, weak statistics,
    candidates, recovery records, weak positions, weak records)."""
    data = np.asarray(data, dtype=np.uint8)
    arr = R.oracle_records(data, kw, drop_eof)
    nbuf = max(data.size // BUF + (0 if drop_eof else 1), 1)
    rec = R.restate_records(data, arr["t"])
    wt = weak_positions(data if not drop_eof else data[: (data.size // BUF) * BUF], nbuf)
    wr = weak_records(data if not drop_eof else data[: (data.size // BUF) * BUF], wt)
    if not signal:
        rec["signal"] = 0
        wr["signal"] = 0
    res = api.Resolver(**R.flag_cfg(kw))
    res.run(arr, R.tiled(arr, nbuf), recovered=rec, weak=(wt, wr))
    return res.take_messages(), res.stats(), res.recovery_stats(), res.weak_stats(), arr, rec, wt, wr
