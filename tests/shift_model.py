"""The frequency shift in front of the decimator (modes_set_input_offset) restated in numpy: the derivation
of its Q14 tables and the whole arithmetic of shift::shift_group in dump1090_b200/csrc/modes_resample_core.cuh.

A 4-10 MS/s capture whose radio was tuned off 1090 MHz has the channel at offset_hz in its baseband.  Input
sample m (counted from the stream's start; a 16-bit stream converted first, tests/input_format_model.py)
with xi = I - 127, xq = Q - 127 (0 outside the stream) is rotated by e^{-j 2 pi offset m / fs}:

    step   = round(offset_hz 2^32 / fs)                 (int64 arithmetic, stored as uint32)
    theta  = (m step) mod 2^32                          (m mod 2^32 first)
    k      = ((theta + 2^21) >> 22) & 1023              (the nearest of 1024 phases)
    u_i    = (xi C[k] + xq S[k] + 8192) >> 14           (int32, arithmetic shift)
    u_q    = (xq C[k] - xi S[k] + 8192) >> 14
    y      = clamp(127 + ((sum_{k<T} h_M[k] u[M n - E + k] + 8192) >> 14), 0, 255)    I and Q separately

with C[k] = round(16384 cos(2 pi k / 1024)), S[k] = round(16384 sin(2 pi k / 1024)) and h_M, E, T the
decimator's (tests/decimate_model.py).  At offset 0, u = x and y is the decimator's output.
"""
from __future__ import annotations

import numpy as np

import decimate_model as DM

PHASES = 1024


def derive_tables() -> tuple[np.ndarray, np.ndarray]:
    """C and S: Q14 cos and sin of the 1024 phases, rounded to nearest (no value is a tie)."""
    a = 2 * np.pi * np.arange(PHASES) / PHASES
    c = np.floor(16384 * np.cos(a) + 0.5).astype(np.int64)
    s = np.floor(16384 * np.sin(a) + 0.5).astype(np.int64)
    return c, s


C, S = derive_tables()


def max_offset(fs: int) -> int:
    """The largest |offset_hz| the decoder takes at fs: fs / 2 - 1 MHz at 4-10 MS/s, 0 elsewhere."""
    return fs // 2 - 1_000_000 if fs in DM.RATES else 0


def step(offset_hz: int, fs: int) -> int:
    """round(offset_hz 2^32 / fs) as uint32.  fs / 2^k is odd at every rate, so there is no tie."""
    return ((int(offset_hz) * (1 << 33) + fs) // (2 * fs)) % (1 << 32)


def applied_hz(offset_hz: int, fs: int) -> float:
    """The shift actually applied: step fs / 2^32, taken as a signed step."""
    st = step(offset_hz, fs)
    return (st - (1 << 32) if st >= 1 << 31 else st) * fs / 2 ** 32


def phases(m0: int, count: int, st: int) -> np.ndarray:
    """k of stream samples m0 .. m0 + count - 1."""
    m = (np.arange(m0, m0 + count, dtype=np.int64) % (1 << 32)).astype(np.uint64)
    theta = (m * np.uint64(st)) % np.uint64(1 << 32)
    return (((theta + np.uint64(1 << 21)) >> np.uint64(22)) & np.uint64(PHASES - 1)).astype(np.int64)


def rotate(xi: np.ndarray, xq: np.ndarray, k: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """u_i, u_q of samples (xi, xq) at phases k."""
    c, s = C[k], S[k]
    return (xi * c + xq * s + 8192) >> 14, (xq * c - xi * s + 8192) >> 14


def shift_decimate_range(data, m: int, offset_hz: int, first: int, count: int, limit: int | None = None,
                         in_first: int = 0) -> np.ndarray:
    """decimate_model.decimate_range with the input rotated: output samples [first, first + count) as I/Q
    bytes of the stream whose input samples from in_first on are `data` (UC8 bytes), every other input
    sample no signal; samples at or past `limit` are 127."""
    h = DM.taps(m)
    e = DM.extent(h, m)
    xi, xq = DM._samples(data)
    k = phases(in_first, xi.size, step(offset_hz, 2_000_000 * m))
    ui, uq = rotate(xi, xq, k)
    assert max(np.abs(ui).max(initial=0), np.abs(uq).max(initial=0)) <= 182
    n = np.arange(first, first + count, dtype=np.int64)
    out = np.empty((count, 2), dtype=np.uint8)
    for ch, u in enumerate((ui, uq)):
        acc = np.zeros(count, dtype=np.int64)
        for t in range(h.size):
            idx = m * n - e + t - in_first
            ok = (idx >= 0) & (idx < u.size)
            v = np.where(ok, u[np.clip(idx, 0, max(u.size - 1, 0))] if u.size else 0, 0)
            acc += int(h[t]) * v
        assert np.abs(acc).max(initial=0) < 2 ** 31
        out[:, ch] = np.clip(127 + ((acc + 8192) >> 14), 0, 255)
    if limit is not None:
        out[n >= limit] = 127
    return out.reshape(-1)


def shift_decimate(data, m: int, offset_hz: int) -> np.ndarray:
    """The whole stream: N_out = ceil(n_in / M) output samples, 2 N_out bytes."""
    n_in = (len(data) + 1) // 2
    return shift_decimate_range(data, m, offset_hz, 0, DM.n_out(n_in, m))
