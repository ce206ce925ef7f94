"""The integer decimator (4, 6, 8 and 10 MS/s -> 2 MHz) restated in numpy: the tap derivation and the whole
arithmetic of dump1090_b200/csrc/modes_resample_core.cuh (include/modes_b200.h, modes_set_input_rate).

Input: UC8 I/Q at 2 M MS/s (M = 2, 3, 4, 5), zero at 127; n_in = ceil(bytes / 2), a trailing odd byte is
an I whose Q is 127, and samples outside [0, n_in) read as (127, 127).  A 16-bit stream is first converted
(tests/input_format_model.py).  Output sample n stands for input samples [M n, M n + M) and, for I and Q
separately,
    y = clamp(127 + ((sum_{k<T} h_M[k] * (x[M n - E + k] - 127) + 8192) >> 14), 0, 255)
with T = M + 2E (int32 sum, arithmetic shift).  The stream has N_out = ceil(n_in / M) output samples.

h_M is symmetric about input M n + (M - 1) / 2: the box (E = 0, every tap 1 / M) or a Kaiser-windowed sinc
over T taps, scaled to sum 1 and rounded to Q14, with the rounding remainder on the middle tap (split
evenly over the two middle taps when T is even), so that every table sums to exactly 16384.
"""
from __future__ import annotations

import numpy as np

Q = 14
RATES = {4_000_000: 2, 6_000_000: 3, 8_000_000: 4, 10_000_000: 5}
# The filter the product uses per M: (E, cutoff Hz or None for the box), chosen by the sweep in DESIGN §6
# (scripts/decimate_quality.py).
FILTER = {2: (2, 0.8e6), 3: (1, 0.8e6), 4: (2, 0.8e6), 5: (2, 0.8e6)}
BETA = 5.0


def derive_taps(m: int, e: int = 0, cutoff_hz: float | None = None, beta: float = BETA) -> np.ndarray:
    """The int16 table of T = m + 2e taps: the box (cutoff None, e = 0) or a Kaiser-windowed sinc of the
    cutoff over +-T/2 input samples about the table's centre, scaled to sum 1, rounded to Q14, and the
    remainder put on the middle tap (the two middle taps when T is even)."""
    t = m + 2 * e
    d = np.abs(np.arange(t) - (t - 1) / 2.0)                   # |offset| from the centre, in input samples
    if cutoff_hz is None:
        assert e == 0
        p = np.ones(t)
    else:
        fs = 2_000_000 * m
        u = np.clip(1.0 - (d / (t / 2.0)) ** 2, 0.0, None)
        p = np.sinc(2.0 * cutoff_hz * d / fs) * np.i0(beta * np.sqrt(u)) / np.i0(beta)
    g = p / p.sum()
    h = np.floor(g * (1 << Q) + 0.5).astype(np.int64)
    rem = (1 << Q) - int(h.sum())
    if t % 2:
        h[t // 2] += rem
    else:
        assert rem % 2 == 0
        h[t // 2 - 1] += rem // 2
        h[t // 2] += rem // 2
    assert h.sum() == 1 << Q and np.array_equal(h, h[::-1])
    return h.astype(np.int16)


def taps(m: int) -> np.ndarray:
    """The product's table for M = m."""
    e, fc = FILTER[m]
    return derive_taps(m, e, fc)


def extent(h: np.ndarray, m: int) -> int:
    """E of a table: the taps on each side of the output's M input samples."""
    return (h.size - m) // 2


def n_out(n_in: int, m: int) -> int:
    """Output samples of a stream of n_in input samples: ceil(n_in / M)."""
    return -(-n_in // m)


def _samples(data) -> tuple[np.ndarray, np.ndarray]:
    a = np.frombuffer(data, dtype=np.uint8) if isinstance(data, (bytes, bytearray)) else np.asarray(data, dtype=np.uint8)
    if a.size % 2:
        a = np.concatenate([a, np.array([127], np.uint8)])
    s = a.reshape(-1, 2).astype(np.int64) - 127
    return s[:, 0], s[:, 1]


def decimate_range(data, m: int, first: int, count: int, h: np.ndarray | None = None, limit: int | None = None,
                   in_first: int = 0) -> np.ndarray:
    """Output samples [first, first + count) as I/Q bytes, of the stream whose input samples from in_first on
    are `data` (UC8 bytes) and whose every other input sample is no signal; first may be negative.  Samples
    at or past `limit` are 127 (the EOF buffer's padding); None: no limit."""
    h = taps(m) if h is None else h
    e = extent(h, m)
    xi, xq = _samples(data)
    n = np.arange(first, first + count, dtype=np.int64)
    out = np.empty((count, 2), dtype=np.uint8)
    for ch, x in enumerate((xi, xq)):
        acc = np.zeros(count, dtype=np.int64)
        for k in range(h.size):
            idx = m * n - e + k - in_first
            ok = (idx >= 0) & (idx < x.size)
            v = np.where(ok, x[np.clip(idx, 0, max(x.size - 1, 0))] if x.size else 0, 0)
            acc += int(h[k]) * v
        assert np.abs(acc).max(initial=0) < 2 ** 31
        out[:, ch] = np.clip(127 + ((acc + 8192) >> Q), 0, 255)
    if limit is not None:
        out[n >= limit] = 127
    return out.reshape(-1)


def decimate(data, m: int, h: np.ndarray | None = None) -> np.ndarray:
    """The whole stream: N_out = ceil(n_in / M) output samples, 2 N_out bytes."""
    n_in = (len(data) + 1) // 2
    return decimate_range(data, m, 0, n_out(n_in, m), h)


def input_span(first: int, count: int, m: int, h: np.ndarray | None = None) -> tuple[int, int]:
    """The input samples [lo, hi) that output samples [first, first + count) read."""
    e = extent(taps(m) if h is None else h, m)
    return m * first - e, m * (first + count) + e


def upsample(data, m: int) -> np.ndarray:
    """Each I/Q sample of a UC8 stream repeated m times: the stream at 2 m MS/s whose box decimation is
    the stream itself."""
    a = np.asarray(data, dtype=np.uint8).reshape(-1, 2)
    return np.repeat(a, m, axis=0).reshape(-1)


class Streaming:
    """The model fed piecewise: it keeps only the input history later outputs need and emits every output
    sample as soon as its input has arrived, as a streaming decode does."""

    def __init__(self, m: int, h: np.ndarray | None = None):
        self.m = m
        self.h = taps(m) if h is None else h
        self.hist = np.zeros(0, np.uint8)   # stream bytes [2 hist0, total)
        self.hist0 = 0                      # in input samples
        self.total = 0
        self.done = 0                       # output samples emitted

    def _emit(self, count: int) -> np.ndarray:
        out = decimate_range(self.hist, self.m, self.done, count, self.h, in_first=self.hist0)
        self.done += count
        keep = max(input_span(self.done, 1, self.m, self.h)[0], 0)
        if keep > self.hist0:
            self.hist = self.hist[2 * (keep - self.hist0):]
            self.hist0 = keep
        return out

    def feed(self, piece) -> np.ndarray:
        self.hist = np.concatenate([self.hist, np.asarray(piece, np.uint8)])
        self.total += len(piece)
        avail = self.total // 2
        m = self.done
        while input_span(m, 1, self.m, self.h)[1] <= avail:
            m += 1
        return self._emit(m - self.done) if m > self.done else np.zeros(0, np.uint8)

    def finish(self) -> np.ndarray:
        end = n_out((self.total + 1) // 2, self.m)
        if end <= self.done:
            return np.zeros(0, np.uint8)
        return self._emit(end - self.done)
