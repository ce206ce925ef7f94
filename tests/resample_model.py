"""The 2.4 MS/s -> 2 MHz resampler restated in numpy: the tap derivation and the whole arithmetic of
dump1090_b200/csrc/modes_resample_core.cuh (include/modes_b200.h, modes_set_input_rate).

Input: UC8 I/Q at 2.4 MS/s, zero at 127; n_in = ceil(bytes / 2), a trailing odd byte is an I whose Q
is 127, and samples outside [0, n_in) read as (127, 127).  Output sample n = 5q + r (r = 0..4) has base
input index b = 6q + r and
    y = clamp(127 + ((sum_k h[r][k] * (x[b + k - T/2 + 1] - 127) + 8192) >> 14), 0, 255)
for I and Q separately (int32 sum, arithmetic shift).  The stream has N_out = ceil(5 n_in / 6) output
samples.  h[r][k] samples one symmetric Kaiser-windowed sinc prototype at the input offset
k - T/2 + 1 - 0.2 r (a whole number of 12 MHz ticks); each branch is scaled to sum 1, rounded to Q14
and its remainder put on its largest tap, so every branch sums to exactly 16384.
"""
from __future__ import annotations

import numpy as np

# The filter the product uses (DESIGN §3 K9, chosen by the sweep in DESIGN §6).
TAPS = 6
CUTOFF_HZ = 1.1e6
BETA = 5.0
IN_RATE = 2_400_000
Q = 14


def prototype(d, taps: int = TAPS, cutoff_hz: float = CUTOFF_HZ, beta: float = BETA) -> np.ndarray:
    """The low-pass prototype at input offsets d (2.4 MS/s samples, any real value): a sinc of the
    cutoff, Kaiser-windowed over +-taps/2 input samples.  Symmetric in d."""
    d = np.asarray(d, dtype=np.float64)
    half = taps / 2.0
    u = np.clip(1.0 - (d / half) ** 2, 0.0, None)
    w = np.i0(beta * np.sqrt(u)) / np.i0(beta)
    return np.where(np.abs(d) <= half, np.sinc(2.0 * cutoff_hz * d / IN_RATE) * w, 0.0)


def offsets(taps: int = TAPS) -> np.ndarray:
    """offsets()[r, k] = k - T/2 + 1 - 0.2 r, the input offset of tap k of branch r, in 12 MHz ticks / 5."""
    k = np.arange(taps)
    r = np.arange(5)[:, None]
    return (5 * (k - taps // 2 + 1) - r) / 5.0


def derive_taps(taps: int = TAPS, cutoff_hz: float = CUTOFF_HZ, beta: float = BETA) -> np.ndarray:
    """The (5, taps) int16 table: each branch of the prototype scaled to sum 1, rounded to Q14, and its
    rounding remainder put on its largest tap."""
    p = prototype(offsets(taps), taps, cutoff_hz, beta)
    g = p / p.sum(axis=1, keepdims=True)
    h = np.floor(g * (1 << Q) + 0.5).astype(np.int64)
    for r in range(5):
        h[r, int(np.argmax(h[r]))] += (1 << Q) - int(h[r].sum())
    assert (h.sum(axis=1) == 1 << Q).all()
    return h.astype(np.int16)


H = derive_taps()


def n_out(n_in: int) -> int:
    """Output samples of a stream of n_in input samples: those with 6n < 5 n_in."""
    return (5 * n_in + 5) // 6


def _samples(data) -> tuple[np.ndarray, np.ndarray]:
    a = np.frombuffer(data, dtype=np.uint8) if isinstance(data, (bytes, bytearray)) else np.asarray(data, dtype=np.uint8)
    if a.size % 2:
        a = np.concatenate([a, np.array([127], np.uint8)])
    s = a.reshape(-1, 2).astype(np.int64) - 127
    return s[:, 0], s[:, 1]


def resample_range(data, first: int, count: int, h: np.ndarray = H, limit: int | None = None) -> np.ndarray:
    """Output samples [first, first + count) of the stream `data` (2.4 MS/s bytes from its start) as I/Q
    bytes; first may be negative (those samples see only no-signal input).  Samples at or past `limit`
    are written as 127 (the EOF buffer's padding); None: no limit."""
    taps = h.shape[1]
    xi, xq = _samples(data)
    n = np.arange(first, first + count, dtype=np.int64)
    q, r = np.divmod(n, 5)
    b = 6 * q + r
    out = np.empty((count, 2), dtype=np.uint8)
    for ch, x in enumerate((xi, xq)):
        acc = np.zeros(count, dtype=np.int64)
        for k in range(taps):
            idx = b + k - taps // 2 + 1
            ok = (idx >= 0) & (idx < x.size)
            v = np.where(ok, x[np.clip(idx, 0, max(x.size - 1, 0))] if x.size else 0, 0)
            acc += h[r, k].astype(np.int64) * v
        assert np.abs(acc).max(initial=0) < 2 ** 31
        y = 127 + ((acc + 8192) >> Q)
        out[:, ch] = np.clip(y, 0, 255)
    if limit is not None:
        out[n >= limit] = 127
    return out.reshape(-1)


def resample(data, h: np.ndarray = H) -> np.ndarray:
    """The whole stream: N_out = ceil(5 n_in / 6) output samples, 2 N_out bytes."""
    n_in = (len(data) + 1) // 2
    return resample_range(data, 0, n_out(n_in), h)


def input_span(first: int, count: int, taps: int = TAPS) -> tuple[int, int]:
    """The input samples [lo, hi) that output samples [first, first + count) read."""
    lo = (6 * first) // 5 - taps // 2 + 1
    hi = (6 * (first + count - 1)) // 5 + taps // 2 + 1
    return lo, hi


class Streaming:
    """The model fed piecewise: it keeps only the input history later outputs need and emits every
    output sample as soon as its input has arrived, as a streaming decode does."""

    def __init__(self, h: np.ndarray = H):
        self.h = h
        self.hist = np.zeros(0, np.uint8)   # stream bytes [hist0, total)
        self.hist0 = 0
        self.total = 0
        self.done = 0                       # output samples emitted

    def _emit(self, count: int, limit=None) -> np.ndarray:
        # the history as a stream that starts at byte hist0 (hist0 is even): input index shifts by hist0 / 2
        first = self.done
        s0 = self.hist0 // 2
        # output n reads input 6n/5 ...: shift n so that the input index is relative to s0 (s0 a multiple of 6
        # is not guaranteed, so evaluate against a zero-prefixed view instead)
        lo, _ = input_span(first, count, self.h.shape[1])
        lo = max(lo, 0)
        assert lo >= s0
        view = np.concatenate([np.full(2 * s0, 127, np.uint8), self.hist])
        out = resample_range(view, first, count, self.h, limit)
        self.done += count
        keep_from = 2 * max(input_span(self.done, 1, self.h.shape[1])[0], 0)
        if keep_from > self.hist0:
            self.hist = self.hist[keep_from - self.hist0:]
            self.hist0 = keep_from
        return out

    def feed(self, piece) -> np.ndarray:
        self.hist = np.concatenate([self.hist, np.asarray(piece, np.uint8)])
        self.total += len(piece)
        avail = self.total // 2
        m = self.done
        while input_span(m, 1, self.h.shape[1])[1] <= avail:
            m += 1
        return self._emit(m - self.done) if m > self.done else np.zeros(0, np.uint8)

    def finish(self) -> np.ndarray:
        end = n_out((self.total + 1) // 2)
        if end <= self.done:
            return np.zeros(0, np.uint8)
        return self._emit(end - self.done)
