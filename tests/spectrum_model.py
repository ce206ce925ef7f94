"""The input spectrum pass (modes_set_spectrum, K13) restated in numpy: the arithmetic of
dump1090_b200/csrc/modes_spectrum_core.cuh and the records a decode gives from a stream's raw bytes.

Reference buffer b stands for input samples [s_b, s_{b+1}), s_b = floor(in b B / out) at the rate's ratio
out : in; its F = floor((s_{b+1} - s_b) / 256) whole frames of 256 samples start at s_b.  A sample is
x = (I - 127, Q - 127) of the UC8 bytes (a 16-bit stream converted first, tests/input_format_model.py), 0 past
the stream's end.  Per frame (int32, arithmetic shifts):
    v[n]  = (x[n] w[n] + 8192) >> 14,  w[n] = (16384 - C[4 n]) >> 1
    radix-2 DIT over the bit-reversed frame, stage s (half = 2^s), k = (i mod half) 2^(7-s), c = C[4k], s = S[4k]:
        t_re = (b_re c + b_im s + 8192) >> 14,  t_im = (b_im c - b_re s + 8192) >> 14,  a + t, a - t
    P[m]  = X_re[m]^2 + X_im[m]^2
and record bin i sums P[(i + 128) mod 256] over the frames.  C and S: tests/shift_model.py.
"""
from __future__ import annotations

import numpy as np

import input_format_model as IF
import shift_model as SM

N = 256
B = 131072                                 # MODES_BUFFER_SAMPLES
RATIOS = {2_000_000: (1, 1), 2_400_000: (5, 6), 4_000_000: (1, 2), 6_000_000: (1, 3), 8_000_000: (1, 4),
          10_000_000: (1, 5)}
WINDOW = (16384 - SM.C[4 * np.arange(N)]) >> 1
DTYPE = np.dtype([("buffer", "<i8"), ("frames", "<u4"), ("pad", "<u4"), ("power", "<u8", (N,))])   # api.SPECTRUM_DTYPE
BITREV = np.array([int(f"{n:08b}"[::-1], 2) for n in range(N)])


def first_sample(rate: int, b: int) -> int:
    out, inp = RATIOS[rate]
    return inp * b * B // out


def frames(rate: int, b: int) -> int:
    return (first_sample(rate, b + 1) - first_sample(rate, b)) // N


def frame_power(x: np.ndarray) -> np.ndarray:
    """x: int array [..., 256, 2] of (I - 127, Q - 127) -> uint64 [..., 256] power in record bin order."""
    x = np.asarray(x, dtype=np.int64)
    v = (x * WINDOW[:, None] + 8192) >> 14
    re = v[..., BITREV, 0].copy()
    im = v[..., BITREV, 1].copy()
    for st in range(8):
        half = 1 << st
        i = np.array([j for j in range(N) if not j & half])
        k = (i & (half - 1)) << (7 - st)
        c, s = SM.C[4 * k], SM.S[4 * k]
        ar, ai, br, bi = re[..., i], im[..., i], re[..., i + half], im[..., i + half]
        tr = (br * c + bi * s + 8192) >> 14
        ti = (bi * c - br * s + 8192) >> 14
        re[..., i], im[..., i] = ar + tr, ai + ti
        re[..., i + half], im[..., i + half] = ar - tr, ai - ti
    p = (re * re + im * im).astype(np.uint64)
    return np.roll(p, N // 2, axis=-1)                                   # bin i = P[(i + 128) mod 256]


def samples(data, fmt: str = "uc8", shift: int | None = None) -> np.ndarray:
    """The stream's samples as int64 [n_in, 2] of (I - 127, Q - 127) (16-bit converted; a trailing odd UC8
    byte is an I whose Q is 127)."""
    a = np.frombuffer(data, np.uint8) if isinstance(data, (bytes, bytearray)) else np.asarray(data, np.uint8)
    if fmt != "uc8":
        a = IF.convert(a, IF.DEFAULT_SHIFT[fmt] if shift is None else shift)
    elif a.size % 2:
        a = np.concatenate([a, np.array([127], np.uint8)])
    return a.reshape(-1, 2).astype(np.int64) - 127


def record(x: np.ndarray, rate: int, b: int, x_first: int = 0) -> np.ndarray:
    """The record of buffer b from the samples x (stream sample x_first at x[0]; 0 outside)."""
    s0, f = first_sample(rate, b), frames(rate, b)
    lo = s0 - x_first
    fr = np.zeros((f * N, 2), dtype=np.int64)
    a, e = max(lo, 0), min(lo + f * N, x.shape[0])
    if e > a:
        fr[a - lo: e - lo] = x[a:e]
    out = np.zeros(1, dtype=DTYPE)
    out["buffer"], out["frames"] = b, f
    out["power"][0] = frame_power(fr.reshape(f, N, 2)).sum(axis=0, dtype=np.uint64) if f else 0
    return out[0]


def n_buffers(nbytes: int, rate: int, fmt: str, drop_eof: int = 0) -> int:
    """Buffers a streaming decode of nbytes decodes: the whole ones, then the EOF buffer unless dropped."""
    if rate == 2_000_000 and fmt == "uc8":
        whole = nbytes // (2 * B)
    else:
        n_in = (nbytes + 1) // 2 if fmt == "uc8" else nbytes // 4
        out, inp = RATIOS[rate]
        whole = (out * n_in + inp - 1) // inp // B
    return whole + (0 if drop_eof else 1)


def expected(data, rate: int = 2_000_000, fmt: str = "uc8", shift: int | None = None, drop_eof: int = 0,
             first: int = 0) -> np.ndarray:
    """The records a streaming decode of `data` gives, buffers first ... (records of earlier ones dropped)."""
    x = samples(data, fmt, shift)
    nbytes = len(data) if isinstance(data, (bytes, bytearray)) else np.asarray(data).size
    n = n_buffers(nbytes, rate, fmt, drop_eof)
    return np.array([record(x, rate, b) for b in range(first, n)], dtype=DTYPE)
