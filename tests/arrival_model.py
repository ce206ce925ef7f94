"""Restatement of the arrival-time definition (include/modes_b200.h, modes_set_arrival) in numpy and
exact rationals, independent of the product's word arithmetic: the pulse pattern is built sample by
sample, the classes are read from it, and the offset is rounded from a Fraction."""
from fractions import Fraction

import numpy as np

MAIN, LATE, EARLY, QUIET, UNUSED = 0, 1, 2, 3, 4


def frame_bits(msg, bits: int) -> np.ndarray:
    return np.unpackbits(np.frombuffer(bytes(msg)[: bits // 8], dtype=np.uint8))[:bits]


def pattern(fbits) -> np.ndarray:
    """e over the window samples 0 .. 17+2b."""
    b = len(fbits)
    e = np.zeros(18 + 2 * b, dtype=np.int64)
    e[[0, 2, 7, 9]] = 1
    for i, bit in enumerate(fbits):
        e[16 + 2 * i + (0 if bit else 1)] = 1
    return e


def classes(fbits) -> np.ndarray:
    """Class of window samples 1 .. 16+2b (index s - 1)."""
    e = pattern(fbits)
    s = np.arange(1, 17 + 2 * len(fbits))
    key = e[s - 1] * 4 + e[s] * 2 + e[s + 1]
    table = np.full(8, UNUSED)
    table[0b010], table[0b100], table[0b001], table[0b000] = MAIN, LATE, EARLY, QUIET
    return table[key]


def round_half_away(x: Fraction) -> int:
    q = int((abs(x) + Fraction(1, 2)).__floor__())
    return q if x >= 0 else -q


def code_from_sums(S, n) -> int:
    """The code from class sums / counts (indexed MAIN, LATE, EARLY, QUIET)."""
    mu = Fraction(int(S[QUIET]), int(n[QUIET]))
    A = Fraction(int(S[MAIN]), int(n[MAIN])) - mu
    L = max(Fraction(int(S[LATE]), int(n[LATE])) - mu, Fraction(0))
    E = max(Fraction(int(S[EARLY]), int(n[EARLY])) - mu, Fraction(0))
    den = A + L + E
    if den <= 0:
        return 0
    off = max(-7, min(7, round_half_away(6 * (L - E) / den)))
    return off + 8


def code_of_window(m, msg, bits: int) -> int:
    """m: magnitudes of window samples 0 .. 16+2b (at least 17+2b values)."""
    cls = classes(frame_bits(msg, bits))
    w = np.asarray(m, dtype=np.int64)[1: 17 + 2 * bits]
    S = [int(w[cls == c].sum()) for c in range(4)]
    n = [int((cls == c).sum()) for c in range(4)]
    assert min(n) > 0
    return code_from_sums(S, n)


def expected_arrival(mag, pos, msgs, bits) -> np.ndarray:
    """Codes of frames (msg bytes, b bits) whose preamble starts at stream sample pos; samples outside
    the stream have magnitude 0."""
    out = np.zeros(len(pos), dtype=np.int64)
    for k, (p, msg, b) in enumerate(zip(pos, msgs, bits)):
        ix = int(p) + np.arange(17 + 2 * int(b))
        ok = (ix >= 0) & (ix < mag.size)
        w = np.where(ok, mag[np.clip(ix, 0, mag.size - 1)], 0)
        out[k] = code_of_window(w, msg, int(b))
    return out


def arrival_ticks(pos, code):
    """The refined 12 MHz arrival of a frame at stream sample pos (6 * pos when not measured)."""
    return 6 * int(pos) + (int(code) - 8 if code else 0)
