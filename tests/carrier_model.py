"""Plain restatement of the carrier measurement (include/modes_b200.h, modes_set_carrier) in numpy.

A decoded attempt at stream sample j with b bits: the pulse sample of bit i is j+16+2i for a 1 and j+17+2i
for a 0, the preamble's pulses are at j+0, 2, 7, 9.  The pairs are the pulse samples two apart: (0, 2),
(7, 9) and the pulses of each two consecutive equal bits.  With z = (I - 127) + i (Q - 127), the record is
sum z_later conj(z_earlier); the code is 16384 + round(atan2(im, re) / (2 pi 1 us) / 100 Hz), halves away
from zero, and 0 for re = im = 0."""
from __future__ import annotations

import math

import numpy as np

CODE_ZERO = 16384
STEP_HZ = 100


def frame_bits(msg, bits: int) -> np.ndarray:
    return np.unpackbits(np.frombuffer(bytes(msg)[:14], dtype=np.uint8))[:bits].astype(np.int64)


def pairs(fbits) -> list[tuple[int, int]]:
    """The (earlier, later) window samples of every pair, relative to j."""
    b = len(fbits)
    out = [(0, 2), (7, 9)]
    for i in range(b - 1):
        if fbits[i] == fbits[i + 1]:
            p = 16 + 2 * i + (1 - int(fbits[i]))
            out.append((p, p + 2))
    return out


def record(iq, j: int, msg, bits: int) -> tuple[int, int]:
    """(re, im) of the attempt at stream sample j of the UC8 bytes iq (samples outside them read 127)."""
    iq = np.asarray(iq, dtype=np.uint8)
    n = iq.size // 2

    def z(s: int) -> tuple[int, int]:
        if 0 <= s < n:
            return int(iq[2 * s]) - 127, int(iq[2 * s + 1]) - 127
        return 0, 0

    re = im = 0
    for a, b in pairs(frame_bits(msg, bits)):
        ia, qa = z(j + a)
        ib, qb = z(j + b)
        re += ia * ib + qa * qb
        im += ia * qb - qa * ib
    return re, im


def code_of(re: int, im: int) -> int:
    if re == 0 and im == 0:
        return 0
    c = math.atan2(im, re) * (1e4 / (2.0 * math.pi))          # f / 100 Hz, with f = phase / (2 pi 1 us)
    return CODE_ZERO + int(math.copysign(math.floor(abs(c) + 0.5), c))


def hz_of(code: int):
    return None if code == 0 else (code - CODE_ZERO) * STEP_HZ


def expected_code(iq, msg) -> int:
    """The code of a delivered message (api.Message) from the 2 MHz bytes it was decoded from."""
    return code_of(*record(iq, int(msg.sample_pos), msg.msg, int(msg.msgbits)))
