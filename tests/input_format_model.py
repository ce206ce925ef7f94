"""The 16-bit input formats (modes_set_input_format) restated in numpy: SC16 / SC16Q11 I/Q to UC8 bytes.

    q    = s ? (v + (1 << (s - 1))) >> s : v        (int32, arithmetic shift: round half up)
    byte = clamp(127 + q, 0, 255)

for each signed little-endian int16 value v (I and Q separately) and the shift s in 0..15.  A stream of
`bytes` bytes has n_in = floor(bytes / 4) samples; 1-3 trailing bytes are ignored.  The converted stream
is then decoded as UC8 at the input rate (at 2.4 MS/s: tests/resample_model.py on the converted bytes).
"""
import numpy as np

FORMATS = {"uc8": 0, "sc16": 1, "sc16q11": 2}
DEFAULT_SHIFT = {"sc16": 8, "sc16q11": 4}


def convert_values(v, shift: int) -> np.ndarray:
    """int16 values (any shape) to their UC8 bytes."""
    v = np.asarray(v, dtype=np.int64)
    q = (v + ((1 << shift) >> 1)) >> shift
    return np.clip(127 + q, 0, 255).astype(np.uint8)


def convert(data, shift: int) -> np.ndarray:
    """A whole 16-bit stream (bytes) to its UC8 bytes: 2 n_in bytes."""
    a = np.frombuffer(data, dtype=np.uint8) if isinstance(data, (bytes, bytearray)) else np.asarray(data, np.uint8)
    n = a.size // 4 * 4
    return convert_values(np.ascontiguousarray(a[:n]).view("<i2"), shift)


def to_sc16(uc8, shift: int) -> np.ndarray:
    """UC8 bytes written as int16 bytes that convert back to them at `shift`: v = 2^s (b - 127) - 2^(s-1)
    (the lowest value that rounds to b; v = b - 127 at s = 0)."""
    b = np.asarray(uc8, dtype=np.int64)
    v = (b - 127) << shift
    if shift:
        v -= 1 << (shift - 1)
    assert v.min(initial=0) >= -32768 and v.max(initial=0) <= 32767
    return v.astype("<i2").view(np.uint8)


class Streaming:
    """The conversion fed piecewise, as a streaming decode sees it: a sample split across pieces is held
    until its last byte arrives."""

    def __init__(self, shift: int):
        self.shift = shift
        self.part = np.zeros(0, np.uint8)

    def feed(self, piece) -> np.ndarray:
        a = np.concatenate([self.part, np.asarray(piece, np.uint8)])
        n = a.size // 4 * 4
        self.part = a[n:]
        return convert(a[:n], self.shift)

    def finish(self) -> np.ndarray:
        self.part = np.zeros(0, np.uint8)              # 1-3 trailing bytes are ignored
        return np.zeros(0, np.uint8)
