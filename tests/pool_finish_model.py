"""The receiver pool's finish schedule (modes_pool_finish, csrc/modes_pool.cpp): which 2 MHz buffers a
finish decodes for a receiver, and in which of its two internal batches.

A receiver that has had `submitted` 2 MHz buffers decoded (at 2.4 MS/s: after in_total UC8 input bytes, the
calls of pool_rate_model.receiver_calls) is finished with a tail of tail_bytes bytes.  The whole stream then
has n_in = in_total / 2 + the tail's samples input samples (a UC8 tail: ceil(bytes / 2), a trailing odd byte
an I whose Q is 127; a 16-bit tail: floor(bytes / 4)) and N_out 2 MHz samples: n_in at 2 MHz, ceil(5 n_in / 6)
at 2.4 MS/s, as modes_finish's finish_held rule gives them.  Buffers [submitted, N_out / B) are whole and are
decoded in batch 1; buffer N_out / B is the EOF buffer (127 past N_out), decoded in batch 2 unless
drop_eof_buffer is set.  A 2 MHz receiver follows modes_finish itself: only a tail of a whole buffer is a
whole buffer, and the EOF buffer holds the rest (a UC8 tail one byte short of a buffer fills it).  Batch 1
holds at most one buffer: at 2 MHz the tail itself when it is a whole buffer, at 2.4 MS/s the buffer whose
filter lookahead had not arrived.  Each batch holds one pair per receiver, as the pool's resolve needs."""
from __future__ import annotations

import pool_rate_model as PM
import resample_model as RM

BUFFER_SAMPLES = PM.BUFFER_SAMPLES
BUFFER_BYTES = 2 * BUFFER_SAMPLES


def buffer_bytes(fmt: str) -> int:
    """A receiver's buffer: MODES_BUFFER_BYTES for UC8, twice that for SC16 / SC16Q11."""
    return BUFFER_BYTES * (1 if fmt == "uc8" else 2)


def tail_samples(tail_bytes: int, fmt: str) -> int:
    return (tail_bytes + 1) // 2 if fmt == "uc8" else tail_bytes // 4


def state_after(rate: int, n_calls: int) -> tuple[int, int]:
    """(submitted, in_total) of a receiver after n_calls whole buffers: 2 MHz buffers decoded, UC8 input bytes."""
    if rate == 2_000_000:
        return n_calls, n_calls * BUFFER_BYTES
    return PM.ready_buffers(n_calls * BUFFER_SAMPLES), n_calls * BUFFER_BYTES


def n_out(rate: int, in_total: int, tail_bytes: int, fmt: str) -> int:
    """2 MHz samples of the whole stream."""
    n_in = in_total // 2 + tail_samples(tail_bytes, fmt)
    return n_in if rate == 2_000_000 else RM.n_out(n_in)


def finish_pairs(rate: int, fmt: str, submitted: int, in_total: int, tail_bytes: int, drop_eof: bool = False):
    """The pairs a finish makes for the receiver: [(batch, 2 MHz buffer, real samples of the buffer)]."""
    if rate == 2_000_000:
        # as modes_finish: a whole tail is an ordinary buffer, the rest is the EOF buffer (a UC8 tail one byte
        # short of a buffer still makes B samples, all in the EOF buffer)
        whole = tail_bytes == buffer_bytes(fmt)
        eof = submitted + whole
        end = eof * BUFFER_SAMPLES + tail_samples(0 if whole else tail_bytes, fmt)
    else:
        end = n_out(rate, in_total, tail_bytes, fmt)
        eof = end // BUFFER_SAMPLES
    pairs = [(1, b, BUFFER_SAMPLES) for b in range(submitted, eof)]
    if not drop_eof:
        pairs.append((2, eof, end - eof * BUFFER_SAMPLES))
    return pairs


def two_pair_tails(rate: int, fmt: str, n_calls: int) -> int | None:
    """The shortest tail after n_calls whole buffers with which a finish makes a whole buffer as well as the
    EOF buffer (None: none does); every longer tail does too."""
    submitted, in_total = state_after(rate, n_calls)
    whole = lambda t: len(finish_pairs(rate, fmt, submitted, in_total, t)) == 2
    lo, hi = 0, buffer_bytes(fmt)
    if not whole(hi):
        return None
    while lo < hi:                                      # n_out grows with the tail: the first t that is whole
        mid = (lo + hi) // 2
        lo, hi = (lo, mid) if whole(mid) else (mid + 1, hi)
    return lo
