"""The receiver pool's schedule for a 2.4 MS/s receiver (modes_pool_set_input_rate, csrc/modes_pool.cpp):
which call completes which 2 MHz buffer, and which input bytes the receiver's device history keeps.

Every call brings MODES_BUFFER_BYTES (131072 input samples) of the receiver's stream.  2 MHz buffer m
completes once its last output sample, with the filter's lookahead, reads no input that has not arrived
(the rule of modes_process at 2.4 MS/s and of resample_model.Streaming's emission).  After a call, the
history keeps the stream bytes from the first one a later buffer (its 238 carry samples included) reads,
rounded down to 16 bytes and never moving back."""
from __future__ import annotations

import resample_model as RM

BUFFER_SAMPLES = 131072
CARRY_SAMPLES = 238


def ready_buffers(n_input_samples: int, buffer_samples: int = BUFFER_SAMPLES, taps: int = RM.TAPS) -> int:
    """2 MHz buffers complete once n_input_samples input samples have arrived."""
    m = max((5 * n_input_samples // 6) // buffer_samples - 1, 0)
    while RM.input_span(0, (m + 1) * buffer_samples, taps)[1] <= n_input_samples:
        m += 1
    return m


def history_keep(next_buffer: int, hist0: int, buffer_samples: int = BUFFER_SAMPLES) -> int:
    """The first stream byte the history keeps when the receiver's next 2 MHz buffer is next_buffer and
    its history started at byte hist0."""
    keep = max(2 * RM.input_span(next_buffer * buffer_samples - CARRY_SAMPLES, 1)[0], 0) // 16 * 16
    return max(keep, hist0)


def receiver_calls(n_calls: int, buffer_samples: int = BUFFER_SAMPLES):
    """A 2.4 MS/s receiver's state before each call c: (hist0, call0, buffer m, completes, keep after it),
    byte positions in its stream."""
    out, hist0, m = [], 0, 0
    for c in range(n_calls):
        call0 = 2 * c * buffer_samples
        done = ready_buffers((c + 1) * buffer_samples, buffer_samples) > m
        keep = history_keep(m + done, hist0, buffer_samples)
        out.append((hist0, call0, m, done, keep))
        m += done
        hist0 = keep
    return out
