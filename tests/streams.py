"""Seeded input streams shared by the CPU (host shim) and GPU parity tests: the demodulator's
nastiest inputs.  TEST INFRASTRUCTURE."""
from __future__ import annotations

import numpy as np

from dump1090_b200 import synth


def tie_rich(seed, n_frames=1500, levels=(0, 0, 1, 40, 100), period=300):
    """Preambles followed by half-bit samples drawn from a few amplitudes: equal pairs (the
    reference's bits[0] == 2 and copied bits, dump1090.c:1675-1689), weak pairs, gate failures,
    all message types.  A preamble every `period` samples; below 240 the bodies are cut short and
    the next preamble lands inside the previous frame."""
    rng = np.random.default_rng(seed)
    n_body = min(224, period - 16)
    iq = np.full((n_frames * period + 1000, 2), 127, dtype=np.uint8)
    for f in range(n_frames):
        s = 50 + f * period + int(rng.integers(0, 3))
        for k in (0, 2, 7, 9):
            iq[s + k, 0] = 127 + 110
        body = rng.choice(np.array(levels), size=n_body)
        if f % 4 == 0:
            body[1] = body[0]                                            # first pair ties
        iq[s + 16: s + 16 + n_body, 0] = 127 + body
        iq[s + 16: s + 16 + n_body, 1] = 127 - rng.choice(np.array(levels), size=n_body) // 2
    return iq.ravel()


def random_alphabet_cases(n_cases=24, seed=2024):
    """Small streams with random amplitude alphabets, preamble jitter, noise and saturation: weak
    and saturated pairs, long indefinite runs, every gate outcome."""
    rng = np.random.default_rng(seed)
    for case in range(n_cases):
        levels = tuple(int(x) for x in rng.choice([0, 0, 1, 2, 3, 5, 8, 20, 40, 70, 100, 127, 128], size=int(rng.integers(2, 6))))
        data = tie_rich(int(rng.integers(1, 1 << 30)), n_frames=int(rng.integers(60, 200)), levels=levels).copy()
        if case % 3 == 0:                                                 # additive noise on top
            noise = rng.integers(-3, 4, size=data.size)
            data = np.clip(data.astype(np.int64) + noise, 0, 255).astype(np.uint8)
        if case % 4 == 1:                                                 # saturated samples
            data[rng.integers(0, data.size, size=data.size // 50)] = 255
        yield case, levels, data


def retry_at_buffer_start(n_buffers=6, seed=3):
    """Frames whose preamble sits exactly at j == 0 of a reference buffer (stream sample
    131072k - 238) and whose first attempt is not a good message: the reference retries them
    WITHOUT phase correction (dump1090.c:1660).  Mix per buffer: unrepairable DF17 (3 flipped
    bits), DF17 with a flipped DF field, an address/parity frame of an unknown aircraft, a clean
    DF17 (control: no retry), each also one sample later (j == 1: corrected retry)."""
    rng = synth.Counter(seed)
    frames = []
    for k in range(1, n_buffers):
        j0 = 131072 * k - 238
        icao = 0x400000 + rng.below(0x3FFFFF)
        good = synth.make_frame(17, 5, icao.to_bytes(3, "big") + bytes(rng.below(256) for _ in range(7)))
        kind = k % 4
        if kind == 0:
            frame = synth.flip_bits(good, [20, 47, 81])
        elif kind == 1:
            frame = synth.flip_bits(good, [2, 60])
        elif kind == 2:
            frame = synth.make_frame(20, 3, bytes(rng.below(256) for _ in range(10)), icao_for_ap=0x123456 + k)
        else:
            frame = good
        frames.append((j0, frame, 70.0 + 5 * k, 0.4 * k, 0.3 if k % 2 else 0.0))
        frames.append((j0 + 65536 + 1, frame, 70.0, 0.2 * k, 0.4))          # far from any seam: normal corrected retry
    return synth.synth_stream(131072 * n_buffers + 3000, frames, sigma=1.2, seed=seed)


def icao_slot(a):
    """The slot of address `a` in the 1024-entry ICAO cache (dump1090.c:898-905)."""
    a = (((a >> 16) ^ a) * 0x45D9F3B) & 0xFFFFFFFF
    a = (((a >> 16) ^ a) * 0x45D9F3B) & 0xFFFFFFFF
    return ((a >> 16) ^ a) & 1023


CHAIN_KINDS = ("df4", "df20", "df11_iid", "evict", "seam")
_ME = bytes([0x58, 0xC3, 0x82, 0xD6, 0x90, 0xC8, 0xAC])                    # an airborne-position ME field
# interrogator ids below 80 with three or more bits set: not the syndrome of one or two flipped
# parity bits, so neither the one-bit nor the aggressive two-bit repair turns them into a clean frame
_IIDS = [v for v in range(1, 80) if bin(v).count("1") >= 3]


def address_chain(n_buffers, kind="df4", seed=1, return_expected=False):
    """A dependency that runs through the ICAO address cache from buffer to buffer, so that no
    buffer's outcome can be known before the previous buffer's is.

    Every reference buffer b >= 1 holds a READER of address X_b followed by a WRITER announcing
    X_{b+1} whose preamble starts exactly where the reference's skip past a good reader ends, one
    sample short of it (j + 2 * (8 + bits) + 1, dump1090.c:1769-1791).  The writer is taken, and
    X_{b+1} enters the cache, only when the reader is NOT validated by the cache, i.e. when
    buffer b - 1 did not write X_b.  Buffer 0 holds only the writer of X_1.  So the reference
    delivers exactly one message per buffer, alternating:
        buffer 0: writer(X_1); buffer 1: reader(X_1); buffer 2: writer(X_3); buffer 3: reader(X_3); ...
    i.e. buffer b delivers its writer when b is even and its reader when b is odd; every reader of
    an even buffer and every writer of an odd buffer is dropped.  Kinds:
      df4       DF4 reader (address/parity field = X_b, 56 bits), DF11 writer 128 samples later
      df20      DF20 reader (112 bits, skip 241), DF17 / DF18 writer (alternately) 240 samples later
      df11_iid  DF11 reader whose parity carries an interrogator id below 80 (validated by the
                cache through its address field, dump1090.c:1204-1209), DF11 writer 128 later
      evict     as df4, but all X_b share one cache slot: a writer overwrites the address the
                previous writer left there instead of filling an empty slot
      seam      as df4, with the writer's preamble at the last positions the reference tests
                (j = 131067..131069): its frame runs into the samples carried to the next buffer
    With return_expected, also returns the expected messages as (sample_pos, df, address)."""
    assert kind in CHAIN_KINDS and n_buffers >= 1
    rng = synth.Counter(seed * 7919 + CHAIN_KINDS.index(kind))
    addrs, slots = [None], set()                                      # addrs[b] = X_b, b >= 1
    want_slot = icao_slot(0x400000 + rng.below(0x3FFFFF))
    while len(addrs) <= n_buffers:
        a = 0x100000 + rng.below(0xEFFFFF)
        s = icao_slot(a)
        if (kind == "evict" and s != want_slot) or (kind != "evict" and s in slots) or a in addrs:
            continue
        addrs.append(a)
        slots.add(s)
    gap = 240 if kind == "df20" else 128

    def reader(b):
        x = addrs[b]
        if kind == "df20":
            return synth.make_frame(20, 0, bytes([0x10, 0x00, 0x1C, 0x38]) + _ME[:6], icao_for_ap=x), 20
        if kind == "df11_iid":
            f = synth.make_frame(11, 5, x.to_bytes(3, "big"))
            iid = _IIDS[b % len(_IIDS)]
            return f[:4] + (int.from_bytes(f[4:], "big") ^ iid).to_bytes(3, "big"), 11
        return synth.make_frame(4, 0, bytes([0x01, 0x85, 0x10 + (b & 7)]), icao_for_ap=x), 4

    def writer(b):
        x = addrs[b + 1] if b + 1 < len(addrs) else addrs[b] ^ 0x5A5A5A
        if kind == "df20":
            df = 17 if (b // 2) % 2 == 0 else 18
            return synth.make_frame(df, 5 if df == 17 else 0, x.to_bytes(3, "big") + _ME), df, x
        return synth.make_frame(11, 5, x.to_bytes(3, "big")), 11, x

    frames, expected = [], []
    for b in range(n_buffers):
        if kind == "seam":
            j_w = 131069 - b % 3
        else:
            j_w = 20238 + 37 * (b % 5) + gap
        w_pos = 131072 * b - 238 + j_w
        wf, wdf, wx = writer(b)
        frames.append((w_pos, wf, 80.0, 0.4 + 0.3 * b, 0.0))
        if b:
            rf, rdf = reader(b)
            frames.append((w_pos - gap, rf, 80.0, 1.1 + 0.2 * b, 0.0))
        if b % 2 == 0:
            expected.append((w_pos, wdf, wx))
        else:
            expected.append((w_pos - gap, rdf, addrs[b]))
    data = synth.synth_stream(131072 * n_buffers, frames, sigma=1.0, seed=seed)
    return (data, expected) if return_expected else data


# name: (kind, buffers) of the chains the parity tests take as inputs, all longer than the device
# resolve's fixed rounds (a chain of n buffers needs about n rounds of guessing)
CHAINS = {"chain_df4": ("df4", 12), "chain_df20": ("df20", 8), "chain_df11_iid": ("df11_iid", 9),
          "chain_evict": ("evict", 10), "chain_seam": ("seam", 8)}


def chain(name):
    kind, n = CHAINS[name]
    return address_chain(n, kind)


def chain_streams():
    """(name, stream) of every chain in CHAINS."""
    for name in CHAINS:
        yield name, chain(name)
