"""Constructed corpora of the recovery, signal and level arithmetic: the windows and buffers at the
edges where those passes go wrong (weight-6 ambiguities, all-equal windows, saturated windows, small
amplitude alphabets, repaired frames).  TEST INFRASTRUCTURE, shared by the host-shim tests
(test_recover.py, test_signal.py, test_levels.py) and the device tests (test_kernel_edges.py), so
both run the same lists.  Every builder is deterministic."""
from __future__ import annotations

import numpy as np

import recover_model as R
import repair_corpus
from dump1090_b200 import api, synth

BUF = api.BUFFER_BYTES

# ---------------------------------------------------------------- recovery: windows of 448 I/Q bytes


def window(frame: bytes, weak=(), flips=(), strong=(60, 0), soft=(40, 39), rng=None):
    """448 I/Q bytes of a frame's 112 bit pairs: the pulse of bit i in its first (1) or second (0)
    sample; `weak` bits get nearly equal samples, and `flips` are sent the wrong way round."""
    out = np.full((112, 4), 127, dtype=np.int64)
    for i in range(112):
        bit = (frame[i >> 3] >> (7 - (i & 7))) & 1
        hi, lo = soft if i in weak else strong
        if rng is not None and i not in weak:
            hi += int(rng.integers(0, 20))
        if i in flips:
            bit ^= 1
        out[i, 0] += hi if bit else lo
        out[i, 2] += lo if bit else hi
    return out.astype(np.uint8).reshape(-1)


def frames(n, seed, df=17):
    rng = synth.Counter(seed)
    return [synth.make_frame(df, 5, (0x400000 + rng.below(0x3FFFFF)).to_bytes(3, "big") + synth._me_airborne(rng))
            for _ in range(n)]


def restated(wins):
    """recover_model.restate of windows of 448 I/Q bytes."""
    wins = np.asarray(wins, dtype=np.uint8).reshape(-1, 448)
    m = R.magnitudes(wins.reshape(-1)).reshape(-1, 224)
    return R.restate(m[:, 0::2], m[:, 1::2])


def recover_random_windows() -> dict:
    """name -> windows: random, saturated and alphabet windows, all-equal windows behind a DF17 / DF18
    prefix (every w = 0: the tie-break on i decides the positions), and noise behind a DF17 prefix."""
    rng = np.random.default_rng(3)
    cases = {
        "random": rng.integers(0, 256, size=(500, 448), dtype=np.uint8),
        "saturated": rng.choice(np.array([0, 255], dtype=np.uint8), size=(300, 448)),
        "alphabet": rng.choice(np.array([0, 1, 126, 127, 128, 200, 254, 255], dtype=np.uint8), size=(300, 448)),
    }
    for df in (17, 18):
        w = np.full((40, 448), 127, dtype=np.uint8)
        for k in range(40):
            w[k] = np.full(448, 127 + k, dtype=np.uint8)
            w[k, :20] = window(bytes([df << 3]) + bytes(13))[:20]
        cases[f"all_equal_df{df}"] = w
    # random windows whose hard DF is 17: the search runs on noise
    noise = rng.integers(100, 155, size=(400, 448), dtype=np.uint8)
    noise[:, :20] = window(bytes([17 << 3]) + bytes(13))[:20]
    cases["noise_df17"] = noise
    return cases


def recover_frame_windows():
    """(windows, sent frames, flips made): clean DF17 / DF18 frames, and each repaired with 1..10 of
    its ten weak bits flipped."""
    rng = np.random.default_rng(4)
    wins, sent, expect = [], [], []
    for k, f in enumerate(frames(60, 11) + frames(20, 12, df=18)):
        wins.append(window(f, rng=rng))                                 # clean: FOUND with no flip
        sent.append(f)
        expect.append(0)
        weak = set(int(x) for x in rng.choice(np.arange(5, 112), size=10, replace=False))
        for e in (1 + k % 10, 1 + (k + 3) % 10):
            flips = set(sorted(weak)[:e])
            wins.append(window(f, weak=weak, flips=flips, rng=rng))
            sent.append(f)
            expect.append(e)
    return np.array(wins), sent, expect


def recover_confident_windows():
    """40 DF17 frames with one confident bit wrong (mostly not FOUND), then nine other formats
    (INELIGIBLE)."""
    rng = np.random.default_rng(5)
    wins = []
    for f in frames(40, 13):
        weak = set(range(20, 30))
        wins.append(window(f, weak=weak, flips={int(rng.integers(40, 112))}, rng=rng))
    for df in (0, 4, 5, 11, 16, 19, 20, 21, 24):
        wins.append(window(bytes([df << 3]) + bytes(rng.integers(0, 256, 13, dtype=np.uint8)), rng=rng))
    return np.array(wins)


def recover_ambiguity_windows():
    """Three bits of each of the 155 weight-6 codewords within 5..111 flipped, its six positions among
    the ten least confident: two solutions of weight 3 (AMBIGUOUS)."""
    cws = [c for c in repair_corpus.long_codewords6() if min(c) >= 5]
    assert len(cws) == 155
    rng = np.random.default_rng(6)
    wins = []
    for cw, f in zip(cws, frames(len(cws), 14)):
        others = [p for p in range(5, 112) if p not in cw]
        weak = set(cw) | set(int(x) for x in rng.choice(others, size=4, replace=False))
        wins.append(window(f, weak=weak, flips=set(cw[:3]), rng=rng))
    return np.array(wins)


# ---------------------------------------------------------------- signal: windows of 224 samples


def signal_windows(rng):
    """(name, windows of 224 samples as I/Q bytes)."""
    yield "random", rng.integers(0, 256, size=(400, 448), dtype=np.uint8)
    yield "saturated", rng.choice(np.array([0, 255], dtype=np.uint8), size=(200, 448))
    yield "saturated_max", np.full((1, 448), 255, dtype=np.uint8)
    yield "no_signal", np.full((2, 448), 127, dtype=np.uint8)
    yield "levels", rng.choice(np.array([0, 1, 126, 127, 128, 200, 254, 255], dtype=np.uint8), size=(200, 448))
    yield "weak", np.clip(rng.normal(127, 4, size=(200, 448)).round(), 0, 255).astype(np.uint8)


# ---------------------------------------------------------------- levels: whole buffers


def level_buffers(rng):
    """(name, one buffer of I/Q bytes)."""
    yield "random", rng.integers(0, 256, size=BUF, dtype=np.uint8)
    yield "all_0", np.zeros(BUF, dtype=np.uint8)
    yield "all_255", np.full(BUF, 255, dtype=np.uint8)                   # every sample at m = 65167: largest sums
    yield "all_127", np.full(BUF, 127, dtype=np.uint8)
    yield "alphabet", rng.choice(np.array([0, 1, 126, 127, 128, 254, 255], dtype=np.uint8), size=BUF)
    yield "weak_noise", np.clip(rng.normal(127, 3, size=BUF).round(), 0, 255).astype(np.uint8)
    yield "rails_254", rng.choice(np.array([254, 1, 127], dtype=np.uint8), size=BUF)   # near the rails, never on them
    one = np.full(BUF, 127, dtype=np.uint8)
    one[[0, 1001, BUF - 1]] = [0, 255, 0]                                 # I, Q, Q on a rail
    yield "three_clipped", one
