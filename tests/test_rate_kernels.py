"""The decimator (K11), its frequency shift (K12) and the input spectrum pass (K13) as whole launches on the GPU,
byte for byte against their numpy restatements (tests/decimate_model.py, tests/shift_model.py,
tests/spectrum_model.py, 16-bit input through tests/input_format_model.py), through the device harness
tests/device_shim/rate_spectrum_device.cu over the product's own kernel objects.

The decoder's batches reach only a narrow slice of what these launches accept: UC8 only through the stage
entries, and spans that start where stage_held starts them, which leaves the window alignment sh of K11/K12 at
{0, 12} (M = 2, 4, 5) or {0, 14} (M = 3) and K13's frame offsets at {0, 2E} bytes.  Here every launch is one
the harness builds: 16-bit input at several shifts, every span alignment, spans cut at both ends, positions past
2^32 and 2^33 input samples, EOF limits anywhere, the bytes a launch must leave alone, grids of hundreds of
buffers and the pool form's 256 jobs.  The CPU half pins why those cases are new and that the case generators
reach them.
"""
from __future__ import annotations

import ctypes
import subprocess

import numpy as np
import pytest

import checker as C
import decimate_model as DM
import input_format_model as IF
import shift_model as SM
import spectrum_model as SPM
import test_spectrum as TS
from dump1090_b200 import api

ROOT = C.ROOT
DSHIM = ROOT / "tests" / "_build" / "librate_spectrum_device.so"
B = api.BUFFER_SAMPLES
BUF = api.BUFFER_BYTES
N = SPM.N
NO_LIMIT = 2 ** 63 - 1
HALO_BYTES = 480                       # kHaloBytes: the carry block's 240 samples
HALO_ALLOC = 512                       # kHaloAlloc: its allocation, no signal after them
GUARD = 256                            # the harness's sentinel bytes after the body and after the carry block
SENTINEL = 0x5A
EXTENT = {m: DM.extent(DM.taps(m), m) for m in (2, 3, 4, 5)}
# K11/K12's input kinds: UC8 (shift -1), SC16 at its shift 8, SC16Q11 at 4, and int16 at shifts 0 and 15
SHIFTS = (-1, 8, 4, 0, 15)


def offsets(m: int) -> tuple[int, ...]:
    """0, +-the largest offset the decoder takes at 2 M MS/s, and an odd offset (a step with every phase)."""
    mx = SM.max_offset(2_000_000 * m)
    return 0, mx, -mx, mx - 123_457


# ---------------------------------------------------------------- the layout a launch writes


def carry_layout() -> dict[str, tuple[int, int]]:
    """Byte ranges of the kHaloAlloc carry block: the 238 carry samples at [kHaloBytes - MODES_CARRY_BYTES,
    kHaloBytes), no signal before and after them."""
    c = HALO_BYTES - api.CARRY_BYTES
    return {"no_signal_lo": (0, c), "carry": (c, HALO_BYTES), "no_signal_hi": (HALO_BYTES, HALO_ALLOC)}


def test_carry_layout():
    lay = carry_layout()
    assert lay == {"no_signal_lo": (0, 4), "carry": (4, 480), "no_signal_hi": (480, 512)}
    # the carry block's 240 samples are 30 whole groups of 8, so with it a launch starts at out_first - 240
    assert (lay["carry"][1] // 2) % 8 == 0


# ---------------------------------------------------------------- where the decoder's batches start their spans


def stage_held_in_first(m: int, o0: int) -> int:
    """The input sample stage_held starts a batch's span at for the batch whose body starts at output sample o0
    (in_lo(rate, o0 - carry) of modes_resample_core.cuh, floored at the stream's start)."""
    return max(m * (o0 - 240) - EXTENT[m], 0)


def window_sh(m: int, n0: int, in_first: int) -> int:
    """K11/K12's window alignment for the group at output sample n0: 2 (M n0 - E - in_first) mod 16."""
    return (2 * (m * n0 - EXTENT[m] - in_first)) % 16


def frame_sh(first: int, in_first: int) -> int:
    """K13's frame alignment (SpanReader) of a buffer whose frames start at stream sample first."""
    return (2 * (first - in_first)) % 16


@pytest.mark.parametrize("m", [2, 3, 4, 5])
def test_decoder_spans_reach_few_alignments(m):
    """The spans stage_held builds give K11/K12 only sh = 0 (later batches) and -2E mod 16 (a stream's first),
    and K13 only frame offsets 0 and 2E: the other alignments run only in this file."""
    e = EXTENT[m]
    got, frames = set(), set()
    for o0 in [0, B, 2 * B, 7 * B] + [((2 ** 32 + k) // (m * B)) * B for k in (0, 3 * B, 2 ** 32)]:
        lo = stage_held_in_first(m, o0)
        first_group = o0 - 240 if o0 else -240     # a stream's first batch has the carry block before sample 0
        got |= {window_sh(m, first_group + 8 * g, lo) for g in range(64)}
        frames |= {frame_sh(SPM.first_sample(2_000_000 * m, o0 // B + k), lo) for k in range(3)}
    assert got == {0, (-2 * e) % 16}
    assert got == ({0, 12} if m != 3 else {0, 14})
    assert frames == {0, 2 * e}


# ---------------------------------------------------------------- case generators


def uc8_corpus(rng, n_samples: int) -> np.ndarray:
    """UC8 bytes: noise, with runs of the 0/255 extremes and their I/Q mixes (which reach |u| = 182 at 45-degree
    phases of the shift)."""
    a = rng.integers(0, 256, 2 * n_samples, dtype=np.uint8)
    pats = [(0, 0), (255, 255), (255, 0), (0, 255), (127, 127)]
    for k in range(0, n_samples, 97):
        i, q = pats[(k // 97) % len(pats)]
        run = min(40, n_samples - k)
        a[2 * k: 2 * (k + run): 2] = i
        a[2 * k + 1: 2 * (k + run): 2] = q
    return a


def int16_specials() -> np.ndarray:
    """int16 values at the conversion's edges: the extremes, the half-way values k 2^s +- 2^(s-1) at every
    shift, and the values on each side of every clamp."""
    v = {-32768, -32767, -1, 0, 1, 32766, 32767}
    for s in range(1, 16):
        for k in (-3, -1, 0, 1, 2):
            for d in (-1, 0, 1):
                v.add((k << s) + (1 << (s - 1)) + d)
                v.add((k << s) - (1 << (s - 1)) + d)
    for s in range(16):
        lo, hi = clamp_edges(s)
        v |= {x for x in lo + hi}
    return np.array(sorted(x for x in v if -32768 <= x <= 32767), np.int64)


def clamp_edges(s: int) -> tuple[list[int], list[int]]:
    """The int16 values on each side of the conversion's low and high clamps at shift s (none where it cannot clamp)."""
    v = np.arange(-32768, 32768, dtype=np.int64)
    q = 127 + ((v + ((1 << s) >> 1)) >> s)
    lo, hi = [], []
    if (q < 0).any():
        x = int(v[q < 0].max())
        lo = [x, x + 1]
    if (q > 255).any():
        x = int(v[q > 255].min())
        hi = [x - 1, x]
    return lo, hi


def int16_corpus(rng, n_samples: int) -> np.ndarray:
    """int16 I/Q bytes: full-range noise, the special values scattered through it, and constant runs of the extremes."""
    v = rng.integers(-32768, 32768, 2 * n_samples, dtype=np.int64)
    sp = int16_specials()
    k = np.arange(0, v.size, 3)
    v[k] = sp[np.arange(k.size) % sp.size]
    for j, c in enumerate((-32768, 32767, 0, -32768)):
        a = (j * 2 * 613) % max(v.size - 60, 1)
        v[a: a + 60] = c
    return v.astype("<i2").view(np.uint8)


def corpus(rng, shift: int, n_samples: int) -> np.ndarray:
    return uc8_corpus(rng, n_samples) if shift < 0 else int16_corpus(rng, n_samples)


def decimate_cases(m: int, shift: int) -> list[dict]:
    """The spans of the main K11/K12 test for one M and input kind: every offset, every in_first mod 8, sizes
    from one group to three buffers (several blocks of 256 threads and a partial last one), positions past 2^32
    and 2^33 input samples.  Each span holds exactly what its outputs read, from the sample at in_first, so
    that in_first mod 8 is the case's residue."""
    cases = []
    e = EXTENT[m]
    for oi, off in enumerate(offsets(m)):
        for r in range(8):
            count = [8, 3 * B if oi in (0, 3) else 2056, 8 * 257, 8 * 1000 + 8, 4096, 8 * 513, 24, 8 * 300][r]
            if r < 4:
                o0 = 8 * (100 + 37 * r)
            else:
                target = 2 ** 32 if r < 6 else 2 ** 33          # the span crosses this input sample
                o0 = ((target // m - count // 2) // 8) * 8 + 8 * (r % 2)
            lo = m * (o0 - 240) - e
            in_first = lo - ((lo - r) % 8)
            n_in = m * (o0 + count) + e - in_first
            cases.append(dict(m=m, shift=shift, offset=off, in_first=in_first, n_in=n_in, o0=o0, count=count, seed=oi * 8 + r))
    return cases


def span_bytes(case: dict, rng) -> np.ndarray:
    bps = 2 if case["shift"] < 0 else 4
    return corpus(rng, case["shift"], case["n_in"])[: bps * case["n_in"] - case.get("cut", 0)]


@pytest.mark.parametrize("m", [2, 3, 4, 5])
def test_decimate_cases_cover(m):
    """The generator reaches every in_first mod 8 (so every window alignment sh) for every M and kind, every
    one of K12's 1024 phases per M, and spans across 2^32 and 2^33 input samples."""
    phases = set()
    crossed = set()
    for shift in SHIFTS:
        cases = decimate_cases(m, shift)
        assert {c["in_first"] % 8 for c in cases} == set(range(8))
        assert {window_sh(m, c["o0"] - 240, c["in_first"]) for c in cases} == set(range(0, 16, 2))
        assert max(c["count"] for c in cases) >= 3 * B and min(c["count"] for c in cases) == 8
        for c in cases:
            if c["offset"]:
                phases |= set(SM.phases(c["in_first"], c["n_in"], SM.step(c["offset"], 2_000_000 * m)).tolist())
            for t in (2 ** 32, 2 ** 33):
                if c["in_first"] < t < c["in_first"] + c["n_in"]:
                    crossed.add(t)
    assert phases == set(range(SM.PHASES))
    assert crossed == {2 ** 32, 2 ** 33}


def test_int16_corpus_covers_conversion_edges():
    """The int16 corpus holds both sides of every clamp the conversion can reach at shifts 0, 1, 4, 8 and 15, the
    half-way values k 2^s +- 2^(s-1), and the int16 extremes."""
    v = np.unique(int16_corpus(np.random.default_rng(1), 5000).view("<i2").astype(np.int64))
    assert {-32768, 32767} <= set(v.tolist())
    for s in (0, 1, 4, 8, 15):
        lo, hi = clamp_edges(s)
        assert set(lo + hi) <= set(v.tolist()), s
        if s:
            assert {k * 2 ** s + 2 ** (s - 1) for k in (-1, 0)} | {k * 2 ** s - 2 ** (s - 1) for k in (0, 1)} <= set(v.tolist())
    # at shift 0 both clamps happen, at 8 only the low one, at 15 neither
    assert clamp_edges(0)[0] and clamp_edges(0)[1] and clamp_edges(8)[0] and not clamp_edges(8)[1]
    assert clamp_edges(15) == ([], [])


def edge_cases(m: int, shift: int) -> list[dict]:
    """Span edges: spans that start after the first sample the outputs read (leading no signal), spans cut
    before the last (int16: in_bytes mod 4 = 1, 2, 3; UC8: odd in_bytes), and out_end at every residue mod 8
    inside a body group, inside the carry block and before out_first."""
    e = EXTENT[m]
    bps = 2 if shift < 0 else 4
    o0, count = 8 * 2000, 8 * 300
    lo, hi = m * (o0 - 240) - e, m * (o0 + count) + e
    base = dict(m=m, shift=shift, o0=o0, count=count, limit=NO_LIMIT)
    cases = []
    for k, d in enumerate((1, 3, 6, 13, 8 * m * 10 + 5, m * 240 + 7)):             # leading no signal
        cases.append(dict(base, offset=offsets(m)[k % 4], in_first=lo + d, n_in=hi - lo - d, seed=100 + k))
    for k, (d, cut) in enumerate((1, t) for t in range(1, bps)):                       # trailing, partial last sample
        for back in (1, 5, m * 8 * 20 + 3):
            cases.append(dict(base, offset=offsets(m)[(k + back) % 4], in_first=lo - 3, n_in=hi - lo + 3 - back,
                              cut=cut, seed=200 + 10 * k + back))
    for k, lim in enumerate([o0 + 8 * 17 + t for t in range(8)] + [o0 - 238 + 8 * 5 + t for t in range(8)]
                            + [o0 - 240 - 5, o0 - 238, o0 - 1, o0, o0 + count - 1]):
        cases.append(dict(base, offset=offsets(m)[k % 4], in_first=lo - (k % 8), n_in=hi - lo + (k % 8), limit=lim,
                          seed=300 + k))
    return cases


def test_edge_cases_cover():
    for m in (2, 3, 4, 5):
        for shift in (-1, 8):
            cases = edge_cases(m, shift)
            bps = 2 if shift < 0 else 4
            lo = m * (cases[0]["o0"] - 240) - EXTENT[m]
            assert any(c["in_first"] > lo for c in cases)
            ends = {(bps * c["n_in"] - c.get("cut", 0)) % bps for c in cases}
            assert ends == set(range(bps)), (m, shift)
            lims = [c["limit"] - c["o0"] for c in cases if c["limit"] != NO_LIMIT]
            assert {x % 8 for x in lims if x >= 0} == set(range(8))
            assert {x % 8 for x in lims if -238 <= x < 0} == set(range(8))
            assert any(x < -238 for x in lims)


# ---------------------------------------------------------------- the spectrum's exact frame power, fast


BITREV = SPM.BITREV
TW = [(SM.C[4 * (np.arange(1 << st) << (7 - st))], SM.S[4 * (np.arange(1 << st) << (7 - st))]) for st in range(8)]


def frame_power(x: np.ndarray) -> np.ndarray:
    """spectrum_model.frame_power over [F, 256, 2] (I - 127, Q - 127), each stage's butterflies as whole-array
    operations on a reshaped frame (same arithmetic, same order of roundings)."""
    f = x.shape[0]
    v = (np.asarray(x, np.int64) * SPM.WINDOW[:, None] + 8192) >> 14
    re, im = v[:, BITREV, 0], v[:, BITREV, 1]
    for st in range(8):
        half = 1 << st
        c, s = TW[st]
        re, im = re.reshape(f, -1, 2, half), im.reshape(f, -1, 2, half)
        ar, ai, br, bi = re[:, :, 0], im[:, :, 0], re[:, :, 1], im[:, :, 1]
        tr = (br * c + bi * s + 8192) >> 14
        ti = (bi * c - br * s + 8192) >> 14
        re = np.stack([ar + tr, ar - tr], axis=2).reshape(f, N)
        im = np.stack([ai + ti, ai - ti], axis=2).reshape(f, N)
    return np.roll((re * re + im * im).astype(np.uint64), N // 2, axis=-1)


def power_sum(x: np.ndarray) -> np.ndarray:
    """The sum of frame_power over the frames of x [F * 256, 2], in chunks."""
    x = x.reshape(-1, N, 2)
    out = np.zeros(N, np.uint64)
    for a in range(0, x.shape[0], 4096):
        out += frame_power(x[a: a + 4096]).sum(axis=0, dtype=np.uint64)
    return out


def test_fast_frame_power_is_the_model():
    rng = np.random.default_rng(4)
    x = np.concatenate([rng.integers(-127, 129, (40, N, 2)), np.full((2, N, 2), 128), np.full((2, N, 2), -127)])
    assert np.array_equal(frame_power(x), SPM.frame_power(x))


def spectrum_record(x: np.ndarray, x_first: int, rate: int, b: int) -> np.ndarray:
    """spectrum_model.record with the fast frame power."""
    s0, f = SPM.first_sample(rate, b), SPM.frames(rate, b)
    fr = np.zeros((f * N, 2), np.int64)
    lo = s0 - x_first
    a, e = max(lo, 0), min(lo + f * N, x.shape[0])
    if e > a:
        fr[a - lo: e - lo] = x[a:e]
    out = np.zeros(1, SPM.DTYPE)
    out["buffer"], out["frames"] = b, f
    out["power"][0] = power_sum(fr) if f else 0
    return out[0]


def test_spectrum_record_is_the_model():
    rng = np.random.default_rng(6)
    x = SPM.samples(rng.integers(0, 256, 2 * 700_000, dtype=np.uint8))
    for rate, b, x_first in ((2_400_000, 3, 300_000), (10_000_000, 0, 1234), (2_000_000, 2, 262_100)):
        assert spectrum_record(x, x_first, rate, b).tobytes() == SPM.record(x, rate, b, x_first).tobytes()


RATIO_RATE = {(1, 1): 2_000_000, (5, 6): 2_400_000, (1, 2): 4_000_000, (1, 3): 6_000_000, (1, 4): 8_000_000,
              (1, 5): 10_000_000}


def spectrum_cases(ratio: tuple[int, int], shift: int) -> list[dict]:
    """K13 spans for one ratio and input kind: every (s_b - in_first) mod 8, spans that begin and end inside a
    buffer's frames, first_buffer 0, 1 and past 2^32 input samples, and the saturated, tone and silent frames
    placed at chosen frames."""
    rate = RATIO_RATE[ratio]
    cases = []
    for r in range(8):
        fb = [0, 1, 2 ** 32 // (ratio[1] * B // ratio[0]) + 1, 3][r % 4]
        nb = 1 if ratio[1] >= 4 else 2
        s0, s1 = SPM.first_sample(rate, fb), SPM.first_sample(rate, fb + nb)
        frames0 = SPM.frames(rate, fb)
        if r in (2, 5):           # begins inside the first buffer's frames
            in_first = s0 + N * (frames0 // 3) - r
            n_in = s1 - in_first + 64
        elif r in (3, 6):         # ends inside the last buffer's frames
            in_first = s0 - r
            n_in = (s1 - s0) - N * 7 - 5
        else:
            in_first = s0 - r
            n_in = s1 - s0 + r + 40
        cases.append(dict(ratio=ratio, rate=rate, shift=shift, fb=fb, nb=nb, in_first=in_first, n_in=n_in,
                          seed=r, place=r % 2 == 0))
    return cases


def test_spectrum_cases_cover():
    for ratio in RATIO_RATE:
        for shift in (-1, 8):
            cases = spectrum_cases(ratio, shift)
            sh = {frame_sh(SPM.first_sample(c["rate"], c["fb"]), c["in_first"]) for c in cases}
            assert sh == set(range(0, 16, 2)), ratio
            fbs = {c["fb"] for c in cases}
            assert {0, 1} <= fbs and any(SPM.first_sample(RATIO_RATE[ratio], b) > 2 ** 32 for b in fbs)
            begins = [c for c in cases if c["in_first"] > SPM.first_sample(c["rate"], c["fb"])]
            ends = [c for c in cases if c["in_first"] + c["n_in"] < SPM.first_sample(c["rate"], c["fb"] + c["nb"])]
            assert begins and ends


# ---------------------------------------------------------------- GPU: the harness


@pytest.fixture(scope="module")
def dshim():
    subprocess.run(["make", "-s", "dshim"], cwd=ROOT, check=True)
    lib = ctypes.CDLL(str(DSHIM))
    lib.rate_error.restype = ctypes.c_char_p
    lib.rate_step.restype = ctypes.c_uint32
    lib.rate_step.argtypes = [ctypes.c_int, ctypes.c_int32]
    lib.decimate_run.restype = ctypes.c_int
    lib.decimate_run.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int32, ctypes.c_void_p, ctypes.c_uint64,
                                 ctypes.c_int64, ctypes.c_int64, ctypes.c_uint64, ctypes.c_int64, ctypes.c_int,
                                 ctypes.c_void_p, ctypes.c_void_p]
    lib.spectrum_run.restype = ctypes.c_int
    lib.spectrum_run.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_uint64,
                                 ctypes.c_int64, ctypes.c_int64, ctypes.c_uint32, ctypes.c_void_p]
    P = ctypes.c_void_p
    lib.spectrum_pool_run.restype = ctypes.c_int
    lib.spectrum_pool_run.argtypes = [ctypes.c_uint32, P, ctypes.c_uint64, P, P, ctypes.c_uint64, P, P, P, P, P, P,
                                      ctypes.c_uint32, P]
    return lib


def _ptr(a: np.ndarray):
    return a.ctypes.data if a.size else None


def run_decimate(dshim, m, shift, offset, span, in_first, o0, count, limit, halo):
    span = np.ascontiguousarray(span, np.uint8)
    body = np.zeros(2 * count + GUARD, np.uint8)
    blk = np.zeros(HALO_ALLOC + GUARD, np.uint8)
    rc = dshim.decimate_run(m, shift, offset, _ptr(span), span.size, in_first, o0, count, limit, int(halo),
                            body.ctypes.data, blk.ctypes.data)
    assert rc == 0, dshim.rate_error()
    return body, blk


def model_decimate(m, shift, offset, span, in_first, first, count, limit):
    """Output samples [first, first + count) of the stream whose input from in_first on is the span."""
    uc8 = np.asarray(span, np.uint8) if shift < 0 else IF.convert(span, shift)
    lim = None if limit == NO_LIMIT else limit
    if offset:
        return SM.shift_decimate_range(uc8, m, offset, first, count, limit=lim, in_first=in_first)
    return DM.decimate_range(uc8, m, first, count, limit=lim, in_first=in_first)


def check_decimate(dshim, case, halo):
    """One launch against the model: body, carry block, the carry block's no-signal bytes and every guard byte."""
    m, shift, off, o0, count = case["m"], case["shift"], case["offset"], case["o0"], case["count"]
    limit = case.get("limit", NO_LIMIT)
    span = span_bytes(case, np.random.default_rng(case["seed"] * 31 + m * 7 + shift))
    body, blk = run_decimate(dshim, m, shift, off, span, case["in_first"], o0, count, limit, halo)
    want = model_decimate(m, shift, off, span, case["in_first"], o0 - 238, count + 238, limit)
    what = {k: case[k] for k in ("m", "shift", "offset", "in_first", "o0", "count")} | dict(halo=halo, limit=limit)
    bad = np.flatnonzero(body[: 2 * count] != want[476:])
    assert bad.size == 0, (what, "body", bad[:8].tolist())
    assert (body[2 * count:] == SENTINEL).all(), (what, "written past the body")
    if halo:
        lay = carry_layout()
        for name, (a, b) in lay.items():
            exp = want[:476] if name == "carry" else np.full(b - a, 127, np.uint8)
            bad = np.flatnonzero(blk[a:b] != exp)
            assert bad.size == 0, (what, name, (bad + a)[:8].tolist())
    assert (blk[HALO_ALLOC if halo else 0:] == SENTINEL).all(), (what, "carry block or its guard written")


# ---------------------------------------------------------------- GPU: K11/K12


@pytest.mark.gpu
def test_harness_refuses_bad_requests(dshim):
    span = np.zeros(64, np.uint8)
    out = np.zeros(2 * 8 + GUARD, np.uint8)
    blk = np.zeros(HALO_ALLOC + GUARD, np.uint8)
    good = dict(m=2, shift=-1, off=0, first=0, o0=0, count=8)
    for bad in (dict(m=1), dict(m=6), dict(shift=16), dict(shift=-2), dict(o0=4), dict(count=12), dict(count=0),
                dict(off=1_000_001), dict(m=3, off=-2_000_001)):
        a = good | bad
        assert dshim.decimate_run(a["m"], a["shift"], a["off"], span.ctypes.data, span.size, a["first"], a["o0"],
                                  a["count"], NO_LIMIT, 1, out.ctypes.data, blk.ctypes.data) == -1, bad
    assert dshim.rate_step(2, 1_000_000) == SM.step(1_000_000, 4_000_000)
    for m in (2, 3, 4, 5):
        for off in offsets(m)[1:]:
            assert dshim.rate_step(m, off) == SM.step(off, 2_000_000 * m), (m, off)
    rec = np.zeros(2, SPM.DTYPE)
    assert dshim.spectrum_run(-1, 2, 3, span.ctypes.data, span.size, 0, 0, 1, rec.ctypes.data) == -1
    assert dshim.spectrum_run(16, 1, 1, span.ctypes.data, span.size, 0, 0, 1, rec.ctypes.data) == -1
    assert dshim.spectrum_run(-1, 1, 1, span.ctypes.data, span.size, 0, 0, 0, rec.ctypes.data) == -1


@pytest.mark.gpu
@pytest.mark.parametrize("shift", SHIFTS)
@pytest.mark.parametrize("m", [2, 3, 4, 5])
def test_decimate_equals_model(dshim, m, shift):
    """Every offset x every in_first mod 8, with and without the carry block, one group to three buffers,
    positions across 2^32 and 2^33 input samples: every byte of the launch's zones and guards."""
    for case in decimate_cases(m, shift):
        for halo in (True, False):
            if case["count"] >= B and not halo:
                continue
            check_decimate(dshim, case, halo)


@pytest.mark.gpu
@pytest.mark.parametrize("shift", [-1, 8, 0])
@pytest.mark.parametrize("m", [2, 3, 4, 5])
def test_decimate_span_edges(dshim, m, shift):
    """Leading no signal, trailing partial samples, and out_end anywhere: in a group, in the carry block, before
    out_first."""
    for case in edge_cases(m, shift):
        for halo in (True, False):
            check_decimate(dshim, case, halo)


# ---------------------------------------------------------------- GPU: K13


def spectrum_span(case: dict, rng) -> np.ndarray:
    """The case's span bytes; with place, the saturated, tone and silent frames (and, for int16, frames of the
    int16 extremes) written at chosen frames of its first buffer."""
    shift, n_in = case["shift"], case["n_in"]
    span = corpus(rng, shift, n_in)
    if not case.get("place"):
        return span
    uc8 = TS._saturated_frames()
    special = uc8 if shift < 0 else IF.to_sc16(uc8, min(shift, 8))   # (above 8 the rails are not int16 values)
    bps = 2 if shift < 0 else 4
    s0 = SPM.first_sample(case["rate"], case["fb"])
    at = s0 + N * 2 - case["in_first"]                 # from the buffer's third frame on
    if 0 <= at and at * bps + special.size <= span.size:
        span[at * bps: at * bps + special.size] = special
    if shift >= 0:
        ext = np.tile(np.array([-32768, 32767, 32767, -32768, -32768, -32768, 32767, 32767], "<i2"), N)
        a2 = at + special.size // bps + 3 * N + 17
        ext = ext.view(np.uint8)
        if a2 * bps + ext.size <= span.size:
            span[a2 * bps: a2 * bps + ext.size] = ext
    return span


def run_spectrum(dshim, shift, ratio, span, in_first, fb, nb):
    span = np.ascontiguousarray(span, np.uint8)
    rec = np.zeros(nb + 1, SPM.DTYPE)
    rc = dshim.spectrum_run(shift, ratio[0], ratio[1], _ptr(span), span.size, in_first, fb, nb, rec.ctypes.data)
    assert rc == 0, dshim.rate_error()
    return rec


def assert_records(got, want, what):
    """Every byte of every record."""
    assert got.size == want.size, (what, got.size, want.size)
    bad = [k for k in range(want.size) if got[k].tobytes() != want[k].tobytes()]
    assert not bad, f"{what}: records {bad[:5]} differ (of {want.size})"


def check_records(got, want, what):
    """The launch's records and its guard record, left as the harness filled it."""
    assert_records(got[:-1], want, what)
    assert (np.frombuffer(got[-1:].tobytes(), np.uint8) == SENTINEL).all(), (what, "guard record written")


@pytest.mark.gpu
@pytest.mark.parametrize("shift", [-1, 0, 4, 8, 15])
@pytest.mark.parametrize("ratio", list(RATIO_RATE))
def test_spectrum_equals_model(dshim, ratio, shift):
    """Every frame alignment, spans cut inside a buffer's frames, first_buffer 0, 1 and past 2^32 input samples,
    the saturated, tone and silent frames and the int16 extremes: every record and the guard record, exactly."""
    for case in spectrum_cases(ratio, shift):
        span = spectrum_span(case, np.random.default_rng(case["seed"] + 11 * shift + 101 * ratio[1]))
        x = SPM.samples(span, "uc8" if shift < 0 else "sc16", None if shift < 0 else shift)
        want = np.array([spectrum_record(x, case["in_first"], case["rate"], case["fb"] + k) for k in range(case["nb"])],
                        SPM.DTYPE)
        got = run_spectrum(dshim, shift, ratio, span, case["in_first"], case["fb"], case["nb"])
        check_records(got, want, {k: case[k] for k in ("ratio", "shift", "fb", "in_first", "n_in")})


@pytest.mark.gpu
def test_spectrum_grid_of_300_buffers(dshim):
    """One launch over 300 buffers of 2 MHz UC8 noise (78 MB, 300 x 2 blocks of frames): every buffer is one
    of five base buffers with one frame of its own, so each record is its base's sum with that frame swapped."""
    rng = np.random.default_rng(21)
    nb, nbase = 300, 5
    base = np.stack([np.clip(rng.normal(127, sd, 2 * B), 0, 255).astype(np.uint8) for sd in (3, 20, 60, 120, 400)])
    own = rng.integers(0, 256, (nb, 2 * N), dtype=np.uint8)
    slot = (np.arange(nb) * 37) % (B // N)
    span = np.tile(base, (nb // nbase + 1, 1))[:nb].copy()
    span[np.arange(nb)[:, None], 2 * N * slot[:, None] + np.arange(2 * N)] = own
    base_p = np.stack([frame_power(b.reshape(-1, N, 2).astype(np.int64) - 127) for b in base])
    own_p = frame_power(own.reshape(nb, N, 2).astype(np.int64) - 127)
    want = np.zeros(nb, SPM.DTYPE)
    want["buffer"], want["frames"] = 7 + np.arange(nb), B // N
    for k in range(nb):
        want["power"][k] = base_p[k % nbase].sum(axis=0, dtype=np.uint64) - base_p[k % nbase][slot[k]] + own_p[k]
    assert (want["power"].sum(axis=1) > 0).all()
    got = run_spectrum(dshim, -1, (1, 1), span.reshape(-1), 7 * B, 7, nb)
    check_records(got, want, "300 buffers")


@pytest.mark.gpu
def test_spectrum_ten_mhz_sc16_eight_buffers(dshim):
    """10 MS/s SC16: eight buffers (20480 frames) in one launch from a span past 2^32 input samples."""
    rng = np.random.default_rng(23)
    fb, nb = 2 ** 32 // (5 * B) + 3, 8
    s0, s1 = SPM.first_sample(10_000_000, fb), SPM.first_sample(10_000_000, fb + nb)
    in_first = s0 - 5
    span = (rng.normal(0, 3000, 2 * (s1 - in_first)).clip(-32768, 32767)).astype("<i2").view(np.uint8)
    x = SPM.samples(span, "sc16", 8)
    want = np.array([spectrum_record(x, in_first, 10_000_000, fb + k) for k in range(nb)], SPM.DTYPE)
    check_records(run_spectrum(dshim, 8, (1, 5), span, in_first, fb, nb), want, "10 MS/s sc16")


# ---------------------------------------------------------------- GPU: K13's pool form


def pool_model(job: dict, hist: np.ndarray, stage: np.ndarray) -> np.ndarray:
    """The record of a pool job: stream bytes [hist0, call0) from its history, [call0, call0 + BUF) from its
    call, 127 elsewhere; frames from stream sample `first`."""
    lo, f = 2 * job["first"], job["frames"]
    b = np.full(2 * N * f, 127, np.uint8)
    for src, a0, n in ((hist[job["ho"]:], job["hist0"], job["call0"] - job["hist0"]), (stage[job["so"]:], job["call0"], BUF)):
        a, e = max(a0, lo), min(a0 + n, lo + b.size)
        if e > a:
            b[a - lo: e - lo] = src[a - a0: e - a0]
    out = np.zeros(1, SPM.DTYPE)
    out["buffer"], out["frames"] = job["buffer"], f
    out["power"][0] = power_sum(b.reshape(-1, 2).astype(np.int64) - 127)
    return out[0]


def pool_jobs(rng, n_jobs: int) -> tuple[list[dict], np.ndarray, np.ndarray]:
    """Jobs of three kinds, in turn: 2.4 MS/s buffers whose frames cross call0 with the frame start at each
    even offset mod 16 (and some that start before hist0 or end past call0 + BUF), and 2 MHz buffers
    (hist0 = call0 = 2 first)."""
    jobs, hist_parts, stage_parts = [], [], []
    ho = so = 0
    for k in range(n_jobs):
        kind = k % 3
        if kind == 2:                                       # 2 MHz
            b = 5 + k
            first = b * B
            job = dict(buffer=b, first=first, frames=B // N, hist0=2 * first, call0=2 * first)
            h = np.zeros(0, np.uint8)
        else:
            b = 3 + k // 3 * 7 + kind
            first = SPM.first_sample(2_400_000, b) // 8 * 8 + (k // 3) % 8     # every first mod 8
            frames = SPM.frames(2_400_000, b)
            lo = 2 * first
            cross = lo + 2 * N * (1 + (k * 13) % (frames - 2)) + 2 * (k % 7)
            call0 = cross // 16 * 16
            variant = (k // 3) % 4
            hist0 = (lo - 64) // 16 * 16 if variant != 1 else (lo + 2 * N * 3 + 6) // 16 * 16   # 1: frames before hist0
            if variant == 2:                                # the call ends inside the frames
                call0 = (lo + 2 * N * frames - BUF - 2 * N * 40 - 10) // 16 * 16
            hist0 = min(hist0, call0)
            job = dict(buffer=b, first=first, frames=frames, hist0=hist0, call0=call0)
            h = rng.integers(0, 256, call0 - hist0, dtype=np.uint8)
        s = np.clip(rng.normal(127, 10 + 7 * (k % 11), BUF), 0, 255).astype(np.uint8)
        job["ho"], job["so"] = ho, so
        hist_parts.append(h)
        stage_parts.append(s)
        ho += h.size
        so += BUF
        jobs.append(job)
    return jobs, np.concatenate(hist_parts + [np.zeros(16, np.uint8)]), np.concatenate(stage_parts)


def run_pool(dshim, jobs, hist, stage, max_frames=None):
    n = len(jobs)
    col = lambda key, dt: np.array([j[key] for j in jobs], dt)  # noqa: E731
    ho, so = col("ho", np.uint64), col("so", np.uint64)
    h0, c0, buf, first = col("hist0", np.int64), col("call0", np.int64), col("buffer", np.int64), col("first", np.int64)
    fr = col("frames", np.uint32)
    rec = np.zeros(n + 1, SPM.DTYPE)
    rc = dshim.spectrum_pool_run(n, hist.ctypes.data, hist.size, ho.ctypes.data, stage.ctypes.data, stage.size,
                                 so.ctypes.data, h0.ctypes.data, c0.ctypes.data, buf.ctypes.data, first.ctypes.data,
                                 fr.ctypes.data, int(fr.max()) if max_frames is None else max_frames, rec.ctypes.data)
    assert rc == 0, dshim.rate_error()
    return rec


def test_pool_jobs_cover():
    jobs, _, _ = pool_jobs(np.random.default_rng(0), 256)
    r24 = [j for j in jobs if j["frames"] != B // N]
    assert {(2 * j["first"]) % 16 for j in r24} == set(range(0, 16, 2))
    inside = lambda j, p: 2 * j["first"] < p < 2 * (j["first"] + N * j["frames"])  # noqa: E731
    assert all(inside(j, j["call0"]) or inside(j, j["call0"] + BUF) for j in r24)
    assert any(j["hist0"] > 2 * j["first"] for j in r24)
    assert any(j["call0"] + BUF < 2 * (j["first"] + N * j["frames"]) for j in r24)
    assert {j["frames"] for j in jobs} == {512, 614}


@pytest.mark.gpu
def test_spectrum_pool_equals_model(dshim):
    """256 jobs in one launch, 512- and 614-frame buffers mixed, frames across hist0, call0 and call0 + BUF at
    every frame alignment: every record and the guard record; and with a larger max_frames the same."""
    jobs, hist, stage = pool_jobs(np.random.default_rng(31), 256)
    want = np.array([pool_model(j, hist, stage) for j in jobs], SPM.DTYPE)
    check_records(run_pool(dshim, jobs, hist, stage), want, "256 pool jobs")
    check_records(run_pool(dshim, jobs[:7], hist, stage, max_frames=700), want[:7], "7 pool jobs, max_frames 700")


# ---------------------------------------------------------------- GPU: the receiver pool end to end


@pytest.mark.gpu
def test_pool_of_256_receivers():
    """ReceiverPool(256, max_batch=256, spectrum=True) of UC8, SC16 and SC16Q11 receivers at 2 MHz and 2.4 MS/s
    with staggered starts: each receiver's records are spectrum_model's records of its own stream."""
    kinds = [(2_000_000, "uc8"), (2_400_000, "uc8"), (2_000_000, "sc16"), (2_400_000, "sc16q11"),
             (2_000_000, "sc16q11"), (2_400_000, "sc16")]
    n_rx, calls = 256, 3
    rng = np.random.default_rng(77)
    streams = []
    for r in range(n_rx):
        rate, fmt = kinds[r % len(kinds)]
        if fmt == "uc8":
            s = np.clip(rng.normal(127, 5 + r % 40, calls * BUF), 0, 255).astype(np.uint8)
        else:
            sd = (5 + r % 40) * (256 if fmt == "sc16" else 16)
            s = rng.normal(0, sd, calls * BUF).clip(-32768, 32767).astype("<i2").view(np.uint8)
        streams.append(s)
    with api.ReceiverPool(n_rx, max_batch=n_rx, spectrum=True) as pool:
        for r in range(n_rx):
            pool.set_input_rate(r, kinds[r % len(kinds)][0])
            pool.set_input_format(r, kinds[r % len(kinds)][1])
        start = [r % 3 for r in range(n_rx)]
        for c in range(calls + 2):
            ids = [r for r in range(n_rx) if start[r] <= c < start[r] + calls]
            bufs = []
            for r in ids:
                nb = streams[r].size // calls
                k = c - start[r]
                bufs.append(streams[r][k * nb: (k + 1) * nb])
            pool.ingest(ids, bufs)
        for r in range(n_rx):
            rate, fmt = kinds[r % len(kinds)]
            got = pool.take_spectra(r)
            nb = pool.buffers(r)
            assert nb >= 2 and got.size == nb, (r, nb, got.size)
            x = SPM.samples(streams[r], fmt)
            want = np.array([spectrum_record(x, 0, rate, b) for b in range(nb)], SPM.DTYPE)
            assert_records(got, want, f"receiver {r} {rate} {fmt}")
