"""Every decode path past 2^32 stream samples: positions, timestamps and input offsets of a live receiver
after half an hour.

A stream's absolute positions cross the 32-bit limits early: the 2 MHz output sample index crosses 2^32
after 35.8 minutes, the 2.4 MS/s input sample index after 29.8, an SC16 input byte offset after 7.5-8.9.
The code keeps them in 64 bits; these tests make sure each place that computes one does.

CPU tests: the host build of the resampler at absolute positions (against tests/resample_model.py), the
host resolve at large buffer bases (every path, shifted by base x 131072 with identical statistics and
Beast timestamps mod 2^48), and the pool's host half after 32 770 calls.  GPU tests: K9, K10 and the
pool's resampling and history launches at the same positions, byte for byte; then a silent prefix that
ends past 2^32 output samples, followed by traffic, through the decoder, the receiver pool and the C
host.  Silence is an exact prefix (UC8 127 and int16 zero are magnitude 0, the resampler maps a constant
127 to 127), so the result must be the decode of the traffic alone, shifted by the prefix."""
import ctypes
import subprocess
import threading
from fractions import Fraction

import numpy as np
import pytest

import checker as C
import input_format_model as M
import pool_rate_model as PM
import recover_model as R
import resample_model as RM
import streams as S
import weak_model as W
from dump1090_b200 import api, synth
from test_signal import parse_beast

ROOT = C.ROOT
BUF = api.BUFFER_BYTES
B = api.BUFFER_SAMPLES
CARRY = api.CARRY_BYTES
NO_LIMIT = 2 ** 63 - 1
WRAP = 1 << 48
LIMITS = (2 ** 31, 2 ** 32)
FAR = 2 ** 40                     # samples: a position far beyond both limits
SHIFTS = (0, 4, 8, 15)            # every default (SC16 8, SC16Q11 4) and edge shift

# Absolute quantities a launch computes, per 2 MHz output sample: the output sample and 5q (1), at 2.4 MS/s
# 6q and the input sample (6/5), the input byte at 2 and at 4 bytes a sample (12/5, 24/5); at 2 MHz the
# input byte of a 16-bit stream (4).
RATIOS = {2_400_000: (Fraction(1), Fraction(6, 5), Fraction(12, 5), Fraction(24, 5)),
          2_000_000: (Fraction(1), Fraction(4))}


def crossing_buffers(rate: int) -> list[int]:
    """For each quantity and each 32-bit limit: the first 2 MHz buffer in which the quantity reaches the
    limit, the buffer before and the buffer after it; and one buffer around 2^40 output samples."""
    out = {FAR // B + 3}
    for c in RATIOS[rate]:
        for lim in LIMITS:
            b = int(Fraction(lim) / (c * B))
            assert c * b * B <= lim < c * (b + 1) * B
            out |= {b - 1, b, b + 1}
    bufs = sorted(out)
    # more than one rounding of K9's first period to a multiple of 8 periods (the carry block included)
    assert len({((b * B - CARRY // 2) // 5) % 8 for b in bufs}) > 1
    return bufs


def test_crossing_buffers_reach_the_limits():
    b24, b20 = crossing_buffers(2_400_000), crossing_buffers(2_000_000)
    assert {16383, 16384, 16385, 32767, 32768, 32769} <= set(b20) & set(b24)
    assert 6 * 13653 * B < 5 * 2 ** 31 < 6 * 13654 * B and 13653 in b24                     # 6q, input sample
    assert 4 * 8192 * B == 2 ** 32 and 8192 in b20                                          # SC16 byte at 2 MHz
    assert max(b24) * B > FAR


# ---------------------------------------------------------------- CPU: host build at absolute positions


@pytest.fixture(scope="module")
def shim():
    subprocess.run(["make", "-s", "shim"], cwd=ROOT, check=True)
    lib = ctypes.CDLL(str(ROOT / "tests" / "_build" / "libresample_core_host.so"))
    lib.shim_resample.restype = ctypes.c_int
    lib.shim_resample.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int64, ctypes.c_int64, ctypes.c_size_t,
                                  ctypes.c_int64, ctypes.c_void_p]
    return lib


def _span(rng, first, count, bps=2):
    """Random input bytes of exactly the input samples output samples [first, first + count) read (from
    input sample lo on): a span that holds only the history."""
    lo, hi = RM.input_span(first, count)
    return lo, rng.integers(0, 256, bps * (hi - lo), dtype=np.uint8)


def model_range(data, first, count, in_first, limit=None):
    """Output samples [first, first + count) of the stream whose input samples from in_first on are `data`
    (UC8 bytes at 2.4 MS/s) and no signal elsewhere, by resample_model: the model is the same 5k output
    samples later on input 6k samples later, so the stream is evaluated 5k samples earlier with the
    input after in_first - 6k prefixed by that many no-signal samples."""
    k = in_first // 6
    pad = np.full(2 * (in_first - 6 * k), 127, np.uint8)
    return RM.resample_range(np.concatenate([pad, np.asarray(data, np.uint8)]), first - 5 * k, count,
                             limit=None if limit is None else limit - 5 * k)


def _limited(want, first, limit):
    out = want.copy()
    if limit is not None:
        out[2 * max(limit - first, 0):] = 127
    return out


def test_host_build_at_absolute_positions(shim):
    rng = np.random.default_rng(31)
    for b in crossing_buffers(2_400_000):
        first, count = b * B - CARRY // 2, B + CARRY // 2
        lo, span = _span(rng, first, count)
        want = model_range(span, first, count, lo)
        assert (want != 127).sum() > count                   # the span is signal, not no-signal
        for limit in (None, b * B + 17, first + 3):
            got = np.zeros(2 * count, np.uint8)
            assert shim.shim_resample(span.ctypes.data, span.size, lo, first, count,
                                      NO_LIMIT if limit is None else limit, got.ctypes.data) == 0
            assert np.array_equal(got, _limited(want, first, limit)), (b, limit, np.flatnonzero(got != want)[:5])
        # short ranges starting at every output phase
        for d in range(5):
            f = b * B + d
            lo2, sp2 = _span(rng, f, 23)
            got = np.zeros(46, np.uint8)
            assert shim.shim_resample(sp2.ctypes.data, sp2.size, lo2, f, 23, f + 11, got.ctypes.data) == 0
            assert np.array_equal(got, model_range(sp2, f, 23, lo2, limit=f + 11)), (b, d)


def test_model_range_at_absolute_positions():
    """model_range, on which every resampling test below relies: a stream whose input starts 6k samples
    later gives the same output 5k samples later, and an input start that is not a multiple of 6 samples
    equals the stream prefixed by no-signal samples."""
    rng = np.random.default_rng(3)
    x = rng.integers(0, 256, 4001, dtype=np.uint8)
    want = RM.resample_range(x, -238, 1800, limit=900)
    for k in (1, 2 ** 30 // 5, 2 ** 40 // 5):
        assert np.array_equal(model_range(x, 5 * k - 238, 1800, 6 * k, limit=5 * k + 900), want), k
    for lo in range(1, 13):
        padded = np.concatenate([np.full(2 * lo, 127, np.uint8), x])
        assert np.array_equal(model_range(x, -238, 1800, lo), RM.resample_range(padded, -238, 1800)), lo


# ---------------------------------------------------------------- CPU: host resolve at large buffer bases


# and a base near 2^48 / 6 / 131072 = 357913941.33, chosen per stream so that 6 * sample_pos crosses the
# Beast wrap inside the run
BASES = [0, 2 ** 14, 2 ** 15 - 1, 2 ** 15, 2 ** 15 + 1, 2 ** 24]


def _resolve_streams():
    yield "modes1", C.modes1()
    for kind in ("df4", "seam"):
        yield f"chain_{kind}", S.address_chain(8, kind, seed=5)


def _shifted(msgs, base):
    out = []
    for m in msgs:
        c = m.copy()
        c.sample_pos += base * B
        out.append(c)
    return out


def _check_beast(got, base_msgs, base):
    """The Beast frames at the shifted positions: the base-0 frames with timestamps moved by
    6 x base x 131072 ticks, mod 2^48.  Returns how many wrapped."""
    wrapped = 0
    for g, w in zip(got, base_msgs):
        (tg, ts, sg, fg), = parse_beast(g.beast())
        (tw, tsw, sw, fw), = parse_beast(w.beast())
        assert (tg, sg, fg) == (tw, sw, fw)
        ticks = 6 * (int(w.sample_pos) + base * B) + (int(w.arrival) - 8 if w.arrival else 0)
        assert ts == ticks % WRAP, (base, int(w.sample_pos))
        wrapped += ticks >= WRAP
    return wrapped


@pytest.mark.parametrize("name", ["modes1", "chain_df4", "chain_seam"])
def test_host_resolve_at_large_buffer_bases(name, checker_libs):
    data = dict(_resolve_streams())[name]
    nbuf = data.size // BUF + 1
    msgs, stats, rstats, wstats, arr, rec, wt, wr = W.cpu_decode(data, {}, signal=True)
    tiles = R.tiled(arr, nbuf)
    base0 = api.Resolver()
    base0.run(arr, tiles)
    plain, plain_st = base0.take_messages(), base0.stats()
    assert len(plain) >= 8
    cut = sorted({0, nbuf // 3, 2 * nbuf // 3, nbuf})
    assert len(cut) >= 3
    shards = []
    for a, b in zip(cut[:-1], cut[1:]):
        sel = arr[((arr["t"] >> 17) >= a) & ((arr["t"] >> 17) < b)].copy()
        sel["t"] -= a << 17
        shards.append((sel, R.tiled(sel, b - a), a))
    # the wrap falls at 6 x (base x 131072 + x) = 2^48, x = 43690.67 + k x 131072: the first k past the first message
    x0 = WRAP // 6 - WRAP // 6 // B * B
    wrap_base = WRAP // 6 // B - max(0, -(-(int(plain[0].sample_pos) + 1 - x0) // B))
    wrapped = 0
    for base in BASES + [wrap_base]:
        want = [bytes(m) for m in _shifted(plain, base)]
        res = api.Resolver()
        res.run(arr, tiles, base)
        got = res.take_messages()
        assert [bytes(m) for m in got] == want and res.stats() == plain_st, ("run", base)
        wrapped += _check_beast(got, plain, base)
        res = api.Resolver()
        res.run_shards([(c, t, a + base) for c, t, a in shards])
        assert [bytes(m) for m in res.take_messages()] == want and res.stats() == plain_st, ("shards", base)
        res = api.Resolver()
        for c, t, a in shards:
            res.run_tentative(c, t, a + base)
            res.commit()
        assert [bytes(m) for m in res.take_messages()] == want and res.stats() == plain_st, ("tentative", base)
        res = api.Resolver()
        res.run(arr, tiles, base, recovered=rec, weak=(wt, wr))
        got = res.take_messages()
        assert [bytes(m) for m in got] == [bytes(m) for m in _shifted(msgs, base)], ("weak", base)
        assert (res.stats(), res.recovery_stats(), res.weak_stats()) == (stats, rstats, wstats), ("weak", base)
        _check_beast(got, msgs, base)
    # at the last base the run crosses the 2^48 wrap: some timestamps wrapped and some did not
    assert 0 < wrapped < len(plain)


def _pool_records(batch):
    recs = C.oracle_scan_candidates(batch, fix=1, aggressive=0, cap=400000)
    cands = np.frombuffer(b"".join(bytes(c) for c in recs), dtype=api.CANDIDATE_DTYPE) if recs \
        else np.zeros(0, api.CANDIDATE_DTYPE)
    g = (cands["t"] + 2) // api.TILE_SAMPLES
    cnt = np.bincount(g, minlength=api.tiles_for(batch.size // BUF)).astype(np.uint32)
    tiles = np.zeros(cnt.size, dtype=api.TILE_DTYPE)
    tiles["count"] = cnt
    tiles["offset"] = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.uint32)
    return cands, tiles


def test_pool_resolve_after_32770_calls(checker_libs):
    """modes_pool_resolve on two receivers for 32 770 calls without candidates, one receiver 3 calls
    more, then each its own stream: each equals a single-stream resolve shifted by its own buffer
    count, with identical statistics."""
    n_buf = 6
    streams = [S.address_chain(n_buf, "df4", seed=3), synth.random_traffic(n_buf * B, 700, seed=41)]
    prefix = [32773, 32770]
    empty = np.zeros(0, api.CANDIDATE_DTYPE)
    with api.ReceiverPool(2) as pool:
        for k in range(prefix[1]):
            pool.resolve([k & 1, 1 - (k & 1)], empty, np.zeros(api.tiles_for(4), api.TILE_DTYPE))
        for _ in range(prefix[0] - prefix[1]):
            pool.resolve([0], empty, np.zeros(api.tiles_for(2), api.TILE_DTYPE))
        assert [pool.buffers(r) for r in range(2)] == prefix
        assert all(not any(pool.stats(r).values()) and not pool.take(r) for r in range(2))
        for k in range(n_buf):
            ids = [0, 1] if k % 2 else [1, 0]
            batch = np.full(2 * len(ids) * BUF, 127, dtype=np.uint8)
            for i, r in enumerate(ids):
                if k:
                    batch[(2 * i + 1) * BUF - CARRY: (2 * i + 1) * BUF] = streams[r][k * BUF - CARRY: k * BUF]
                batch[(2 * i + 1) * BUF: (2 * i + 2) * BUF] = streams[r][k * BUF: (k + 1) * BUF]
            pool.resolve(ids, *_pool_records(batch))
        for r in range(2):
            assert pool.buffers(r) == prefix[r] + n_buf
            arr = R.oracle_records(streams[r], {}, drop_eof=1)
            solo = api.Resolver()
            solo.run(arr, R.tiled(arr, n_buf))
            want = solo.take_messages()
            got = pool.take(r)
            assert len(want) > 5
            assert [bytes(m) for m in got] == [bytes(m) for m in _shifted(want, prefix[r])], r
            assert pool.stats(r) == solo.stats(), r


# ---------------------------------------------------------------- GPU: the launches at absolute positions


@pytest.mark.gpu
def test_k9_uc8_at_absolute_positions(gpu_decoder_factory):
    import torch
    dec = gpu_decoder_factory()
    rng = np.random.default_rng(32)
    out = torch.zeros(BUF, dtype=torch.uint8, device="cuda")
    for b in crossing_buffers(2_400_000):
        first, count = b * B - CARRY // 2, B + CARRY // 2
        lo, span = _span(rng, first, count)
        want = model_range(span, first, count, lo)
        d_span = torch.zeros(span.size + 16, dtype=torch.uint8, device="cuda")
        d_span[: span.size] = torch.from_numpy(span).cuda()
        for limit, carry in ((None, True), (b * B + 17, True), (first + 5, False), (None, False)):
            out.fill_(0x5A)
            got_carry = dec.resample_device(d_span.data_ptr(), span.size, lo, b, 1, out.data_ptr(),
                                            out_end=-1 if limit is None else limit, want_carry=carry)
            w = _limited(want, first, limit)
            got = out.cpu().numpy()
            assert np.array_equal(got, w[CARRY:]), (b, limit, carry, np.flatnonzero(got != w[CARRY:])[:5])
            if carry:
                assert got_carry == w[:CARRY].tobytes(), (b, limit)


@pytest.fixture(scope="module")
def dshim_input():
    subprocess.run(["make", "-s", "dshim"], cwd=ROOT, check=True)
    lib = ctypes.CDLL(str(ROOT / "tests" / "_build" / "libinput_device.so"))
    lib.input_error.restype = ctypes.c_char_p
    lib.input_run.restype = ctypes.c_int
    lib.input_run.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int64, ctypes.c_int64, ctypes.c_uint64,
                              ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    return lib


def _input_run(lib, span, in_first, out_first, out_end, halo, rate24, shift):
    body = np.zeros(BUF, np.uint8)
    blk = np.zeros(512, np.uint8)
    rc = lib.input_run(span.ctypes.data, span.size, in_first, out_first, B, NO_LIMIT if out_end is None else out_end,
                       int(halo), int(rate24), shift, body.ctypes.data, blk.ctypes.data)
    assert rc == 0, lib.input_error()
    return body, blk


def _carry_block(want476):
    blk = np.full(512, 127, np.uint8)
    blk[4:480] = want476
    return blk


@pytest.mark.gpu
@pytest.mark.parametrize("rate", [2_000_000, 2_400_000], ids=["k10", "k9_int16"])
def test_int16_launches_at_absolute_positions(dshim_input, rate):
    rng = np.random.default_rng(33)
    for b in crossing_buffers(rate):
        o0 = b * B
        if rate == 2_400_000:
            first, count = o0 - CARRY // 2, B + CARRY // 2
            lo, span = _span(rng, first, count, bps=4)
        else:                                        # K10's span starts at the carry block's 240 samples
            first, count = o0 - 240, B + 240
            lo, span = first, rng.integers(0, 256, 4 * count, dtype=np.uint8)
        for s in SHIFTS:
            y = M.convert(span, s)
            want = model_range(y, first, count, lo) if rate == 2_400_000 else y
            for limit, halo in ((None, True), (o0 + 17, True), (o0 + 5, False)):
                w = _limited(want, first, limit)
                body, blk = _input_run(dshim_input, span, lo, o0, limit, halo, rate == 2_400_000, s)
                assert np.array_equal(body, w[-BUF:]), (b, s, limit, np.flatnonzero(body != w[-BUF:])[:5])
                if halo:
                    assert np.array_equal(blk, _carry_block(w[-BUF - CARRY: -BUF])), (b, s, limit)
                else:
                    assert (blk == 0x5A).all(), (b, s)


@pytest.fixture(scope="module")
def dshim_pool():
    subprocess.run(["make", "-s", "dshim"], cwd=ROOT, check=True)
    lib = ctypes.CDLL(str(ROOT / "tests" / "_build" / "libresample_pool_device.so"))
    args = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t,
            ctypes.c_void_p, ctypes.c_uint32]
    for name in ("rpool_resample", "rpool_history"):
        getattr(lib, name).restype = ctypes.c_int
        getattr(lib, name).argtypes = args
    lib.rpool_error.restype = ctypes.c_char_p
    return lib


RS_JOB = np.dtype([(f, np.int64) for f in ("hist_off", "stage_off", "hist0", "call0", "out_first", "pad_tail_off", "data_off")])
HIST_JOB = np.dtype([(f, np.int64) for f in ("hist_off", "stage_off", "hist0", "call0", "keep", "out_off")])


def _receiver_call(c):
    """A 2.4 MS/s pool receiver's state before its call c (as pool_rate_model.receiver_calls, for any c):
    (hist0, call0, buffer m, completes, keep after the call), stream byte positions."""
    m = PM.ready_buffers(c * (BUF // 2))
    hist0 = PM.history_keep(m, 0)
    done = PM.ready_buffers((c + 1) * (BUF // 2)) > m
    return hist0, c * BUF, m, done, PM.history_keep(m + done, hist0)


def _pool_calls():
    """Calls whose stream byte offsets straddle 2^31, 2^32 and 2^33, and whose output crosses 2^32 samples."""
    picks = set()
    for lim in (2 ** 31, 2 ** 32, 2 ** 33):
        c = lim // BUF
        picks |= set(range(c - 2, c + 3))
    c = 6 * 2 ** 32 // (5 * (BUF // 2))                       # the call that completes 2 MHz buffer 32768
    picks |= set(range(c - 3, c + 4))
    picks.add(FAR // B)
    return sorted(picks)


@pytest.mark.gpu
def test_pool_launches_at_absolute_positions(dshim_pool):
    rng = np.random.default_rng(34)
    calls = [(c, *_receiver_call(c)) for c in _pool_calls()]
    rs = [x for x in calls if x[4]]
    assert len(rs) >= 8 and any(h < 2 ** 32 <= c0 for _, h, c0, _, _, _ in calls)   # a history across 2^32
    assert any(m * B < 2 ** 32 <= (m + 1) * B for _, _, _, m, _, _ in rs)
    assert any(k > 2 ** 32 for *_, k in calls)                  # a history job whose keep is past 2^32
    half = 600_000
    hist = np.full(2 * len(calls) * half, 0xA5, np.uint8)
    stage = np.zeros(len(calls) * BUF, np.uint8)
    local = []
    for i, (c, hist0, call0, m, done, keep) in enumerate(calls):
        x = rng.integers(0, 256, call0 + BUF - hist0, dtype=np.uint8)   # stream bytes [hist0, call0 + BUF)
        assert call0 - hist0 <= half
        hist[2 * i * half: 2 * i * half + call0 - hist0] = x[: call0 - hist0]
        stage[i * BUF: (i + 1) * BUF] = x[call0 - hist0:]
        local.append(x)
    jobs = np.zeros(len(rs), RS_JOB)
    want = []
    for p, (c, hist0, call0, m, done, keep) in enumerate(rs):
        i = [x[0] for x in calls].index(c)
        jobs[p] = (2 * i * half if call0 > hist0 else -1, i * BUF, hist0, call0, m * B, (2 * p + 1) * BUF - CARRY,
                   (2 * p + 1) * BUF)
        want.append(model_range(local[i], m * B - CARRY // 2, B + CARRY // 2, hist0 // 2))
    out = np.full(2 * len(rs) * BUF, 0x3C, np.uint8)
    rc = dshim_pool.rpool_resample(hist.ctypes.data, hist.size, stage.ctypes.data, stage.size, out.ctypes.data, out.size,
                                   jobs.ctypes.data, jobs.size)
    assert rc == 0, dshim_pool.rpool_error()
    for p in range(len(rs)):
        assert (out[2 * p * BUF: (2 * p + 1) * BUF - CARRY] == 0x3C).all(), p
        got = out[(2 * p + 1) * BUF - CARRY: (2 * p + 2) * BUF]
        assert np.array_equal(got, want[p]), (rs[p][:4], np.flatnonzero(got != want[p])[:5])
    # the history step: the other half holds the stream bytes [keep, call0 + BUF)
    hjobs = np.zeros(len(calls), HIST_JOB)
    for i, (c, hist0, call0, m, done, keep) in enumerate(calls):
        hjobs[i] = (2 * i * half if call0 > hist0 else -1, i * BUF, hist0, call0, keep, (2 * i + 1) * half)
    hout = hist.copy()
    rc = dshim_pool.rpool_history(hist.ctypes.data, hist.size, stage.ctypes.data, stage.size, hout.ctypes.data, hout.size,
                                  hjobs.ctypes.data, hjobs.size)
    assert rc == 0, dshim_pool.rpool_error()
    for i, (c, hist0, call0, m, done, keep) in enumerate(calls):
        n = call0 + BUF - keep
        o = (2 * i + 1) * half
        assert np.array_equal(hout[o: o + n], local[i][keep - hist0:]), c
        assert (hout[o + n: o + half] == 0xA5).all(), c


# ---------------------------------------------------------------- GPU: a silent prefix, then traffic

PREFIX_BUFFERS = 32770                      # 2 MHz buffers of silence: past 2^32 output samples
PINNED = 192 << 20
ODD_CALL = 12_345_679                       # one call of this size, so that calls and batches do not line up
CHUNK = 100003


@pytest.fixture(scope="module")
def pinned():
    """One reusable page-locked buffer the silent prefixes are fed from."""
    buf = api.PinnedBuffer(PINNED)
    yield buf
    buf.free()


# name: (input_format, input_rate)
INPUTS = {"uc8_2m": ("uc8", 2_000_000), "uc8_24": ("uc8", 2_400_000), "sc16q11_2m": ("sc16q11", 2_000_000),
          "sc16_24": ("sc16", 2_400_000)}
SILENCE = {"uc8": 127, "sc16": 0, "sc16q11": 0}
SCALE = {"uc8": 1.0, "sc16": 256.0, "sc16q11": 16.0}
_x = {}


def traffic(name):
    """About 10 buffers of a 10 dB fleet (weak frames, known aircraft) in the input's format and rate."""
    if name not in _x:
        fmt, rate = INPUTS[name]
        _x[name] = synth.fleet_at_rate(10, 3200, 11, sample_rate=rate, dtype="uc8" if fmt == "uc8" else "sc16",
                                       scale=SCALE[fmt])[0]
    return _x[name]


def prefix_bytes(name) -> int:
    """The silent prefix: PREFIX_BUFFERS 2 MHz buffers (at 2.4 MS/s 6 x 131072 x 6554 input samples)."""
    fmt, rate = INPUTS[name]
    n_in = PREFIX_BUFFERS * B if rate == 2_000_000 else 6 * B * (PREFIX_BUFFERS // 5)
    assert 5 * n_in == (6 if rate == 2_400_000 else 5) * PREFIX_BUFFERS * B
    return n_in * (2 if fmt == "uc8" else 4)


def feed_prefix(feed, pinned, fmt, total):
    """Feed `total` bytes of silence from the pinned buffer: one odd-sized call, then whole buffers."""
    pinned.array[:] = SILENCE[fmt]
    left = total
    first = True
    while left:
        n = min(ODD_CALL if first else PINNED, left)
        feed(pinned.ptr, n)
        left -= n
        first = False


def fields(m) -> tuple:
    return tuple(bytes(getattr(m, f)) if f in ("msg", "flight", "pad1") else getattr(m, f) for f, _ in api.Message._fields_)


def _run_decoder(factory, name, pinned, with_prefix, **kw):
    fmt, rate = INPUTS[name]
    dec = factory(input_format=fmt, input_rate=rate, **kw)
    prefix_levels = np.zeros(0, api.LEVEL_DTYPE)
    if with_prefix:
        feed_prefix(dec.process_ptr, pinned, fmt, prefix_bytes(name))
        assert not dec.take_messages() and not any(dec.stats().values())
        if kw.get("levels"):
            lv = dec.take_levels()
            assert list(lv["buffer"]) == list(range(lv.size)) and lv.size >= PREFIX_BUFFERS - 1
            assert (lv["peak"] == 0).all() and (lv["clipped"] == 0).all() and (lv["sum_mag"] == 0).all()
            assert (lv["sum_power"] == 0).all() and (lv["n_samples"] == B).all()
            prefix_levels = lv
    x = traffic(name)
    for off in range(0, x.size, CHUNK):
        dec.process(x[off: off + CHUNK])
    dec.finish()
    res = dict(msgs=dec.take_messages(), stats=dec.stats())
    if kw.get("levels"):
        lv = dec.take_levels()
        res["levels"] = np.concatenate([prefix_levels, lv])
    if kw.get("recover"):
        res["recovery"] = dec.recovery_stats()
        res["weak"] = dec.weak_recovery_stats()
    dec.close()
    return res


def _assert_shifted(got, want, shift_buffers, what):
    assert len(got["msgs"]) == len(want["msgs"]) > 20, (what, len(got["msgs"]), len(want["msgs"]))
    for k, (g, w) in enumerate(zip(got["msgs"], _shifted(want["msgs"], shift_buffers))):
        assert fields(g) == fields(w), (what, k, g.raw_line(), w.raw_line(), g.sample_pos, w.sample_pos)
        assert g.beast() == w.beast(), (what, k)
    assert all(int(m.sample_pos) >= 2 ** 32 for m in got["msgs"]), what
    for key in ("stats", "recovery", "weak"):
        assert got.get(key) == want.get(key), (what, key)
    if "levels" in want:
        lv, wl = got["levels"], want["levels"].copy()
        assert lv.size == shift_buffers + wl.size, what
        assert list(lv["buffer"][:shift_buffers]) == list(range(shift_buffers))
        assert (lv["peak"][:shift_buffers] == 0).all() and (lv["clipped"][:shift_buffers] == 0).all()
        wl["buffer"] += shift_buffers
        assert np.array_equal(lv[shift_buffers:], wl), what


ALL_PASSES = dict(signal=True, arrival=True, levels=True, recover=True, weak_preambles=True)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(INPUTS))
def test_decoder_after_silent_prefix(name, pinned, gpu_decoder_factory):
    for drop in (0, 1):
        kw = dict(ALL_PASSES, drop_eof_buffer=drop)
        want = _run_decoder(gpu_decoder_factory, name, pinned, False, **kw)
        got = _run_decoder(gpu_decoder_factory, name, pinned, True, **kw)
        _assert_shifted(got, want, PREFIX_BUFFERS, (name, drop))
        assert any(m.arrival for m in got["msgs"]) and any(m.signal for m in got["msgs"]), name


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["uc8_2m", "sc16_24"])
@pytest.mark.parametrize("kw", [dict(gpu_resolve=1, signal=True), dict(n_gpus=2, signal=True)], ids=["gpu_resolve", "gpus2"])
def test_decoder_after_silent_prefix_other_paths(name, kw, pinned, gpu_decoder_factory):
    want = _run_decoder(gpu_decoder_factory, name, pinned, False, **kw)
    got = _run_decoder(gpu_decoder_factory, name, pinned, True, **kw)
    _assert_shifted(got, want, PREFIX_BUFFERS, (name, kw))


POOL_PREFIX_CALLS = 39330                  # at this count the 2.4 MS/s receiver's output passes 2^32 samples too


@pytest.mark.gpu
def test_pool_after_silent_prefix(gpu_decoder_factory):
    """ReceiverPool(2): a 2 MHz and a 2.4 MS/s receiver, 39 330 calls of silence from one pinned buffer,
    then each its own traffic, out of lock step; each equals its single-stream decode shifted by its own
    prefix."""
    rates = [2_000_000, 2_400_000]
    n_calls = [10, 12]
    xs = [np.ascontiguousarray(synth.fleet_at_rate(10, 3400, 21 + r, sample_rate=rates[r])[0][: n_calls[r] * BUF])
          for r in range(2)]
    assert all(x.size == n * BUF for x, n in zip(xs, n_calls))
    kw = dict(signal=True, arrival=True)
    buf = api.PinnedBuffer(BUF)
    try:
        buf.array[:] = 127
        with api.ReceiverPool(2, **kw) as pool:
            pool.set_input_rate(1, rates[1])
            ids = np.array([0, 1], dtype=np.uint32)
            ptrs = (ctypes.c_void_p * 2)(buf.ptr, buf.ptr)
            for _ in range(POOL_PREFIX_CALLS):
                pool.ingest_ptrs(ids, ptrs)
            done = [pool.buffers(r) for r in range(2)]
            assert done[0] == POOL_PREFIX_CALLS and done[1] == PM.ready_buffers(POOL_PREFIX_CALLS * (BUF // 2))
            assert all(not any(pool.stats(r).values()) for r in range(2))
            shift = [POOL_PREFIX_CALLS, 5 * POOL_PREFIX_CALLS // 6]      # 2 MHz buffers of each prefix
            assert shift[1] * B > 2 ** 32 and 6 * shift[1] == 5 * POOL_PREFIX_CALLS
            nxt = [0, 0]
            k = 0
            while nxt[0] < n_calls[0] or nxt[1] < n_calls[1]:
                part = [r for r in ((0, 1) if k % 3 else (1,)) if nxt[r] < n_calls[r]]
                pool.ingest(part, [xs[r][nxt[r] * BUF: (nxt[r] + 1) * BUF] for r in part])
                for r in part:
                    nxt[r] += 1
                k += 1
            for r in range(2):
                dec = gpu_decoder_factory(input_rate=rates[r], **kw)
                dec.process(xs[r])                                   # every complete buffer, no EOF buffer
                want = dict(msgs=dec.take_messages(), stats=dec.stats())
                got = dict(msgs=pool.take(r), stats=pool.stats(r))
                _assert_shifted(got, want, shift[r], ("pool", r))
                want_buffers = n_calls[0] if r == 0 else PM.ready_buffers(n_calls[1] * (BUF // 2))
                assert pool.buffers(r) == shift[r] + want_buffers, r
    finally:
        buf.free()


# C host: `--ifile -` fed from a thread; name: (input, extra options)
CLI = {"uc8_2m": [], "sc16q11_24": ["--sample-rate", "2400000", "--iformat", "SC16Q11"]}


def _cli_x(name):
    if name == "uc8_2m":
        return traffic("uc8_2m")
    return synth.fleet_at_rate(10, 3200, 12, sample_rate=2_400_000, dtype="sc16", scale=SCALE["sc16q11"])[0]


def _run_cli(args, x, prefix_total, fill):
    """The C host on stdin: prefix_total bytes of `fill` from one reusable buffer, then x, written by a
    thread that is joined before returning."""
    proc = subprocess.Popen([str(ROOT / "dump1090-b200"), "--ifile", "-", *args], stdin=subprocess.PIPE,
                            stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    block = np.full(64 << 20, fill, np.uint8)
    err = []

    def write():
        try:
            left = prefix_total
            first = True
            while left:
                n = min(ODD_CALL if first else block.size, left)
                proc.stdin.write(memoryview(block)[:n])
                left -= n
                first = False
            proc.stdin.write(x.tobytes())
        except Exception as e:                               # the host exited early: its return code says why
            err.append(e)
        finally:
            proc.stdin.close()

    stderr = []
    threads = [threading.Thread(target=write), threading.Thread(target=lambda: stderr.append(proc.stderr.read()))]
    for t in threads:
        t.start()
    out = proc.stdout.read()
    for t in threads:
        t.join()
    rc = proc.wait()
    assert rc == 0 and not err, (args, rc, stderr[0][-500:], err)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CLI))
def test_c_host_after_silent_prefix(name):
    x = _cli_x(name)
    fill, bps = (127, 2) if name == "uc8_2m" else (0, 4)
    n_in = PREFIX_BUFFERS * B if name == "uc8_2m" else 6 * B * (PREFIX_BUFFERS // 5)
    P = PREFIX_BUFFERS * B                                    # 2 MHz samples of the prefix
    raw = _run_cli(CLI[name] + ["--raw"], x, bps * n_in, fill)
    assert _run_cli(CLI[name] + ["--raw"], x, 0, fill) == raw and raw.count(b"\n") > 20
    got = parse_beast(_run_cli(CLI[name] + ["--beast", "--arrival"], x, bps * n_in, fill))
    want = parse_beast(_run_cli(CLI[name] + ["--beast", "--arrival"], x, 0, fill))
    assert len(got) == len(want) == raw.count(b"\n")
    assert [(t, s, f) for t, _, s, f in got] == [(t, s, f) for t, _, s, f in want]
    assert [ts for _, ts, _, _ in got] == [(ts + 6 * P) % WRAP for _, ts, _, _ in want]
