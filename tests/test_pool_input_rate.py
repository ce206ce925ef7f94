"""2.4 MS/s receivers in the receiver pool (modes_pool_set_input_rate): each receiver's messages, fields,
sample_pos, statistics and level records equal the 2 MHz decode (without the EOF buffer) of the first
modes_pool_buffers(r) buffers of its resampled stream (tests/resample_model.py), with 2 MHz and 2.4 MS/s
receivers mixed in one call.

CPU tests check the schedule (tests/pool_rate_model.py: which call completes which 2 MHz buffer) against
the streaming model, and the setter's refusals that need no device.  GPU tests check the pool's resampling launches byte for byte
through a device harness over the product's own object, and the contract through ReceiverPool."""
import ctypes
import subprocess

import numpy as np
import pytest

import checker as C
import pool_rate_model as PM
import resample_model as RM
from dump1090_b200 import api, synth
from test_pool import _schedule

ROOT = C.ROOT
DSHIM = ROOT / "tests" / "_build" / "libresample_pool_device.so"
BUF = api.BUFFER_BYTES
B = api.BUFFER_SAMPLES
CARRY = api.CARRY_BYTES
IN_PER_CALL = BUF // 2                     # input samples one call brings
FLAG_SETS = [dict(), dict(aggressive=1), dict(fix=0), dict(check_crc=0)]   # test_pool's four


# ---------------------------------------------------------------- CPU: the schedule


def test_ready_buffers_is_the_streaming_schedule():
    """A 2 MHz buffer completes in the call after which the streaming model has emitted all of its
    samples: at most one per call, none on the first call, and the exact count after every call."""
    s = RM.Streaming()
    rng = np.random.default_rng(5)
    emitted = 0
    per_call = []
    for k in range(1, 61):
        emitted += s.feed(rng.integers(0, 256, BUF, dtype=np.uint8)).size // 2
        assert PM.ready_buffers(k * IN_PER_CALL) == emitted // B, k
        per_call.append(emitted // B)
    steps = np.diff([0] + per_call)
    assert per_call[0] == 0 and steps.max() == 1
    assert 8 <= int((steps == 0).sum()) <= 12                  # about one call in six completes nothing
    # the rule itself: buffer m completes once the input its last sample reads has arrived
    assert [PM.ready_buffers(n) for n in (0, 157_288, 157_289)] == [0, 0, 1]
    for n in (157_289, 157_290, 5 * IN_PER_CALL, 10 ** 7):
        m = PM.ready_buffers(n)
        assert RM.input_span(0, m * B)[1] <= n < RM.input_span(0, (m + 1) * B)[1]


def test_setter_refusals_without_a_device():
    with api.ReceiverPool(3, max_batch=2) as pool:
        with pytest.raises(RuntimeError, match="not supported"):
            pool.set_input_rate(0, 2_400_001)
        with pytest.raises(RuntimeError, match="not supported"):
            pool.set_input_rate(0, 0)
        with pytest.raises(RuntimeError, match="out of range"):
            pool.set_input_rate(3, 2_400_000)
        pool.set_input_rate(1, 2_400_000)                       # before any call: accepted, and again
        pool.set_input_rate(1, 2_000_000)
        pool.set_input_rate(1, 2_400_000)
    with pytest.raises(RuntimeError, match="not supported"):
        api.ReceiverPool(2, input_rate=2_400_001)
    with api.ReceiverPool(2, input_rate=2_400_000) as pool:
        for r in range(2):
            pool.set_input_rate(r, 2_400_000)
    assert "modes_pool_set_input_rate" in api.EXPORTS


# ---------------------------------------------------------------- GPU: the launches byte for byte


@pytest.fixture(scope="module")
def dshim():
    subprocess.run(["make", "-s", "dshim"], cwd=ROOT, check=True)
    lib = ctypes.CDLL(str(DSHIM))
    args = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t,
            ctypes.c_void_p, ctypes.c_uint32]
    for name in ("rpool_resample", "rpool_history"):
        getattr(lib, name).restype = ctypes.c_int
        getattr(lib, name).argtypes = args
    lib.rpool_error.restype = ctypes.c_char_p
    return lib


RS_JOB = np.dtype([(f, np.int64) for f in ("hist_off", "stage_off", "hist0", "call0", "out_first", "pad_tail_off", "data_off")])
HIST_JOB = np.dtype([(f, np.int64) for f in ("hist_off", "stage_off", "hist0", "call0", "keep", "out_off")])


def _call(lib, name, hist, stage, out, jobs):
    rc = getattr(lib, name)(hist.ctypes.data, hist.size, stage.ctypes.data, stage.size, out.ctypes.data, out.size,
                            jobs.ctypes.data, jobs.size)
    assert rc == 0, lib.rpool_error().decode()


@pytest.mark.gpu
def test_pool_kernels_equal_model(dshim):
    """One launch resamples receivers at different input phases (the first buffer, whose carry is made of
    negative samples, included) with histories in both halves, beside 2 MHz pass-through jobs; the
    history step keeps exactly the bytes later calls read."""
    rng = np.random.default_rng(12)
    n_calls = 14
    x = [rng.integers(0, 256, n_calls * BUF, dtype=np.uint8) for _ in range(3)]
    calls = PM.receiver_calls(n_calls)
    done_at = [c for c, st in enumerate(calls) if st[3]]
    assert done_at[0] == 1 and len(done_at) >= 10
    picks = [done_at[0], done_at[1], done_at[2], done_at[5], done_at[6], done_at[-1]]
    assert {c % 2 for c in picks} == {0, 1}                     # histories in both halves
    half = 600_000                                              # bytes per history half (the pool's: about 577 000)
    hist = np.full(2 * len(picks) * half, 0xA5, np.uint8)
    n_pass = 3
    stage = np.zeros((len(picks) + n_pass) * BUF, np.uint8)
    n_pairs = len(picks) + n_pass
    sentinel = 0x3C
    batch = np.full(2 * n_pairs * BUF, sentinel, np.uint8)
    jobs = np.zeros(n_pairs, RS_JOB)
    hjobs = np.zeros(len(picks), HIST_JOB)
    want = {}
    order = rng.permutation(n_pairs)                            # jobs and pairs in mixed order
    for i, c in enumerate(picks):
        hist0, call0, m, done, keep = calls[c]
        xs = x[i % 3]
        h_off = (2 * i + c % 2) * half
        hist[h_off: h_off + call0 - hist0] = xs[hist0: call0]
        stage[i * BUF: (i + 1) * BUF] = xs[call0: call0 + BUF]
        p = int(order[i])
        jobs[p] = (h_off if call0 > hist0 else -1, i * BUF, hist0, call0, m * B, (2 * p + 1) * BUF - CARRY, (2 * p + 1) * BUF)
        want[p] = RM.resample_range(xs, m * B - CARRY // 2, B + CARRY // 2)
        hjobs[i] = (h_off if call0 > hist0 else -1, i * BUF, hist0, call0, keep, (2 * i + 1 - c % 2) * half)
    for k in range(n_pass):
        i = len(picks) + k
        stage[i * BUF: (i + 1) * BUF] = rng.integers(0, 256, BUF, dtype=np.uint8)
        p = int(order[i])
        jobs[p] = (-1, i * BUF, 0, 0, -1, 0, (2 * p + 1) * BUF)
        want[p] = np.concatenate([np.full(CARRY, sentinel, np.uint8), stage[i * BUF: (i + 1) * BUF]])
    out = batch.copy()
    _call(dshim, "rpool_resample", hist, stage, out, jobs)
    for p in range(n_pairs):
        pad, data = out[2 * p * BUF: (2 * p + 1) * BUF], out[(2 * p + 1) * BUF: (2 * p + 2) * BUF]
        assert (pad[: BUF - CARRY] == sentinel).all(), p          # the pad buffer's head is never written
        got = np.concatenate([pad[BUF - CARRY:], data])
        bad = np.flatnonzero(got != want[p])
        assert bad.size == 0, (p, bad[:5])
    first = int(order[0])                                       # picks[0] is the receiver's first buffer: its
    assert (out[(2 * first + 1) * BUF - CARRY: (2 * first + 1) * BUF - 16] == 127).all()   # carry sees no input but at its end
    # the history step: the new half holds the stream bytes [keep, call0 + BUF), the old half is untouched
    hout = hist.copy()
    _call(dshim, "rpool_history", hist, stage, hout, hjobs)
    for i, c in enumerate(picks):
        hist0, call0, m, done, keep = calls[c]
        xs = x[i % 3]
        o = (2 * i + 1 - c % 2) * half
        n = call0 + BUF - keep
        assert n <= half
        assert np.array_equal(hout[o: o + n], xs[keep: call0 + BUF]), c
        assert (hout[o + n: o + half] == 0xA5).all(), c
        h = (2 * i + c % 2) * half
        assert np.array_equal(hout[h: h + half], hist[h: h + half]), c


# ---------------------------------------------------------------- GPU: the contract


N_CALLS = 5                                                     # calls per receiver


def _fleet(seed, snr):
    nframes = -(-N_CALLS * IN_PER_CALL // 480) + 2
    s = synth.fleet_at_rate(snr, nframes, seed)[0]
    assert s.size >= N_CALLS * BUF
    return np.ascontiguousarray(s[: N_CALLS * BUF])


def _mixed_streams():
    """Receivers 0-3 at 2.4 MS/s (two fleets, two random_traffic streams read as 2.4 MS/s), 4-6 at 2 MHz."""
    s = [_fleet(30, 14), _fleet(31, 20)]
    for r in (2, 3):
        s.append(synth.random_traffic(N_CALLS * B, 120 * N_CALLS + 37 * r, seed=200 + r))
    for r in (4, 5, 6):
        s.append(synth.random_traffic(N_CALLS * B, 120 * N_CALLS + 37 * r, seed=100 + r))
    return s, [2_400_000] * 4 + [2_000_000] * 3


def _pool(n_rx, rates, **kw):
    pool = api.ReceiverPool(n_rx, **kw)
    for r, hz in enumerate(rates):
        pool.set_input_rate(r, hz)
    return pool


def _run_schedule(pool, streams, schedule, max_batch):
    nxt = [0] * len(streams)
    for ids in schedule:
        for lo in range(0, len(ids), max_batch):
            part = ids[lo: lo + max_batch]
            pool.ingest(part, [streams[r][nxt[r] * BUF: (nxt[r] + 1) * BUF] for r in part])
            for r in part:
                nxt[r] += 1
    return nxt


def _decoded(stream, rate, k):
    """The 2 MHz bytes of a receiver's first k buffers."""
    return RM.resample_range(stream, 0, k * B) if rate == 2_400_000 else stream[: k * BUF]


def fields(m) -> tuple:
    return tuple(bytes(getattr(m, f)) if f in ("msg", "flight", "pad1") else getattr(m, f) for f, _ in api.Message._fields_)


def _assert_same(got, want, what):
    assert len(got) == len(want), (what, len(got), len(want))
    for k, (g, w) in enumerate(zip(got, want)):
        assert fields(g) == fields(w), (what, k, g.raw_line(), w.raw_line())


@pytest.mark.gpu
@pytest.mark.parametrize("kw", FLAG_SETS, ids=lambda k: "-".join(f"{a}{b}" for a, b in k.items()) or "default")
def test_mixed_pool_equals_oracle(kw, checker_libs, gpu_decoder_factory):
    streams, rates = _mixed_streams()
    n_rx = len(streams)
    cfg = dict(fix_errors=kw.get("fix", 1), aggressive=kw.get("aggressive", 0), check_crc=kw.get("check_crc", 1))
    with _pool(n_rx, rates, max_batch=5, **cfg) as pool:
        _run_schedule(pool, streams, _schedule(n_rx, N_CALLS, seed=4), 5)
        for r in range(n_rx):
            k = pool.buffers(r)
            assert k == (PM.ready_buffers(N_CALLS * IN_PER_CALL) if rates[r] == 2_400_000 else N_CALLS), r
            msgs, stats = C.oracle_decode(_decoded(streams[r], rates[r], k), drop_eof=1, **kw)
            got = pool.take(r)
            assert [m.raw_line() for m in got] == [m.hexline() for m in msgs], f"receiver {r}"
            assert [C.msg_fields(m, with_pos=True) for m in got] == [C.msg_fields(m, with_pos=True) for m in msgs], r
            assert list(pool.stats(r).values()) == stats, f"receiver {r}"
            if r == 0:
                got0 = got
        # receiver 0 against the single-stream 2.4 MS/s decoder on the same bytes, at the same buffers
        dec = gpu_decoder_factory(input_rate=2_400_000, **cfg)
        dec.process(streams[0])
        _assert_same(got0, dec.take_messages(), "single stream")
        assert dec.stats() == pool.stats(0)


SWITCHES = [dict(signal=True), dict(arrival=True, signal=True), dict(levels=True), dict(recover=True),
            dict(recover=True, weak_preambles=True)]


@pytest.mark.gpu
@pytest.mark.parametrize("sw", SWITCHES, ids=["signal", "arrival", "levels", "recover", "weak"])
def test_every_switch_equals_single_stream(sw, gpu_decoder_factory):
    streams, rates = _mixed_streams()
    n_rx = len(streams)
    with _pool(n_rx, rates, max_batch=5, **sw) as pool:
        _run_schedule(pool, streams, _schedule(n_rx, N_CALLS, seed=9), 5)
        for r in range(n_rx):
            dec = gpu_decoder_factory(input_rate=rates[r], **sw)
            dec.process(streams[r])                              # every complete buffer, no EOF buffer
            got = pool.take(r)
            _assert_same(got, dec.take_messages(), (sw, r))
            assert pool.stats(r) == dec.stats(), (sw, r)
            if rates[r] == 2_400_000 and r < 2:
                assert got, r                                   # the fleets decode at 2.4 MS/s
            if sw.get("signal") and got:
                assert any(m.signal for m in got), r
            if sw.get("arrival") and got:
                assert any(m.arrival for m in got), r
            if sw.get("levels"):
                lv = pool.take_levels(r)
                assert list(lv["buffer"]) == list(range(pool.buffers(r))), r
                assert np.array_equal(lv, dec.take_levels()), r
            if sw.get("recover"):
                assert pool.recovery_stats(r) == dec.recovery_stats(), r
                assert pool.weak_recovery_stats(r) == dec.weak_recovery_stats(), r


def _expect_lines(stream, rate, k):
    return [m.hexline() for m in C.oracle_decode(_decoded(stream, rate, k), drop_eof=1)[0]]


@pytest.mark.gpu
def test_ingest_shapes(checker_libs):
    streams, rates = _mixed_streams()
    n_rx = len(streams)
    k24 = PM.ready_buffers(N_CALLS * IN_PER_CALL)
    with _pool(n_rx, rates, max_batch=5) as pool:
        # a call in which no named receiver completes a buffer (every first call of a 2.4 MS/s receiver):
        # nothing is decoded, and the collect still pairs with the submit
        pool.ingest([0, 1], [streams[r][:BUF] for r in (0, 1)])
        assert pool.buffers(0) == pool.buffers(1) == 0 and pool.take(0) == [] and pool.take(1) == []
        with pytest.raises(RuntimeError, match="in progress"):
            pool.set_input_rate(0, 2_000_000)
        pool.set_input_rate(4, 2_000_000)                       # not named yet: no stream in progress
    with _pool(n_rx, rates, max_batch=5) as pool:
        # two batches in flight, 2.4 MS/s receivers 0 and 2 in both (each completes nothing in its first
        # call) and a 2 MHz receiver beside them
        nxt = {0: 0, 2: 0, 4: 0}

        def submit(ids):
            pool.submit(ids, [streams[r][nxt[r] * BUF: (nxt[r] + 1) * BUF] for r in ids])
            for r in ids:
                nxt[r] += 1

        submit([0, 4])
        for k in range(1, N_CALLS):
            submit([2, 0, 4])
            pool.collect()
        submit([2])
        pool.collect()
        pool.collect()
        with pytest.raises(RuntimeError, match="no batch in flight"):
            pool.collect()
        assert pool.buffers(0) == pool.buffers(2) == k24 and pool.buffers(4) == N_CALLS
        for r in (0, 2, 4):
            assert [m.raw_line() for m in pool.take(r)] == _expect_lines(streams[r], rates[r], pool.buffers(r)), r
        # the strided upload (all buffers of a call in one host block) and the per-buffer upload
        for strided in (True, False):
            for r in range(5):
                pool.reset(r)
                pool.take(r)
            for k in range(N_CALLS):
                bufs = [streams[r][k * BUF: (k + 1) * BUF] for r in range(5)]
                if strided:
                    block = np.stack(bufs)
                    bufs = [block[r] for r in range(5)]
                else:
                    bufs = [np.array(b) for b in bufs[::-1]][::-1]
                pool.ingest(list(range(5)), bufs)
            for r in range(5):
                assert pool.buffers(r) == (k24 if rates[r] == 2_400_000 else N_CALLS)
                assert [m.raw_line() for m in pool.take(r)] == _expect_lines(streams[r], rates[r], pool.buffers(r)), (strided, r)
        # reset keeps the rate; the rate switched 2.4 MS/s -> 2 MHz -> 2.4 MS/s across resets
        pool.reset(1)
        pool.ingest([1], [streams[1][:BUF]])
        with pytest.raises(RuntimeError, match="in progress"):
            pool.set_input_rate(1, 2_000_000)
        pool.reset(1)
        pool.set_input_rate(1, 2_000_000)
        pool.take(1)
        for k in range(3):
            pool.ingest([1], [streams[5][k * BUF: (k + 1) * BUF]])
        assert pool.buffers(1) == 3
        assert [m.raw_line() for m in pool.take(1)] == _expect_lines(streams[5], 2_000_000, 3)
        with pytest.raises(RuntimeError, match="in progress"):
            pool.set_input_rate(1, 2_400_000)
        pool.reset(1)
        pool.set_input_rate(1, 2_400_000)
        for k in range(N_CALLS):
            pool.ingest([1, 6], [streams[1][k * BUF: (k + 1) * BUF], streams[6][k * BUF: (k + 1) * BUF]])
        assert pool.buffers(1) == k24
        assert [m.raw_line() for m in pool.take(1)] == _expect_lines(streams[1], 2_400_000, k24)
