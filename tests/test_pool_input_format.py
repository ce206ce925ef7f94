"""16-bit receivers in the receiver pool (modes_pool_set_input_format): a receiver's call brings
BUFFER_SAMPLES int16 I/Q samples (2 * BUFFER_BYTES bytes), and everything the pool delivers for it equals
what it delivers for a UC8 receiver at the same rate fed the converted bytes (tests/input_format_model.py),
at 2 MHz and at 2.4 MS/s, with UC8 and 16-bit receivers mixed in one call.

CPU tests check the setter's refusals, the buffer sizes ReceiverPool checks, and the host conversion of a
2 MHz receiver's carry.  GPU tests check the conversion launch byte for byte through a device harness
of its own, and the contract through ReceiverPool against the oracle, the single-stream decoder and a UC8
receiver of the same pool."""
import ctypes
import subprocess

import numpy as np
import pytest

import checker as C
import input_format_model as M
import pool_rate_model as PM
import resample_model as RM
from dump1090_b200 import api, synth
from test_pool import _schedule
from test_pool_scale import _banks, _planted, _stream

ROOT = C.ROOT
SHIM = ROOT / "tests" / "_build" / "libpool_carry_host.so"
DSHIM = ROOT / "tests" / "_build" / "libconvert_pool_device.so"
BUF = api.BUFFER_BYTES
B = api.BUFFER_SAMPLES
CARRY = api.CARRY_BYTES
R2, R24 = 2_000_000, 2_400_000
FLAG_SETS = [dict(), dict(aggressive=1), dict(fix=0), dict(check_crc=0)]   # test_pool's four
SCALE = {"sc16": 256.0, "sc16q11": 16.0}          # int16 units per UC8 LSB at full scale
N_CALLS = 5                                       # calls per receiver


def _shift(fmt, shift=None):
    return 0 if fmt == "uc8" else (M.DEFAULT_SHIFT[fmt] if shift is None else shift)


def _noisy16(y, s, seed):
    """UC8 bytes written as int16 that convert back to them at shift s, with random low bits."""
    v = M.to_sc16(y, s).view("<i2").astype(np.int64)
    if s:
        v += np.random.default_rng(seed).integers(0, 1 << s, v.size)
    return v.astype("<i2").view(np.uint8)


# ---------------------------------------------------------------- CPU


def test_setter_refusals_without_a_device():
    with api.ReceiverPool(3, max_batch=2) as pool:
        with pytest.raises(ValueError):
            pool.set_input_format(0, "sc8")
        with pytest.raises(RuntimeError, match="format 3 is not supported"):
            pool._check(api.lib().modes_pool_set_input_format(pool._h, 0, 3, -1))
        with pytest.raises(RuntimeError, match="shift 16 is not supported"):
            pool.set_input_format(0, "sc16", 16)
        with pytest.raises(RuntimeError, match="not supported with UC8"):
            pool.set_input_format(0, "uc8", 3)
        with pytest.raises(RuntimeError, match="out of range"):
            pool.set_input_format(3, "sc16")
        # before any call: accepted, and again; format and rate in either order
        pool.set_input_format(1, "sc16")
        pool.set_input_format(1, "sc16q11", 0)
        pool.set_input_format(1, "uc8", 0)
        pool.set_input_format(1, "uc8")
        pool.set_input_format(1, "sc16", 15)
        pool.set_input_rate(1, R24)
        pool.set_input_rate(2, R24)
        pool.set_input_format(2, "sc16q11")
        pool.set_input_rate(2, R2)
        assert pool._bytes == [BUF, 2 * BUF, 2 * BUF]
    with pytest.raises(ValueError):
        api.ReceiverPool(2, input_format="cs16")
    with pytest.raises(RuntimeError, match="shift 16"):
        api.ReceiverPool(2, input_format="sc16", input_shift=16)
    with api.ReceiverPool(2, input_format="sc16q11", input_shift=2, input_rate=R24) as pool:
        assert pool._bytes == [2 * BUF, 2 * BUF]
        for r in range(2):
            pool.set_input_format(r, "sc16")
    assert "modes_pool_set_input_format" in api.EXPORTS


def test_ingest_checks_buffer_sizes_first():
    """A buffer of the wrong size for its receiver's format is refused before the pool is called: no
    stream starts, so the setters still accept."""
    with api.ReceiverPool(3, max_batch=3) as pool:
        pool.set_input_format(1, "sc16")
        pool.set_input_format(2, "sc16q11")
        one, two = np.zeros(BUF, np.uint8), np.zeros(2 * BUF, np.uint8)
        for ids, bufs in (([0, 1], [one, one]), ([1], [two[:-4]]), ([0, 2], [two, two]), ([2], [np.zeros(BUF // 2, "<i4")])):
            for call in (pool.ingest, pool.submit):
                with pytest.raises(ValueError, match="input format takes"):
                    call(ids, bufs)
        for r, fmt in enumerate(("sc16", "uc8", "sc16")):
            pool.set_input_format(r, fmt)
            pool.set_input_rate(r, R24)


def test_host_carry_conversion_equals_model():
    """The carry of a 2 MHz 16-bit receiver (its last 238 samples, converted on the host) against the
    model, on the last 952 bytes of a buffer: edge shifts, saturating values, values at the half."""
    subprocess.run(["make", "-s", "shim"], cwd=ROOT, check=True)
    lib = ctypes.CDLL(str(SHIM))
    lib.shim_pool_convert_samples.restype = ctypes.c_int
    lib.shim_pool_convert_samples.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_void_p]
    rng = np.random.default_rng(3)
    edge = np.array([-32768, 32767, -32767, 0, -1, 1, 127, -128, 2047, -2048, 16384, -16384], np.int64)
    for s in (0, 1, 4, 8, 15):
        v = rng.integers(-32768, 32768, 2 * B)
        half = (1 << (s - 1)) if s else 0
        v[-2 * (CARRY // 2):][: 4 * edge.size] = np.concatenate([edge, edge + half, edge - half, -edge])[: 4 * edge.size]
        buf = np.clip(v, -32768, 32767).astype("<i2").view(np.uint8)
        assert buf.size == 2 * BUF
        tail = np.ascontiguousarray(buf[-2 * CARRY:])
        out = np.full(CARRY, 0x5A, np.uint8)
        assert lib.shim_pool_convert_samples(tail.ctypes.data, CARRY // 2, s, out.ctypes.data) == 0
        assert np.array_equal(out, M.convert(tail, s)), s
        assert np.array_equal(out, M.convert(buf, s)[-CARRY:]), s
    assert lib.shim_pool_convert_samples(tail.ctypes.data, 1, 16, out.ctypes.data) == -1


# ---------------------------------------------------------------- GPU: the conversion launch


@pytest.fixture(scope="module")
def dshim():
    subprocess.run(["make", "-s", "dshim"], cwd=ROOT, check=True)
    lib = ctypes.CDLL(str(DSHIM))
    lib.cpool_convert.restype = ctypes.c_int
    lib.cpool_convert.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p,
                                  ctypes.c_uint32]
    lib.cpool_error.restype = ctypes.c_char_p
    return lib


CONV_JOB = np.dtype([(f, np.int64) for f in ("in_off", "out_off", "shift")])


@pytest.mark.gpu
def test_convert_pool_kernel_equals_model(dshim):
    """One launch of 260 jobs (more than a full max_batch = 256 call makes) in mixed order over SC16- and
    SC16Q11-scaled buffers with full-scale, saturating and half-way values at shifts 0, 4, 8 and 15, each
    into its own destination between sentinel bytes; no byte outside the destinations changes."""
    rng = np.random.default_rng(17)
    n_in, n_jobs, gap, sentinel = 12, 260, 4096, 0xC3
    bufs = []
    for k in range(n_in):
        lim = 32768 if k % 2 == 0 else 2048
        v = rng.integers(-lim, lim, 2 * B)
        v[rng.integers(0, v.size, 4000)] = -32768
        v[rng.integers(0, v.size, 4000)] = 32767
        for s in (4, 8, 15):                                         # values that round at the half
            idx = rng.integers(0, v.size, 3000)
            v[idx] = (rng.integers(-(32768 >> s), 32768 >> s, idx.size) << s) + (1 << (s - 1))
        bufs.append(np.clip(v, -32768, 32767).astype("<i2").view(np.uint8))
    src = np.concatenate(bufs)
    shifts = (0, 4, 8, 15)
    jobs = np.zeros(n_jobs, CONV_JOB)
    order = rng.permutation(n_jobs)                                  # job i writes destination order[i]
    pitch = BUF + gap
    out = np.full(n_jobs * pitch + gap, sentinel, np.uint8)
    want = {}
    model = {}
    for i in range(n_jobs):
        k, s = int(rng.integers(0, n_in)), shifts[i % 4]
        jobs[i] = (k * 2 * BUF, gap + int(order[i]) * pitch, s)
        if (k, s) not in model:
            model[k, s] = M.convert(bufs[k], s)
        want[int(order[i])] = model[k, s]
    got = out.copy()
    rc = dshim.cpool_convert(src.ctypes.data, src.size, got.ctypes.data, got.size, jobs.ctypes.data, n_jobs)
    assert rc == 0, dshim.cpool_error().decode()
    for d in range(n_jobs):
        o = gap + d * pitch
        assert (got[o - gap: o] == sentinel).all(), d
        bad = np.flatnonzero(got[o: o + BUF] != want[d])
        assert bad.size == 0, (d, bad[:5])
    assert (got[-gap:] == sentinel).all()
    assert {0, 255} <= set(np.unique(model[0, 0]).tolist())          # saturation reached both ends


# ---------------------------------------------------------------- GPU: the contract


def _fleet16(fmt, rate, seed, snr, shift=None, n_calls=N_CALLS):
    """A synthetic fleet as the receiver's 16-bit bytes (n_calls buffers) at a scale its shift resolves."""
    s = _shift(fmt, shift)
    nframes = -(-n_calls * B * R2 // rate // 400) + 2
    x = synth.fleet_at_rate(snr, nframes, seed, sample_rate=rate, dtype="sc16", scale=float(1 << s))[0]
    assert x.size >= n_calls * 2 * BUF
    return np.ascontiguousarray(x[: n_calls * 2 * BUF])


def _fleet8(rate, seed, snr, n_calls=N_CALLS):
    nframes = -(-n_calls * B * R2 // rate // 400) + 2
    x = synth.fleet_at_rate(snr, nframes, seed, sample_rate=rate)[0]
    return np.ascontiguousarray(x[: n_calls * BUF])


class Rx:
    """A pool receiver: its format, shift (None: default), rate and input bytes."""

    def __init__(self, fmt, rate, x, shift=None):
        self.fmt, self.rate, self.x, self.shift = fmt, rate, x, shift
        self.size = BUF if fmt == "uc8" else 2 * BUF

    def buf(self, k):
        return self.x[k * self.size: (k + 1) * self.size]

    def uc8(self):
        """The bytes the receiver decodes as a UC8 receiver at its rate."""
        return self.x if self.fmt == "uc8" else M.convert(self.x, _shift(self.fmt, self.shift))

    def decoded(self, k):
        """The 2 MHz bytes of its first k decoded buffers."""
        y = self.uc8()
        return RM.resample_range(y, 0, k * B) if self.rate == R24 else y[: k * BUF]


def _mixed():
    """UC8 at both rates, SC16 and SC16Q11 at both rates, and SC16Q11 at shift 2, all with real frames."""
    return [Rx("uc8", R2, synth.random_traffic(N_CALLS * B, 120 * N_CALLS + 37, seed=101)),
            Rx("uc8", R24, _fleet8(R24, 31, 20)),
            Rx("sc16", R2, _fleet16("sc16", R2, 41, 14)),
            Rx("sc16q11", R2, _fleet16("sc16q11", R2, 42, 20)),
            Rx("sc16", R24, _fleet16("sc16", R24, 43, 20)),
            Rx("sc16q11", R24, _fleet16("sc16q11", R24, 44, 14)),
            Rx("sc16q11", R2, _fleet16("sc16q11", R2, 45, 10, shift=2), shift=2)]


def _pool(rxs, **kw):
    pool = api.ReceiverPool(len(rxs), **kw)
    for r, rx in enumerate(rxs):
        pool.set_input_rate(r, rx.rate)
        pool.set_input_format(r, rx.fmt, rx.shift)
    return pool


def _run_schedule(pool, rxs, schedule, max_batch):
    nxt = [0] * len(rxs)
    for ids in schedule:
        for lo in range(0, len(ids), max_batch):
            part = ids[lo: lo + max_batch]
            pool.ingest(part, [rxs[r].buf(nxt[r]) for r in part])
            for r in part:
                nxt[r] += 1


def _want_buffers(rate, n_calls=N_CALLS):
    return PM.ready_buffers(n_calls * B) if rate == R24 else n_calls          # B input samples a call


def _same(got, want, what):
    assert len(got) == len(want), (what, len(got), len(want))
    for k, (g, w) in enumerate(zip(got, want)):
        assert bytes(g) == bytes(w), (what, k, g.raw_line(), w.raw_line())


def _single(factory, rx, **kw):
    return factory(input_format=rx.fmt, input_shift=rx.shift, input_rate=rx.rate, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("kw", FLAG_SETS, ids=lambda k: "-".join(f"{a}{b}" for a, b in k.items()) or "default")
def test_mixed_pool_equals_oracle(kw, checker_libs, gpu_decoder_factory):
    rxs = _mixed()
    cfg = dict(fix_errors=kw.get("fix", 1), aggressive=kw.get("aggressive", 0), check_crc=kw.get("check_crc", 1))
    with _pool(rxs, max_batch=4, **cfg) as pool:
        _run_schedule(pool, rxs, _schedule(len(rxs), N_CALLS, seed=6), 4)
        for r, rx in enumerate(rxs):
            k = pool.buffers(r)
            assert k == _want_buffers(rx.rate), r
            msgs, stats = C.oracle_decode(rx.decoded(k), drop_eof=1, **kw)
            got = pool.take(r)
            assert [m.raw_line() for m in got] == [m.hexline() for m in msgs], f"receiver {r}"
            assert [C.msg_fields(m, with_pos=True) for m in got] == [C.msg_fields(m, with_pos=True) for m in msgs], r
            assert list(pool.stats(r).values()) == stats, f"receiver {r}"
            if rx.fmt != "uc8":
                assert len(got) > 20, (r, len(got))                    # 16-bit receivers carry real frames
            dec = _single(gpu_decoder_factory, rx, **cfg)
            dec.process(rx.x)
            _same(got, dec.take_messages(), ("single stream", r))
            assert dec.stats() == pool.stats(r), r


@pytest.mark.gpu
def test_16bit_receiver_equals_uc8_receiver():
    """In one pool and the same calls, a 16-bit receiver and a UC8 receiver fed its converted bytes
    deliver the same messages and statistics, at both rates."""
    base = [Rx("sc16", R2, _fleet16("sc16", R2, 51, 12)),
            Rx("sc16q11", R24, _fleet16("sc16q11", R24, 52, 12)),
            Rx("sc16q11", R2, _noisy16(synth.random_traffic(N_CALLS * B, 700, seed=53), 3, 54), shift=3),
            Rx("sc16", R24, _fleet16("sc16", R24, 55, 16, shift=6), shift=6)]
    rxs = base + [Rx("uc8", rx.rate, rx.uc8()) for rx in base]
    n = len(base)
    sched = [ids + [r + n for r in ids] for ids in _schedule(n, N_CALLS, seed=8)]
    with _pool(rxs, max_batch=2 * n, signal=True) as pool:
        _run_schedule(pool, rxs, sched, 2 * n)
        for r in range(n):
            assert pool.buffers(r) == pool.buffers(r + n) == _want_buffers(base[r].rate)
            got, want = pool.take(r), pool.take(r + n)
            assert got, r
            _same(got, want, r)
            assert pool.stats(r) == pool.stats(r + n), r


SWITCHES = [dict(signal=True), dict(arrival=True, signal=True), dict(levels=True), dict(recover=True),
            dict(recover=True, weak_preambles=True)]


@pytest.mark.gpu
@pytest.mark.parametrize("sw", SWITCHES, ids=["signal", "arrival", "levels", "recover", "weak"])
def test_every_switch_equals_single_stream(sw, gpu_decoder_factory):
    rxs = _mixed()
    with _pool(rxs, max_batch=5, **sw) as pool:
        _run_schedule(pool, rxs, _schedule(len(rxs), N_CALLS, seed=10), 5)
        for r, rx in enumerate(rxs):
            dec = _single(gpu_decoder_factory, rx, **sw)
            dec.process(rx.x)                                        # every complete buffer, no EOF buffer
            got = pool.take(r)
            _same(got, dec.take_messages(), (sw, r))
            assert pool.stats(r) == dec.stats(), (sw, r)
            if sw.get("signal") and rx.fmt != "uc8":
                assert any(m.signal for m in got), r
            if sw.get("arrival") and rx.fmt != "uc8":
                assert any(m.arrival for m in got), r
            if sw.get("levels"):
                lv = pool.take_levels(r)
                assert list(lv["buffer"]) == list(range(pool.buffers(r))), r
                assert np.array_equal(lv, dec.take_levels()), r
            if sw.get("recover"):
                assert pool.recovery_stats(r) == dec.recovery_stats(), r
                assert pool.weak_recovery_stats(r) == dec.weak_recovery_stats(), r


def _lines(rx, k):
    return [m.hexline() for m in C.oracle_decode(rx.decoded(k), drop_eof=1)[0]]


@pytest.mark.gpu
def test_ingest_shapes(checker_libs):
    rxs = _mixed()
    n = len(rxs)
    with _pool(rxs, max_batch=5) as pool:
        # the first call of a 2.4 MS/s SC16 receiver completes nothing; the collect still pairs with it
        pool.ingest([4], [rxs[4].buf(0)])
        assert pool.buffers(4) == 0 and pool.take(4) == []
        with pytest.raises(RuntimeError, match="in progress"):
            pool.set_input_format(4, "sc16q11")
        pool.set_input_format(3, "sc16q11")                          # not named yet: no stream in progress
    with _pool(rxs, max_batch=5) as pool:
        # two batches in flight, 16-bit receivers of both rates in both, beside UC8 ones
        nxt = [0] * n

        def submit(ids):
            pool.submit(ids, [rxs[r].buf(nxt[r]) for r in ids])
            for r in ids:
                nxt[r] += 1

        submit([4, 2, 0])
        for k in range(1, N_CALLS):
            submit([2, 5, 4, 1] if k % 2 else [5, 4, 2, 0, 1])
            pool.collect()
        submit([5, 1, 0])
        pool.collect()
        pool.collect()
        with pytest.raises(RuntimeError, match="no batch in flight"):
            pool.collect()
        for r in (0, 1, 2, 4, 5):
            assert nxt[r] >= 4 and pool.buffers(r) == _want_buffers(rxs[r].rate, nxt[r]), r
            assert [m.raw_line() for m in pool.take(r)] == _lines(rxs[r], pool.buffers(r)), r
        # a mixed call's uploads: all buffers in one host block at a 512 KiB pitch (UC8 ones in the first
        # half of their row: both groups strided), one block per format group, and one copy per buffer
        for shape in ("pitch", "groups", "single"):
            for r in range(n):
                pool.reset(r)
                pool.take(r)
            order = [3, 0, 4, 1, 6, 5, 2]
            for k in range(N_CALLS):
                bufs = [rxs[r].buf(k) for r in order]
                if shape == "pitch":
                    block = np.zeros((n, 2 * BUF), np.uint8)
                    for i, b in enumerate(bufs):
                        block[i, : b.size] = b
                    bufs = [block[i, : b.size] for i, b in enumerate(bufs)]
                elif shape == "groups":
                    b8 = np.stack([b for b in bufs if b.size == BUF])
                    b16 = np.stack([b for b in bufs if b.size == 2 * BUF])
                    it8, it16 = iter(range(len(b8))), iter(range(len(b16)))
                    bufs = [b8[next(it8)] if b.size == BUF else b16[next(it16)] for b in bufs]
                else:
                    bufs = [np.array(b) for b in bufs[::-1]][::-1]
                for lo in range(0, n, 5):
                    pool.ingest(order[lo: lo + 5], bufs[lo: lo + 5])
            for r in range(n):
                assert pool.buffers(r) == _want_buffers(rxs[r].rate), (shape, r)
                assert [m.raw_line() for m in pool.take(r)] == _lines(rxs[r], pool.buffers(r)), (shape, r)
        # reset keeps the format; UC8 -> SC16 -> SC16Q11 -> UC8 across resets, refused in between
        u8, s16 = rxs[0], Rx("sc16", R2, _noisy16(rxs[0].x, 8, 61))
        s11 = Rx("sc16q11", R2, _noisy16(rxs[0].x, 4, 62))
        pool.reset(0)
        pool.take(0)
        for rx in (u8, s16, s11, u8):
            pool.reset(0)
            pool.set_input_format(0, rx.fmt)
            for k in range(3):
                pool.ingest([0], [rx.buf(k)])
                with pytest.raises(RuntimeError, match="in progress"):
                    pool.set_input_format(0, "sc16" if rx.fmt == "uc8" else "uc8")
            assert pool.buffers(0) == 3
            assert [m.raw_line() for m in pool.take(0)] == _lines(u8, 3), rx.fmt
            with pytest.raises(ValueError):
                pool.ingest([0], [s16.buf(0) if rx.fmt == "uc8" else u8.buf(0)])
            pool.reset(0)                                            # reset keeps the format
            pool.ingest([0], [rx.buf(0)])
            assert pool.buffers(0) == 1
            assert [m.raw_line() for m in pool.take(0)] == _lines(u8, 1), rx.fmt


@pytest.mark.gpu
def test_modes1_through_the_pool(checker_libs):
    """modes1 written as SC16 and as SC16Q11 at each format's default shift, fed in whole buffers to 2 MHz
    receivers, gives the reference's lines of those buffers without the EOF buffer."""
    y = C.modes1()
    k = y.size // BUF
    want = [m.hexline() for m in C.oracle_decode(y[: k * BUF], drop_eof=1)[0]]
    assert k == 1 and len(want) == 119
    with api.ReceiverPool(2) as pool:
        for r, fmt in enumerate(("sc16", "sc16q11")):
            pool.set_input_format(r, fmt)
        x = [M.to_sc16(y, M.DEFAULT_SHIFT[f]) for f in ("sc16", "sc16q11")]
        for j in range(k):
            pool.ingest([1, 0], [x[1][j * 2 * BUF: (j + 1) * 2 * BUF], x[0][j * 2 * BUF: (j + 1) * 2 * BUF]])
        for r in range(2):
            assert [m.raw_line() for m in pool.take(r)] == want, r


# ---------------------------------------------------------------- GPU: at full batch size

FULL_RX = 256
KINDS = [("uc8", R2), ("sc16", R2), ("uc8", R24), ("sc16q11", R24), ("sc16q11", R2), ("sc16", R24)]
FULL_CALLS = 4


@pytest.fixture(scope="module")
def full_world():
    """test_pool_scale's streams with their planted frames, each receiver at one of the six format and rate
    combinations (16-bit ones written so that they convert back to the UC8 stream), and the calls: every
    receiver at once first, then random subsets in mixed order."""
    banks = _banks(with_24=True)
    rxs, plants = [], []
    for r in range(FULL_RX):
        fmt, rate = KINDS[r % len(KINDS)]
        s, p = _stream(r, FULL_CALLS, rate, banks)
        rxs.append(Rx(fmt, rate, s if fmt == "uc8" else _noisy16(s, M.DEFAULT_SHIFT[fmt], 7000 + r)))
        plants.append(p)
    rng = np.random.default_rng(33)
    calls = [list(rng.permutation(FULL_RX))]
    left = [FULL_CALLS - 1] * FULL_RX
    while any(left):
        ids = [r for r in rng.permutation(FULL_RX) if left[r] and rng.random() < 0.6]
        for r in ids:
            left[r] -= 1
        if ids:
            calls.append([int(r) for r in ids])
    return dict(rxs=rxs, plants=plants, calls=calls, every={f for p in plants for _, f in p})


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["ingest", "pipelined"])
def test_full_batch_equals_single_stream(mode, full_world, gpu_decoder_factory):
    rxs, calls = full_world["rxs"], full_world["calls"]
    nxt = [0] * FULL_RX
    with _pool(rxs, max_batch=FULL_RX) as pool:
        pending = 0
        for ci, ids in enumerate(calls):
            bufs = [rxs[r].buf(nxt[r]) for r in ids]
            if ci % 2 == 0:                                          # one host block at a 512 KiB pitch
                block = np.zeros((len(ids), 2 * BUF), np.uint8)
                for i, b in enumerate(bufs):
                    block[i, : b.size] = b
                bufs = [block[i, : b.size] for i, b in enumerate(bufs)]
            for r in ids:
                nxt[r] += 1
            if mode == "ingest":
                pool.ingest(ids, bufs)
                continue
            pool.submit(ids, bufs)
            pending += 1
            if pending == 2:
                pool.collect()
                pending -= 1
        for _ in range(pending):
            pool.collect()
        decs = {}
        n_msgs = 0
        for r, rx in enumerate(rxs):
            key = (rx.fmt, rx.rate)
            if key not in decs:
                decs[key] = _single(gpu_decoder_factory, rx)
            dec = decs[key]
            dec.reset()
            dec.process(rx.x)
            k = pool.buffers(r)
            assert k == _want_buffers(rx.rate, FULL_CALLS), r
            got = pool.take(r)
            _same(got, dec.take_messages(), (mode, r))
            assert pool.stats(r) == dec.stats(), (mode, r)
            _planted(got, full_world["plants"][r], k, full_world["every"])
            n_msgs += len(got)
    print(f"\npool formats at {FULL_RX}: {len(calls)} calls, named {[len(c) for c in calls]}, {n_msgs} messages")
