"""4-10 MS/s captures tuned off 1090 MHz (modes_set_input_offset, modes_resample_device_shift): an exact
frequency shift in front of the integer decimator.

The contract: decoding a 2 M MS/s stream with input offset o gives exactly what the 2 MHz decoder gives on the
bytes tests/shift_model.py makes from it (a 16-bit stream converted first, tests/input_format_model.py).  At
offset 0 they are the decimator's bytes (tests/decimate_model.py).  CPU tests check the tables, the step and
phase arithmetic and the rate rules (host build of modes_resample_core.cuh against the model), and that a
frame sent off centre and shifted back decodes through the oracle; GPU tests check the kernel byte for byte
and the contract on every decode path."""
import ctypes
import subprocess

import numpy as np
import pytest

import checker as C
import decimate_model as DM
import input_format_model as IF
import shift_model as SM
from dump1090_b200 import api, synth

ROOT = C.ROOT
SHIM = ROOT / "tests" / "_build" / "libshift_core_host.so"
BUF = api.BUFFER_BYTES
B = api.BUFFER_SAMPLES
NO_LIMIT = 2 ** 63 - 1
MS = (2, 3, 4, 5)
FORMATS = {"uc8": (-1, 1.0), "sc16": (8, 256.0), "sc16q11": (4, 16.0)}      # default shift, synth scale
FLAGS = [(0, 0, 0), (0, 0, 1), (1, 0, 1), (1, 1, 1)]                         # fix_errors, aggressive, check_crc


def odd(m: int) -> int:
    """An offset in range at 2 M MS/s that is no round number of Hz."""
    return 1_234_567 if m > 2 else 765_433


def offsets(m: int) -> list:
    mx = (m - 1) * 1_000_000
    return sorted({mx, -mx, 1_000_000, -1_000_000, odd(m), 0}, key=lambda o: (abs(o), o))


# ---------------------------------------------------------------- CPU: arithmetic


@pytest.fixture(scope="module")
def shim():
    subprocess.run(["make", "-s", "shim"], cwd=ROOT, check=True)
    lib = ctypes.CDLL(str(SHIM))
    lib.shim_shift_decimate.restype = ctypes.c_int
    lib.shim_shift_decimate.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int64, ctypes.c_int64,
                                        ctypes.c_size_t, ctypes.c_int64, ctypes.c_int, ctypes.c_uint32, ctypes.c_void_p]
    lib.shim_shift_tables.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    lib.shim_shift_step.restype = ctypes.c_uint32
    lib.shim_shift_step.argtypes = [ctypes.c_int32, ctypes.c_uint32]
    lib.shim_shift_max_offset.restype = ctypes.c_int32
    lib.shim_shift_max_offset.argtypes = [ctypes.c_uint32, ctypes.c_int32, ctypes.c_void_p]
    return lib


def _shim_range(shim, m, offset, span, in_first, out_first, count, limit=NO_LIMIT, shift=-1):
    span = np.ascontiguousarray(span, dtype=np.uint8)
    out = np.zeros(2 * count, dtype=np.uint8)
    st = SM.step(offset, 2_000_000 * m)
    assert shim.shim_shift_decimate(m, span.ctypes.data if span.size else None, span.size, in_first, out_first, count,
                                    limit, shift, st, out.ctypes.data) == 0
    return out


def test_tables_are_the_derivation(shim):
    c = np.zeros(1024, np.int16)
    s = np.zeros(1024, np.int16)
    shim.shim_shift_tables(c.ctypes.data, s.ctypes.data)
    assert np.array_equal(c, SM.C) and np.array_equal(s, SM.S)
    a = 2 * np.pi * np.arange(1024) / 1024
    assert np.abs(c - 16384 * np.cos(a)).max() <= 0.5 and np.abs(s - 16384 * np.sin(a)).max() <= 0.5
    assert (np.abs(SM.C) + np.abs(SM.S)).max() == 23170                  # the bound on |u| (<= 182)


def test_step_phase_and_rates(shim):
    fits = ctypes.c_int32()
    for hz, m in DM.RATES.items():
        mx = (m - 1) * 1_000_000
        assert shim.shim_shift_max_offset(hz, 0, ctypes.byref(fits)) == mx == SM.max_offset(hz) and fits.value == 1
        for o in (mx, -mx, 1, -1, odd(m), -odd(m)):
            assert shim.shim_shift_max_offset(hz, o, ctypes.byref(fits)) == mx and fits.value == 1, (hz, o)
        for o in (mx + 1, -mx - 1, 2 ** 31 - 1, -2 ** 31):
            assert shim.shim_shift_max_offset(hz, o, ctypes.byref(fits)) == mx and fits.value == 0, (hz, o)
        for o in (mx, -mx, 0, 1, -1, 999_999, odd(m), -odd(m), 3_141_593, -4_000_000, 4_000_000):
            assert shim.shim_shift_step(o, hz) == SM.step(o, hz), (hz, o)
            if abs(o) <= mx:
                assert abs(SM.applied_hz(o, hz) - o) < 0.002, (hz, o)
    for hz in (2_000_000, 2_400_000):                                       # no bandwidth to shift into
        assert shim.shim_shift_max_offset(hz, 0, ctypes.byref(fits)) == 0 and fits.value == 1
        for o in (1, -1, 1_000_000):
            assert shim.shim_shift_max_offset(hz, o, ctypes.byref(fits)) == 0 and fits.value == 0, (hz, o)
    assert shim.shim_shift_max_offset(3_000_000, 0, ctypes.byref(fits)) == -1
    assert np.array_equal(SM.phases(2 ** 32 - 3, 7, 5 << 22), [(5 * x) % 1024 for x in range(-3, 4)])


def _windows(rng, m):
    yield "random", rng.integers(0, 256, 2 * 3000 * m + 1, dtype=np.uint8)
    for v in (0, 255):                                                     # xi, xq at their extremes
        yield f"const{v}", np.full(2 * 1500 * m, v, np.uint8)
    ext = rng.choice(np.array([0, 255], np.uint8), 2 * 1500 * m)
    yield "extremes", ext
    yield "mixed", np.stack([ext[0::2], 255 - ext[1::2]], 1).reshape(-1)


@pytest.mark.parametrize("m", MS)
def test_host_build_equals_model(shim, m):
    """Random and extreme UC8 and converted-int16 windows, at offsets of both signs, every one of the 1024
    phases met, output ranges before the stream start, past 2^32 and 2^33 input samples, with the EOF limit."""
    rng = np.random.default_rng(40 + m)
    hz = 2_000_000 * m
    x16 = rng.integers(-2 ** 15, 2 ** 15, 2 * 3000 * m, dtype=np.int64).astype("<i2").view(np.uint8)
    seen = set()
    for name, x in _windows(rng, m):
        for o in offsets(m) + [-odd(m), 7, -313_373]:
            for base in (0, 2 ** 32 // m - 700, 2 ** 32 // m + 9, 2 ** 33 // m - 3, 2 ** 33 // m + 1):
                for first, count in [(-240, 240), (-7, 50), (13, 1003), (2500, 400)] + [(0, 2900)] * (base == 0):
                    o0 = base + first
                    lo, hi = DM.input_span(o0, count, m)
                    b0 = m * base
                    want = SM.shift_decimate_range(x, m, o, o0, count, in_first=b0)
                    slo = max(lo, b0)
                    got = _shim_range(shim, m, o, x[2 * (slo - b0): 2 * (hi - b0)], slo, o0, count)
                    assert np.array_equal(got, want), (m, name, o, base, first)
                    seen.update(SM.phases(slo, hi - slo, SM.step(o, hz)).tolist())
                if name == "random":                                        # int16 at two shifts, the limit
                    for shift in (8, 4):
                        conv = IF.convert(x16, shift)
                        want = SM.shift_decimate_range(conv, m, o, base - 5, 1200, in_first=m * base)
                        got = _shim_range(shim, m, o, x16, m * base, base - 5, 1200, shift=shift)
                        assert np.array_equal(got, want), (m, o, base, shift)
                    lim = base + 17
                    assert np.array_equal(_shim_range(shim, m, o, x, m * base, base, 100, lim),
                                          SM.shift_decimate_range(x, m, o, base, 100, limit=lim, in_first=m * base))
    assert seen == set(range(1024)), len(seen)


@pytest.mark.parametrize("m", MS)
def test_offset_zero_is_the_decimator(shim, m):
    rng = np.random.default_rng(m)
    x = rng.integers(0, 256, 2 * 2000 * m + 1, dtype=np.uint8)
    want = DM.decimate(x, m)
    assert np.array_equal(SM.shift_decimate(x, m, 0), want)
    assert np.array_equal(_shim_range(shim, m, 0, x, 0, 0, want.size // 2), want)


def test_carrier_and_dc_are_opt_in():
    frames = [(100, synth.make_frame(17, 5, bytes(range(10))), 30.0, 1.0, 0.25)]
    base = synth.synth_stream_at(2000, frames, sigma=2.0, seed=3, sample_rate=8_000_000)
    assert np.array_equal(synth.synth_stream_at(2000, frames, sigma=2.0, seed=3, sample_rate=8_000_000, carrier_hz=0,
                                                dc=None), base)
    a, t = synth.fleet_at_rate(15, 20, 1, sample_rate=8_000_000)
    b, u = synth.fleet_at_rate(15, 20, 1, sample_rate=8_000_000, carrier_hz=0.0, dc=None)
    assert np.array_equal(a, b) and t == u
    moved = synth.synth_stream_at(2000, frames, sigma=2.0, seed=3, sample_rate=8_000_000, carrier_hz=2e6)
    assert not np.array_equal(moved, base)
    d = synth.synth_stream_at(2000, frames, sigma=0.0, seed=3, sample_rate=8_000_000, dc=(10.0, -5.0)).astype(int)
    assert d[0] == 137 and d[1] == 122


def _df17(msgs, truth):
    got = [bytes(x.msg[:14]).hex() for x in msgs if x.msgtype == 17 and x.msgbits == 112]
    true = sum(1 for h in got if h in truth)
    return true, len(got) - true


@pytest.mark.parametrize("m", (4, 5))
def test_shift_back_recovers_off_centre_frames(checker_libs, m):
    """A fleet sent 2 MHz off centre decodes to almost nothing unshifted, and shifted back decodes like the
    same fleet sent at the centre, with no false frames."""
    hz = 2_000_000 * m
    snr = 18 - 10 * np.log10(m)
    x0, truth = synth.fleet_at_rate(snr, 200, 2, sample_rate=hz)
    x2, truth2 = synth.fleet_at_rate(snr, 200, 2, sample_rate=hz, carrier_hz=2e6)
    assert truth == truth2
    centred = _df17(C.oracle_decode(DM.decimate(x0, m))[0], truth)
    off = _df17(C.oracle_decode(DM.decimate(x2, m))[0], truth)
    back = _df17(C.oracle_decode(SM.shift_decimate(x2, m, 2_000_000))[0], truth)
    assert centred[1] == off[1] == back[1] == 0
    assert off[0] < 0.1 * centred[0] and back[0] >= 0.95 * centred[0] > 100, (centred, off, back)


# ---------------------------------------------------------------- GPU

_inputs = {}


def traffic_off(m: int, fmt: str, carrier: float, n_samples: int | None = None, seed: int = 3) -> np.ndarray:
    """Random traffic at 2 M MS/s sent at `carrier` Hz off centre, with a DC spike, in the format: by default
    300 000 output samples, so that the EOF buffer is not the whole stream."""
    n_samples = 300_000 * m if n_samples is None else n_samples
    key = (m, fmt, carrier, n_samples, seed)
    if key not in _inputs:
        _, truth = synth.random_traffic(n_samples // m, max(50, n_samples // (1000 * m)), seed, return_truth=True)
        rng = synth.Counter(seed + 1000)
        frames = []
        for pos, frame, flips in truth:
            amp = 12.0 + 98.0 * rng.uniform()
            frac = 0.15 + 0.7 * rng.uniform() if rng.below(2) else 0.0
            frames.append((pos, synth.flip_bits(frame, flips), amp, 2 * np.pi * rng.uniform(), frac))
        _inputs[key] = synth.synth_stream_at(n_samples, frames, sigma=1.5 * np.sqrt(m), seed=seed,
                                             sample_rate=2_000_000 * m, dtype="uc8" if fmt == "uc8" else "sc16",
                                             scale=FORMATS[fmt][1], carrier_hz=carrier, dc=(9.0, -6.0))
    return _inputs[key]


def shifted(x, m, fmt, offset) -> np.ndarray:
    return SM.shift_decimate(x if fmt == "uc8" else IF.convert(x, FORMATS[fmt][0]), m, offset)


def fields(x) -> tuple:
    return tuple(bytes(getattr(x, f)) if f in ("msg", "flight", "pad1") else getattr(x, f) for f, _ in api.Message._fields_)


def assert_same(got, want, what):
    assert len(got) == len(want), (what, len(got), len(want))
    for k, (g, w) in enumerate(zip(got, want)):
        assert fields(g) == fields(w), (what, k, g.raw_line(), w.raw_line(), g.sample_pos, w.sample_pos)


def _dec(m, fmt, offset, **kw):
    return api.Decoder(input_rate=2_000_000 * m, input_format=fmt, input_offset=offset, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("m", MS)
def test_resample_device_shift_equals_model(m):
    """The stage entry byte for byte against the model at every offset, on spans anywhere in the stream
    (past 2^32 input samples, where theta wraps), with and without the carry block; offset 0 is _at."""
    import torch
    rng = np.random.default_rng(80 + m)
    hz = 2_000_000 * m
    x = np.concatenate([traffic_off(m, "uc8", 1e6, 2 * B * m), rng.integers(0, 256, 1001, dtype=np.uint8)])
    n_total = DM.n_out((x.size + 1) // 2, m)
    with api.Decoder() as dec:
        d_x = torch.from_numpy(x).cuda()
        for o in offsets(m):
            for first, nb, base in [(0, 1, 0), (1, 1, 0), (0, 3, 0), (1, 1, 2 ** 32 // (m * B) + 1),
                                    (0, 2, 2 ** 33 // (m * B))]:
                out = torch.zeros(nb * BUF, dtype=torch.uint8, device="cuda")
                o0 = first * B
                lo, hi = DM.input_span(o0 - 240, nb * B + 240, m)
                lo = max(lo, 0)
                hi = min(hi, (x.size + 1) // 2)
                span = torch.zeros(2 * (hi - lo) + 16, dtype=torch.uint8, device="cuda")
                span[: min(2 * hi, x.size) - 2 * lo] = d_x[2 * lo: 2 * hi]
                sb = base * B                                           # the stream moved m sb input samples later
                carry = dec.resample_device_shift(hz, o, span.data_ptr(), min(2 * hi, x.size) - 2 * lo, lo + m * sb,
                                                  first + base, nb, out.data_ptr(), out_end=n_total + sb)
                want = SM.shift_decimate_range(x, m, o, o0 - 238 + sb, nb * B + 238, limit=n_total + sb, in_first=m * sb)
                assert carry == want[:476].tobytes(), (m, o, first, nb, base)
                got = out.cpu().numpy()
                assert np.array_equal(got, want[476:]), (m, o, first, nb, base, np.flatnonzero(got != want[476:])[:5])
        out = torch.zeros(2 * BUF, dtype=torch.uint8, device="cuda")
        o = (m - 1) * 1_000_000
        launches = dec.launch_count()
        assert dec.resample_device_shift(hz, o, d_x.data_ptr(), x.size, 0, 1, 2, out.data_ptr(), want_carry=False) is None
        torch.cuda.synchronize()
        assert dec.launch_count() - launches == 1
        assert np.array_equal(out.cpu().numpy(), SM.shift_decimate_range(x, m, o, B, 2 * B))
        a = dec.resample_device_shift(hz, 0, d_x.data_ptr(), x.size, 0, 1, 1, out.data_ptr())
        b = dec.resample_device_at(hz, d_x.data_ptr(), x.size, 0, 1, 1, out.data_ptr() + BUF)
        torch.cuda.synchronize()
        assert a == b and torch.equal(out[:BUF], out[BUF:])
        for bad in (o + 1, -o - 1):
            with pytest.raises(RuntimeError, match="not supported"):
                dec.resample_device_shift(hz, bad, d_x.data_ptr(), 100, 0, 0, 1, out.data_ptr())
        with pytest.raises(RuntimeError, match="not supported"):
            dec.resample_device_shift(2_400_000, 1, d_x.data_ptr(), 100, 0, 0, 1, out.data_ptr())


def _oracle_check(y, want, want_st, fix, aggressive, check_crc, drop, what):
    ora, ora_st = C.oracle_decode(y, fix=fix, aggressive=aggressive, check_crc=check_crc, drop_eof=drop)
    assert [x.raw_line() for x in want] == [x.hexline() for x in ora], what
    assert [x.sample_pos for x in want] == [x.sample_pos for x in ora], what
    assert list(want_st.values()) == ora_st, what


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", list(FORMATS))
@pytest.mark.parametrize("m", MS)
def test_contract(checker_libs, m, fmt):
    """Decoder(input_rate=2 M MHz, input_format=fmt, input_offset=o) on X == Decoder() on the model's bytes
    == the oracle on them, at every offset, under four flag sets and both EOF outcomes."""
    for o in offsets(m):
        x = traffic_off(m, fmt, o if o else 1.5e6)
        y = shifted(x, m, fmt, o)
        for fix, aggressive, check_crc in FLAGS:
            cfg = dict(fix_errors=fix, aggressive=aggressive, check_crc=check_crc)
            for drop in (0, 1):
                with _dec(m, fmt, o, drop_eof_buffer=drop, **cfg) as dm, api.Decoder(drop_eof_buffer=drop, **cfg) as d2:
                    want = d2.decode(y)
                    want_st = d2.stats()
                    _oracle_check(y, want, want_st, fix, aggressive, check_crc, drop, (m, fmt, o))
                    got = dm.decode(x, chunk=100003 if drop else None)
                    assert_same(got, want, (m, fmt, o, fix, aggressive, check_crc, drop))
                    assert dm.stats() == want_st, (m, fmt, o, drop)
                    if o and (fix, aggressive, check_crc, drop) == (1, 0, 1, 0):
                        assert len(want) > 20, (m, fmt, o)


SWITCHES = [dict(signal=True), dict(arrival=True, signal=True), dict(levels=True), dict(levels=True, drop_eof_buffer=1),
            dict(recover=True), dict(recover=True, weak_preambles=True), dict(gpu_resolve=1)]


@pytest.mark.gpu
@pytest.mark.parametrize("m,fmt,o", [(2, "uc8", 1_000_000), (3, "sc16q11", -2_000_000), (4, "uc8", 1_234_567),
                                     (5, "sc16", -4_000_000)])
def test_contract_with_switches(m, fmt, o):
    x = traffic_off(m, fmt, o)
    y = shifted(x, m, fmt, o)
    for kw in SWITCHES:
        with _dec(m, fmt, o, **kw) as dm, api.Decoder(**kw) as d2:
            want = d2.decode(y)
            got = dm.decode(x, chunk=100003)
            assert_same(got, want, (m, fmt, o, kw))
            assert dm.stats() == d2.stats(), (m, fmt, o, kw)
            if kw.get("levels"):
                assert np.array_equal(dm.take_levels(), d2.take_levels()), (m, fmt, o, kw)
            if kw.get("recover"):
                assert dm.recovery_stats() == d2.recovery_stats(), (m, fmt, o, kw)
                assert dm.weak_recovery_stats() == d2.weak_recovery_stats(), (m, fmt, o, kw)
            if kw.get("arrival"):
                assert any(x.arrival for x in want)


@pytest.mark.gpu
@pytest.mark.parametrize("m,fmt", [(2, "uc8"), (5, "sc16")])
def test_gpus_chunks_and_offset_zero(m, fmt):
    """Two GPUs with one-buffer batches, random odd call sizes, and offset 0 against no offset at all: the
    same messages and the same launches."""
    o = -(m - 1) * 1_000_000
    x = traffic_off(m, fmt, o, 3 * m * B + 4321, 5)
    y = shifted(x, m, fmt, o)
    with api.Decoder() as d2:
        want = d2.decode(y)
    kw = dict(n_gpus=2, max_batch_bytes=BUF, levels=True, recover=True)
    with _dec(m, fmt, o, **kw) as dm, api.Decoder(**kw) as d2:
        assert_same(dm.decode(x), d2.decode(y), (m, fmt, "n_gpus"))
        assert np.array_equal(dm.take_levels(), d2.take_levels()) and dm.recovery_stats() == d2.recovery_stats()
    with _dec(m, fmt, o, max_batch_bytes=2 * BUF) as dm:
        rng = np.random.default_rng(3)
        dm.reset()
        off = 0
        while off < x.size:
            n = 2 * int(rng.integers(1, 400_000)) + 1
            dm.process(x[off: off + n])
            off += n
        dm.finish()
        assert_same(dm.take_messages(), want, (m, fmt, "random calls"))
    runs = []
    for kw in ({}, dict(input_offset=0)):
        with api.Decoder(input_rate=2_000_000 * m, input_format=fmt, n_gpus=2, max_batch_bytes=BUF, **kw) as d:
            msgs = d.decode(x, chunk=100003)
            runs.append(([fields(x) for x in msgs], d.launch_count(), d.stats()))
    assert runs[0] == runs[1]


@pytest.mark.gpu
def test_setters():
    x = traffic_off(4, "uc8", 3e6)
    with api.Decoder() as dec:
        for o in (1, -1, 1_000_000):                                        # 2 MHz, then 2.4 MS/s
            with pytest.raises(RuntimeError, match="not supported"):
                dec.set_input_offset(o)
        dec.set_input_offset(0)
        dec.set_input_rate(2_400_000)
        with pytest.raises(RuntimeError, match="not supported"):
            dec.set_input_offset(1)
        for hz, m in DM.RATES.items():
            dec.set_input_rate(hz)
            mx = (m - 1) * 1_000_000
            for bad in (mx + 1, -mx - 1):
                with pytest.raises(RuntimeError, match="not supported"):
                    dec.set_input_offset(bad)
            dec.set_input_offset(mx)
            dec.set_input_offset(-mx)
            dec.set_input_offset(0)
        dec.set_input_rate(8_000_000)
        dec.set_input_offset(3_000_000)
        for hz in (2_000_000, 2_400_000, 4_000_000, 6_000_000):             # ranges that exclude 3 MHz
            with pytest.raises(RuntimeError, match="not supported"):
                dec.set_input_rate(hz)
        dec.set_input_rate(10_000_000)
        dec.set_input_rate(8_000_000)
        dec.reset()
        dec.process(x[:1000])
        with pytest.raises(RuntimeError, match="in progress"):
            dec.set_input_offset(0)
        dec.finish()
        dec.reset()                                                         # reset keeps the offset
        dec.process(x)
        dec.finish()
        with api.Decoder() as d2:
            assert_same(dec.take_messages(), d2.decode(shifted(x, 4, "uc8", 3_000_000)), "after reset")
    with pytest.raises(RuntimeError, match="not supported"):
        api.Decoder(input_offset=1_000_000)


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["uc8", "sc16"])
def test_cli(tmp_path, fmt):
    o = -2_000_000
    x = traffic_off(3, fmt, o)
    px = tmp_path / "x6.bin"
    x.tofile(px)
    exe = str(ROOT / "dump1090-b200")
    with api.Decoder(input_rate=6_000_000, input_format=fmt, input_offset=o) as dec:
        want = "".join(f"{x.raw_line()}\n" for x in dec.decode(x))
    p2 = tmp_path / "x2.bin"
    shifted(x, 3, fmt, o).tofile(p2)
    for mode in (["--raw"], ["--beast", "--arrival", "--levels"]):
        a = subprocess.run([exe, "--ifile", str(px), "--sample-rate", "6000000", "--iformat", fmt.upper(), *mode,
                            "--input-offset", str(o), "--chunk", "100003"], capture_output=True, check=True)
        b = subprocess.run([exe, "--ifile", str(p2), *mode], capture_output=True, check=True)
        assert a.stdout == b.stdout and a.stderr == b.stderr and len(a.stdout) > 0, mode
        if mode == ["--raw"]:
            assert a.stdout.decode() == want
    for args in (["--input-offset", "1000000"], ["--sample-rate", "4000000", "--input-offset", "2000000"],
                 ["--sample-rate", "6000000", "--input-offset", "1e6"]):
        r = subprocess.run([exe, "--ifile", str(px), *args], capture_output=True)
        assert r.returncode != 0 and b"--input-offset" in r.stderr, args
