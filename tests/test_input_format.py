"""16-bit input (modes_set_input_format): SC16 and SC16Q11 I/Q converted to UC8 in front of the pipeline.

The contract: decoding a 16-bit stream gives exactly what the UC8 decoder gives on the stream's converted
bytes, at either input rate, with the conversion defined by tests/input_format_model.py.  CPU tests check
the arithmetic (host build of modes_input_core.cuh against the model on every value and shift), the
streaming of the model, the round trip of UC8 captures written as 16-bit, and what the shift does to decode
quality through the oracle; GPU tests check both kernels byte for byte and the contract on every decode
path, switch, setter and the C host."""
import ctypes
import hashlib
import re
import subprocess

import numpy as np
import pytest

import checker as C
import input_format_model as M
import resample_model as RM
from dump1090_b200 import api, synth

ROOT = C.ROOT
SHIM = ROOT / "tests" / "_build" / "libinput_core_host.so"
DSHIM = ROOT / "tests" / "_build" / "libinput_device.so"
BUF = api.BUFFER_BYTES
B = api.BUFFER_SAMPLES
NO_LIMIT = 2 ** 63 - 1
FLAGS = [(0, 0, 0), (0, 0, 1), (1, 0, 0), (1, 0, 1), (1, 1, 0), (1, 1, 1)]   # fix_errors, aggressive, check_crc
SCALE = {"sc16": 256.0, "sc16q11": 16.0}          # int16 units per UC8 LSB at full scale
# the reference's --raw output on checker.modes1() (as pinned in tests/test_oracle.py): lines, md5
MODES1_RAW = {0: (147, "f23b14fbd58d"), 1: (119, "896cf3d1da7e")}


def _md5(lines) -> tuple:
    return len(lines), hashlib.md5("".join(h + "\n" for h in lines).encode()).hexdigest()[:12]

# ---------------------------------------------------------------- CPU: arithmetic


@pytest.fixture(scope="module")
def shim():
    subprocess.run(["make", "-s", "shim"], cwd=ROOT, check=True)
    lib = ctypes.CDLL(str(SHIM))
    lib.shim_input_convert.restype = ctypes.c_int
    lib.shim_input_convert.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_void_p]
    lib.shim_input_format.restype = ctypes.c_int
    lib.shim_input_format.argtypes = [ctypes.c_uint32, ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_int)]
    return lib


def test_host_build_equals_model_on_every_value(shim):
    """All 65536 int16 values (as I, and reversed as Q) at all 16 shifts."""
    v = np.arange(-32768, 32768, dtype=np.int64)
    iq = np.stack([v, v[::-1]], 1).astype("<i2").reshape(-1).view(np.uint8)
    for s in range(16):
        out = np.zeros(2 * v.size, np.uint8)
        assert shim.shim_input_convert(iq.ctypes.data, v.size, s, out.ctypes.data) == 0
        assert np.array_equal(out, M.convert(iq, s)), s
        # round half up, then clamp: the definition spelled out for the I values
        want = np.clip(127 + np.floor(v / 2.0 ** s + 0.5).astype(np.int64), 0, 255)
        assert np.array_equal(out[0::2], want), s
    assert shim.shim_input_convert(iq.ctypes.data, 1, 16, out.ctypes.data) == -1


def test_format_constants(shim):
    sb, ds = ctypes.c_int(), ctypes.c_int()
    got = {}
    for name, f in M.FORMATS.items():
        assert shim.shim_input_format(f, ctypes.byref(sb), ctypes.byref(ds)) == 0
        got[name] = (sb.value, ds.value)
    assert got == {"uc8": (2, 0), "sc16": (4, 8), "sc16q11": (4, 4)}
    assert {k: v[1] for k, v in got.items() if k != "uc8"} == M.DEFAULT_SHIFT
    assert shim.shim_input_format(3, ctypes.byref(sb), ctypes.byref(ds)) == -1
    assert api.INPUT_FORMATS == M.FORMATS
    header = (ROOT / "include" / "modes_b200.h").read_text()
    for name, f in M.FORMATS.items():
        assert re.search(rf"#define MODES_INPUT_{name.upper()}\s+{f}u\n", header), name


def test_streaming_model_equals_whole():
    """The model fed in pieces, splits inside a sample included, equals it run whole; 1-3 trailing bytes
    are ignored."""
    rng = np.random.default_rng(4)
    x = rng.integers(0, 256, 4 * 30 + 3, dtype=np.uint8)
    for s in (0, 4, 8, 15):
        whole = M.convert(x, s)
        assert whole.size == 2 * 30
        for cut in range(x.size + 1):
            st = M.Streaming(s)
            got = np.concatenate([st.feed(x[:cut]), st.feed(x[cut:]), st.finish()])
            assert np.array_equal(got, whole), (s, cut)
        st = M.Streaming(s)
        got = np.concatenate([st.feed(x[k: k + 1]) for k in range(x.size)] + [st.finish()])
        assert np.array_equal(got, whole), s
        for extra in (1, 2, 3):
            assert np.array_equal(M.convert(x[: 120 + extra], s), M.convert(x[:120], s))


@pytest.mark.parametrize("fmt", ["sc16q11", "sc16"])
def test_round_trip(checker_libs, fmt):
    """v = 2^s (b - 127) - 2^(s-1) converts back to b for every byte at the format's default shift and
    stays in the format's range; so modes1 written in the format converts back to modes1 and decodes to
    the reference's lines."""
    s = M.DEFAULT_SHIFT[fmt]
    b = np.arange(256, dtype=np.uint8)
    v = M.to_sc16(b, s).view("<i2")
    lim = 2048 if fmt == "sc16q11" else 32768
    assert v.min() >= -lim and v.max() < lim
    assert np.array_equal(M.convert_values(v, s), b)
    y = C.modes1()
    x = M.to_sc16(y, s)
    assert np.array_equal(M.convert(x, s), y)
    for drop in (0, 1):
        msgs, _ = C.oracle_decode(M.convert(x, s), drop_eof=drop)
        assert _md5([m.hexline() for m in msgs]) == MODES1_RAW[drop], drop


def _df17(msgs, truth):
    got = [bytes(m.msg[:14]).hex() for m in msgs if m.msgtype == 17 and m.msgbits == 112]
    true = sum(1 for h in got if h in truth)
    return true, len(got) - true


def test_no_false_frames_at_any_shift(checker_libs):
    """An SC16Q11 fleet (full scale 2048) through the oracle: no false frame at any SNR or shift, and the
    default shift delivers (DESIGN §6)."""
    for snr in (6, 10, 14, 20):
        x, truth = synth.fleet_at_rate(snr, 300, 1, sample_rate=2_000_000, dtype="sc16", scale=SCALE["sc16q11"])
        for s in range(16):
            t, f = _df17(C.oracle_decode(M.convert(x, s))[0], truth)
            assert f == 0, (snr, s)
            if snr >= 14 and s == M.DEFAULT_SHIFT["sc16q11"]:
                assert t >= 150, (snr, t)


def test_smaller_shift_for_a_quiet_capture(checker_libs):
    """A quiet SC16Q11 capture (pulses at 1/64 of full scale): the default shift leaves them below one
    UC8 step, a smaller shift resolves them (DESIGN §6: 0 and 177 true frames at 14 dB)."""
    for snr in (14, 20):
        x, truth = synth.fleet_at_rate(snr, 300, 1, sample_rate=2_000_000, amp=2.0, dtype="sc16", scale=SCALE["sc16q11"])
        default = _df17(C.oracle_decode(M.convert(x, 4))[0], truth)
        small = _df17(C.oracle_decode(M.convert(x, 1))[0], truth)
        assert small[1] == 0 and default[1] == 0
        assert small[0] >= 150 and small[0] > default[0] + 100, (snr, small, default)


def test_synth_uc8_unchanged_and_sc16_is_the_same_signal():
    x8, t8 = synth.fleet_at_rate(12, 50, 1)
    x8b, t8b = synth.fleet_at_rate(12, 50, 1, dtype="uc8", scale=5.0)
    assert t8 == t8b and np.array_equal(x8, x8b)
    x16, t16 = synth.fleet_at_rate(12, 50, 1, dtype="sc16", scale=1.0)
    assert t16 == t8 and x16.size == 2 * x8.size
    # at scale 1 and shift 0 the conversion is the UC8 quantisation itself
    assert np.array_equal(M.convert(x16, 0), x8)

# ---------------------------------------------------------------- GPU: kernels


@pytest.fixture(scope="module")
def dshim():
    subprocess.run(["make", "-s", "dshim"], cwd=ROOT, check=True)
    lib = ctypes.CDLL(str(DSHIM))
    lib.input_error.restype = ctypes.c_char_p
    lib.input_run.restype = ctypes.c_int
    lib.input_run.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int64, ctypes.c_int64, ctypes.c_uint64,
                              ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    return lib


def _run(dshim, span, in_first, out_first, out_samples, out_end, halo, rate24, shift):
    span = np.ascontiguousarray(span, dtype=np.uint8)
    body = np.zeros(2 * out_samples, np.uint8)
    blk = np.zeros(512, np.uint8)
    rc = dshim.input_run(span.ctypes.data if span.size else None, span.size, in_first, out_first, out_samples, out_end,
                         int(halo), int(rate24), shift, body.ctypes.data, blk.ctypes.data)
    assert rc == 0, dshim.input_error()
    return body, blk


def _stream16(seed: int, n: int) -> np.ndarray:
    """Full-range random int16 I/Q (every shift clips some of it) with 3 trailing bytes."""
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, 4 * n + 3, dtype=np.uint8)


def _expect_carry(want476):
    blk = np.full(512, 127, np.uint8)
    blk[4:480] = want476
    return blk


@pytest.mark.gpu
def test_convert_kernel_equals_model(dshim):
    """K10 over spans from several buffers, with and without the carry block, with EOF limits; the span
    starts at the carry block's first sample (or the stream's) and holds only what the batch reads."""
    x = _stream16(3, 3 * B + 5000)
    n_in = x.size // 4
    for s in (0, 1, 4, 8, 15):
        y = M.convert(x, s)
        for first, nb in [(0, 1), (0, 2), (1, 1), (1, 2), (2, 1), (3, 1), (0, 4)]:
            for limit in (None, n_in, first * B + 777):
                o0 = first * B
                lo = max(o0 - 240, 0)
                hi = min(o0 + nb * B, n_in)
                span = x[4 * lo: 4 * hi + (3 if hi == n_in else 0)]
                ys = np.full(2 * (nb * B + 240), 127, np.uint8)           # samples o0 - 240 ... o1 - 1
                a, b = max(o0 - 240, 0), min(o0 + nb * B, n_in)
                ys[2 * (a - (o0 - 240)): 2 * (b - (o0 - 240))] = y[2 * a: 2 * b]
                if limit is not None and limit < o0 + nb * B:
                    ys[2 * max(limit - (o0 - 240), 0):] = 127
                for halo in (True, False):
                    body, blk = _run(dshim, span, lo, o0, nb * B, NO_LIMIT if limit is None else limit, halo, 0, s)
                    assert np.array_equal(body, ys[480:]), (s, first, nb, limit, halo, np.flatnonzero(body != ys[480:])[:5])
                    if halo:
                        assert np.array_equal(blk, _expect_carry(ys[4:480])), (s, first, nb, limit)
                    else:
                        assert (blk == 0x5A).all()


@pytest.mark.gpu
def test_resample_kernel_int16_equals_model(dshim):
    """K9 on int16 spans: convert, then resample, byte for byte, from spans that hold only the history."""
    x = _stream16(5, 3 * 6 * B // 5 + 7000)
    n_in = x.size // 4
    for s in (0, 4, 8, 15):
        y = M.convert(x, s)
        n_total = RM.n_out(n_in)
        for first, nb in [(0, 1), (0, 2), (1, 1), (1, 2), (2, 1)]:
            for limit in (None, n_total, first * B + 501):
                o0 = first * B
                lo, hi = RM.input_span(o0 - 238, nb * B + 238)
                lo, hi = max(lo, 0), min(hi, n_in)
                want = RM.resample_range(y, o0 - 238, nb * B + 238, limit=limit)
                for halo in (True, False):
                    body, blk = _run(dshim, x[4 * lo: 4 * hi], lo, o0, nb * B, NO_LIMIT if limit is None else limit,
                                     halo, 1, s)
                    assert np.array_equal(body, want[476:]), (s, first, nb, limit, np.flatnonzero(body != want[476:])[:5])
                    if halo:
                        assert np.array_equal(blk, _expect_carry(want[:476])), (s, first, nb, limit)
                    else:
                        assert (blk == 0x5A).all()

# ---------------------------------------------------------------- GPU: the contract


def _noisy_sc16(y: np.ndarray, s: int, seed: int) -> np.ndarray:
    """UC8 bytes written as int16 that convert back to them at shift s, with random low bits."""
    v = M.to_sc16(y, s).view("<i2").astype(np.int64)
    if s:
        v += np.random.default_rng(seed).integers(0, 1 << s, v.size)
    return v.astype("<i2").view(np.uint8)


def _traffic(n_samples: int, nframes: int, seed: int, rate: int, scale: float) -> np.ndarray:
    """random_traffic's frames at its positions, as 16-bit I/Q at the rate."""
    _, truth = synth.random_traffic(n_samples * 2_000_000 // rate, nframes, seed, return_truth=True)
    rng = synth.Counter(seed + 1000)
    frames = []
    for pos, frame, flips in truth:
        amp = 12.0 + 98.0 * rng.uniform()
        frac = 0.15 + 0.7 * rng.uniform() if rng.below(2) else 0.0
        frames.append((pos, synth.flip_bits(frame, flips), amp, 2 * np.pi * rng.uniform(), frac))
    return synth.synth_stream_at(n_samples, frames, sigma=1.5, seed=seed, sample_rate=rate, dtype="sc16", scale=scale)


_inputs = {}


def inputs(fmt: str, rate: int) -> dict:
    """16-bit streams of the format at the rate: traffic, a fleet at 10 dB, modes1 (at 2.4 MS/s upsampled),
    and full-range noise; each has 1-3 trailing bytes."""
    key = (fmt, rate)
    if key not in _inputs:
        from test_input_rate import upsampled_modes1
        sc, s = SCALE[fmt], M.DEFAULT_SHIFT[fmt]
        y1 = C.modes1() if rate == 2_000_000 else upsampled_modes1()
        d = {"traffic": _traffic(600_000, 600, 3, rate, sc),
             "fleet10": synth.fleet_at_rate(10, 1200, 1, sample_rate=rate, dtype="sc16", scale=sc)[0],
             "modes1": _noisy_sc16(y1, s, 9),
             "noise": _stream16(7, 300_000)[:-1]}
        for k, v in d.items():
            tail = {"traffic": 1, "fleet10": 2, "modes1": 3, "noise": 0}[k]
            d[k] = np.concatenate([v, np.full(tail, 0x41, np.uint8)]) if tail else v
        _inputs[key] = d
    return _inputs[key]


def fields(m) -> tuple:
    return tuple(bytes(getattr(m, f)) if f in ("msg", "flight", "pad1") else getattr(m, f) for f, _ in api.Message._fields_)


def assert_same(got, want, what):
    assert len(got) == len(want), (what, len(got), len(want))
    for k, (g, w) in enumerate(zip(got, want)):
        assert fields(g) == fields(w), (what, k, g.raw_line(), w.raw_line(), g.sample_pos, w.sample_pos)


RATES = [2_000_000, 2_400_000]


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["sc16", "sc16q11"])
@pytest.mark.parametrize("rate", RATES)
@pytest.mark.parametrize("fix,aggressive,check_crc", FLAGS)
def test_contract(gpu_decoder_factory, fmt, rate, fix, aggressive, check_crc):
    """Decoder(input_format=f, input_rate=r) on X == Decoder(input_rate=r) on convert(X): every message
    field and the statistics, both EOF modes, whole and in 100003-byte calls."""
    cfg = dict(fix_errors=fix, aggressive=aggressive, check_crc=check_crc, input_rate=rate)
    s = M.DEFAULT_SHIFT[fmt]
    for drop in (0, 1):
        d16 = gpu_decoder_factory(input_format=fmt, drop_eof_buffer=drop, **cfg)
        d8 = gpu_decoder_factory(drop_eof_buffer=drop, **cfg)
        for name, x in inputs(fmt, rate).items():
            want = d8.decode(M.convert(x, s))
            want_st = d8.stats()
            for chunk in (None, 100003):
                got = d16.decode(x, chunk=chunk)
                assert_same(got, want, (name, drop, chunk))
                assert d16.stats() == want_st, (name, drop, chunk)


@pytest.mark.gpu
@pytest.mark.parametrize("rate", RATES)
def test_contract_call_sizes(gpu_decoder_factory, rate):
    """One-byte calls across a buffer boundary (samples split across calls), and random call sizes with a
    small max_batch_bytes; at every shift a stream of the other format's scale still decodes as its
    conversion."""
    x = inputs("sc16q11", rate)["traffic"]
    for s in (4, 2, 0):
        want = gpu_decoder_factory(input_rate=rate).decode(M.convert(x, s))
        d16 = gpu_decoder_factory(input_format="sc16q11", input_shift=s, input_rate=rate, max_batch_bytes=2 * BUF)
        # the input byte of the first 2 MHz buffer boundary, give or take 2000 bytes
        cut = 4 * (B if rate == 2_000_000 else 6 * B // 5)
        d16.reset()
        d16.process(x[: cut - 2001])
        for k in range(cut - 2001, cut + 2003):
            d16.process(x[k: k + 1])
        d16.process(x[cut + 2003:])
        d16.finish()
        assert_same(d16.take_messages(), want, ("one byte", s))
        rng = np.random.default_rng(s)
        d16.reset()
        off = 0
        while off < x.size:
            n = int(rng.integers(1, 300_000))
            d16.process(x[off: off + n])
            off += n
        d16.finish()
        assert_same(d16.take_messages(), want, ("random calls", s))
        # a stream of 1-3 bytes decodes as an empty one
        for n in (1, 3):
            assert_same(d16.decode(x[:n], chunk=1), gpu_decoder_factory(input_rate=rate).decode(b""), ("tiny", n))


def _switch_case(factory, x, fmt, rate, **kw):
    s = M.DEFAULT_SHIFT[fmt]
    d16 = factory(input_format=fmt, input_rate=rate, **kw)
    d8 = factory(input_rate=rate, **kw)
    out = {}
    for name, dec, data in (("16", d16, x), ("8", d8, M.convert(x, s))):
        for chunk in ((None, 100003) if name == "16" else (None,)):
            msgs = dec.decode(data, chunk=chunk)
            res = dict(stats=dec.stats())
            if kw.get("levels"):
                res["levels"] = dec.take_levels()
            if kw.get("recover"):
                res["recovery"] = dec.recovery_stats()
                res["weak"] = dec.weak_recovery_stats()
            out.setdefault(name, []).append((msgs, res))
    (want, wres), = out["8"]
    for got, res in out["16"]:
        assert_same(got, want, kw)
        for k, v in wres.items():
            if k == "levels":
                assert np.array_equal(res[k], v), kw
            else:
                assert res[k] == v, (kw, k)
    return want, wres


@pytest.mark.gpu
@pytest.mark.parametrize("rate", RATES)
@pytest.mark.parametrize("kw", [dict(signal=True), dict(arrival=True, signal=True), dict(levels=True),
                                dict(levels=True, drop_eof_buffer=1), dict(recover=True),
                                dict(recover=True, weak_preambles=True), dict(gpu_resolve=1),
                                dict(n_gpus=2, max_batch_bytes=BUF), dict(n_gpus=2, levels=True, recover=True)],
                         ids=["signal", "arrival", "levels", "levels_drop", "recover", "weak", "gpu_resolve", "gpus2",
                              "gpus2_passes"])
def test_contract_with_switches(gpu_decoder_factory, rate, kw):
    for fmt, name in (("sc16q11", "traffic"), ("sc16q11", "fleet10"), ("sc16", "modes1"), ("sc16", "noise")):
        want, wres = _switch_case(gpu_decoder_factory, inputs(fmt, rate)[name], fmt, rate, **kw)
        if kw.get("signal") and name != "noise":
            assert any(m.signal for m in want)
        if kw.get("arrival") and name != "noise":
            assert any(m.arrival for m in want)
        if kw.get("levels") and name == "noise":
            assert wres["levels"]["clipped"].sum() > 0          # the shift saturates full-range noise


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["sc16q11", "sc16"])
def test_modes1_round_trip(gpu_decoder_factory, fmt):
    """modes1 written in the format decodes to the reference's lines on the GPU, both EOF modes."""
    x = _noisy_sc16(C.modes1(), M.DEFAULT_SHIFT[fmt], 1)
    for drop in (0, 1):
        got = gpu_decoder_factory(input_format=fmt, drop_eof_buffer=drop).decode(x)
        assert _md5([m.raw_line() for m in got]) == MODES1_RAW[drop], (fmt, drop)


@pytest.mark.gpu
def test_setter(gpu_decoder_factory):
    dec = gpu_decoder_factory()
    with pytest.raises(ValueError):
        dec.set_input_format("sc8")
    L = api.lib()
    assert L.modes_set_input_format(dec._h, 3, -1) != 0
    assert b"not supported" in L.modes_last_error(dec._h)
    with pytest.raises(RuntimeError, match="shift 16 is not supported"):
        dec.set_input_format("sc16", 16)
    with pytest.raises(RuntimeError, match="with UC8"):
        dec.set_input_format("uc8", 3)
    dec.set_input_format("uc8", 0)
    x = inputs("sc16q11", 2_000_000)["traffic"]
    dec.reset()
    dec.process(x[:1000])
    with pytest.raises(RuntimeError, match="in progress"):
        dec.set_input_format("sc16q11")
    dec.finish()
    dec.set_input_format("sc16q11")                                          # between streams
    want = gpu_decoder_factory().decode(M.convert(x, 4))
    assert_same(dec.decode(x), want, "after finish")
    dec.reset()                                                              # reset keeps the format
    assert_same(dec.decode(x, chunk=100003), want, "after reset")
    dec.reset()
    dec.process(x[:10])
    with pytest.raises(RuntimeError, match="in progress"):
        dec.set_input_format("uc8")
    dec.reset()
    dec.set_input_format("sc16q11", 2)                                       # takes effect at the next stream
    assert_same(dec.decode(x), gpu_decoder_factory().decode(M.convert(x, 2)), "shift 2")
    # an explicit uc8 is the default: the same messages and launches
    d_default = gpu_decoder_factory()
    d_explicit = gpu_decoder_factory(input_format="uc8", input_shift=0)
    d_explicit.set_input_format("uc8")
    y = C.modes1()
    assert_same(d_explicit.decode(y), d_default.decode(y), "explicit uc8")
    assert d_explicit.launch_count() == d_default.launch_count()
    # on two GPUs the format reaches both
    d2 = gpu_decoder_factory(n_gpus=2, max_batch_bytes=BUF, input_format="sc16q11")
    assert_same(d2.decode(x), want, "n_gpus=2")


@pytest.mark.gpu
def test_cli(tmp_path):
    exe = str(ROOT / "dump1090-b200")
    for rate in RATES:
        x = inputs("sc16q11", rate)["traffic"]
        p16, p8 = tmp_path / "x16.bin", tmp_path / "x8.bin"
        x.tofile(p16)
        M.convert(x, 4).tofile(p8)
        rate_arg = ["--sample-rate", str(rate)] if rate != 2_000_000 else []
        for mode in (["--raw"], ["--beast", "--arrival", "--levels"], ["--stats"]):
            a = subprocess.run([exe, "--iformat", "SC16Q11", "--ifile", str(p16), *rate_arg, *mode, "--chunk", "100003"],
                               capture_output=True, check=True)
            b = subprocess.run([exe, "--ifile", str(p8), *rate_arg, *mode], capture_output=True, check=True)
            assert a.stdout == b.stdout and len(a.stdout) > 0, (rate, mode)
            assert a.stderr == b.stderr, (rate, mode)
        # an explicit shift
        a = subprocess.run([exe, "--iformat", "SC16Q11", "--iformat-shift", "3", "--ifile", str(p16), *rate_arg, "--raw"],
                           capture_output=True, check=True)
        M.convert(x, 3).tofile(p8)
        b = subprocess.run([exe, "--ifile", str(p8), *rate_arg, "--raw"], capture_output=True, check=True)
        assert a.stdout == b.stdout and len(a.stdout) > 0, rate
    # modes1 as SC16Q11 and SC16: the reference's lines
    for fmt, spelled in (("sc16q11", "SC16Q11"), ("sc16", "SC16")):
        p = tmp_path / f"modes1_{fmt}.bin"
        M.to_sc16(C.modes1(), M.DEFAULT_SHIFT[fmt]).tofile(p)
        for drop in (0, 1):
            r = subprocess.run([exe, "--iformat", spelled, "--ifile", str(p), "--raw"] + (["--drop-eof-buffer"] if drop else []),
                               capture_output=True, check=True, text=True)
            assert _md5(r.stdout.splitlines()) == MODES1_RAW[drop], (fmt, drop)
    for bad, what in ((["--iformat", "SC8"], b"--iformat"), (["--iformat", "SC16", "--iformat-shift", "16"], b"--iformat-shift"),
                      (["--iformat", "SC16", "--iformat-shift", "x"], b"--iformat-shift"),
                      (["--iformat-shift", "2"], b"UC8")):
        r = subprocess.run([exe, "--ifile", str(tmp_path / "x16.bin"), *bad], capture_output=True)
        assert r.returncode != 0 and what in r.stderr, bad
