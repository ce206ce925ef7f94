"""2.4 MS/s input (modes_set_input_rate, modes_resample_device): the integer 5:6 polyphase resampler in
front of the 2 MHz pipeline.

The contract: decoding a 2.4 MS/s stream gives exactly what the 2 MHz decoder gives on the stream's
resampled bytes, with the resampled bytes defined by tests/resample_model.py.  CPU tests check the
arithmetic (host build of modes_resample_core.cuh against the model), the streaming of the model, the
rate-general signal model of synth, and the decode quality of the resampled stream through the oracle;
GPU tests check the kernel byte for byte and the contract on every decode path."""
import ctypes
import subprocess

import numpy as np
import pytest

import checker as C
import resample_model as RM
from dump1090_b200 import api, synth

ROOT = C.ROOT
SHIM = ROOT / "tests" / "_build" / "libresample_core_host.so"
BUF = api.BUFFER_BYTES
B = api.BUFFER_SAMPLES
NO_LIMIT = 2 ** 63 - 1
FLAGS = [(0, 0, 0), (0, 0, 1), (1, 0, 0), (1, 0, 1), (1, 1, 0), (1, 1, 1)]   # fix_errors, aggressive, check_crc

# ---------------------------------------------------------------- CPU: arithmetic


@pytest.fixture(scope="module")
def shim():
    subprocess.run(["make", "-s", "shim"], cwd=ROOT, check=True)
    lib = ctypes.CDLL(str(SHIM))
    lib.shim_resample.restype = ctypes.c_int
    lib.shim_resample.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int64, ctypes.c_int64, ctypes.c_size_t,
                                  ctypes.c_int64, ctypes.c_void_p]
    lib.shim_resample_taps.restype = ctypes.c_int
    lib.shim_resample_taps.argtypes = [ctypes.c_void_p, ctypes.c_int]
    return lib


def _shim_range(shim, span, in_first, out_first, count, limit=NO_LIMIT):
    span = np.ascontiguousarray(span, dtype=np.uint8)
    out = np.zeros(2 * count, dtype=np.uint8)
    assert shim.shim_resample(span.ctypes.data if span.size else None, span.size, in_first, out_first, count, limit,
                              out.ctypes.data) == 0
    return out


def _shim_whole(shim, data):
    data = np.asarray(data, dtype=np.uint8)
    return _shim_range(shim, data, 0, 0, RM.n_out((data.size + 1) // 2))


def test_tap_table_is_the_derivation(shim):
    taps = np.zeros(5 * 8, dtype=np.int16)
    t = shim.shim_resample_taps(taps.ctypes.data, taps.size)
    assert t == RM.TAPS
    table = taps[: 5 * t].reshape(5, t)
    assert np.array_equal(table, RM.derive_taps())
    assert (table.astype(np.int64).sum(axis=1) == 16384).all()
    ticks = np.arange(-5 * t, 5 * t + 1) / 5.0
    assert np.array_equal(RM.prototype(ticks), RM.prototype(-ticks))        # one symmetric prototype
    # the offsets are whole 12 MHz ticks, and branch r is the prototype 0.2 r input samples later
    assert np.array_equal(RM.offsets() * 5, np.round(RM.offsets() * 5))


def _cases(rng):
    yield "random", rng.integers(0, 256, 60006, dtype=np.uint8)
    yield "random_odd", rng.integers(0, 256, 20001, dtype=np.uint8)
    for v in (0, 127, 255):
        yield f"const{v}", np.full(12000, v, np.uint8)
    for k in (1, 2, 3):                                                     # full scale, runs of k samples
        ch = np.tile(np.r_[np.zeros(k), np.full(k, 255)], 2000 // k).astype(np.uint8)
        yield f"alternation{k}", np.stack([ch, 255 - ch], 1).reshape(-1)
    yield "alternation_i", np.tile(np.array([0, 127, 255, 127], np.uint8), 3001)
    for n in (1, 2, 3, 11, 12, 13, 23, 25):                                 # short, and not a multiple of 6 samples
        yield f"len{n}", rng.integers(0, 256, n, dtype=np.uint8)


def test_host_build_equals_model(shim):
    rng = np.random.default_rng(11)
    for name, data in _cases(rng):
        assert np.array_equal(_shim_whole(shim, data), RM.resample(data)), name
    # full-scale runs of 2 samples overshoot and clamp at both ends
    y = RM.resample(dict(_cases(rng))["alternation2"])
    assert y.min() == 0 and y.max() == 255
    assert (RM.resample(np.full(6000, 127, np.uint8)) == 127).all()


def test_impulse_at_every_phase(shim):
    """A single full-scale sample at every input phase: each output sees the taps of its branch."""
    for pos in range(30, 42):
        for val in (0, 255):
            data = np.full(2 * 80, 127, np.uint8)
            data[2 * pos] = val
            data[2 * pos + 1] = 255 - val
            got = _shim_whole(shim, data)
            assert np.array_equal(got, RM.resample(data)), (pos, val)
            y = got.reshape(-1, 2).astype(np.int64)[:, 0] - 127
            n = np.arange(y.size)
            q, r = np.divmod(n, 5)
            k = pos - (6 * q + r) + RM.TAPS // 2 - 1
            ok = (k >= 0) & (k < RM.TAPS)
            want = np.zeros(y.size, np.int64)
            want[ok] = (RM.H[r[ok], k[ok]].astype(np.int64) * (val - 127) + 8192) >> 14
            assert np.array_equal(y, want), (pos, val)


def test_host_build_spans_and_limits(shim):
    """Output ranges anywhere in the stream (negative ones: the first batch's carry) from an input span,
    every other input byte no signal, and the EOF limit."""
    rng = np.random.default_rng(2)
    x = rng.integers(0, 256, 30001, dtype=np.uint8)
    for first, count in [(-238, 238), (-7, 50), (0, 12500), (1000, 2003), (12000, 1000)]:
        lo, hi = RM.input_span(first, count)
        lo = max(lo, 0)
        span = x[2 * lo: 2 * hi]
        want = RM.resample_range(x, first, count)
        assert np.array_equal(_shim_range(shim, span, lo, first, count), want), (first, count)
        assert np.array_equal(_shim_range(shim, x, 0, first, count, first + 17),
                              RM.resample_range(x, first, count, limit=first + 17)), (first, count)
    assert (RM.resample_range(x, -238, 238)[: 2 * 230] == 127).all()          # the stream start's carry


def test_streaming_model_equals_whole():
    """The model fed in pieces, keeping only the history it needs, equals it run whole: every split
    point of a short stream, and one-byte pieces."""
    rng = np.random.default_rng(4)
    x = rng.integers(0, 256, 121, dtype=np.uint8)
    whole = RM.resample(x)
    for cut in range(x.size + 1):
        s = RM.Streaming()
        got = np.concatenate([s.feed(x[:cut]), s.feed(x[cut:]), s.finish()])
        assert np.array_equal(got, whole), cut
    s = RM.Streaming()
    got = np.concatenate([s.feed(x[k: k + 1]) for k in range(x.size)] + [s.finish()])
    assert np.array_equal(got, whole)
    assert s.hist.size <= 2 * (RM.TAPS + 4) + 1                               # only the history is kept


def test_synth_at_2mhz_is_synth_stream():
    rng = synth.Counter(5)
    frames = []
    for k in range(40):
        fr = synth.make_frame(17, 5, bytes(rng.below(256) for _ in range(10)))
        frac = [0.0, 0.5, 0.15 + 0.7 * rng.uniform()][k % 3]
        frames.append((100 + 300 * k + rng.below(50), fr, 5 + 100 * rng.uniform(), 6.28 * rng.uniform(), frac))
    n = 100 + 300 * 40
    assert np.array_equal(synth.synth_stream_at(n, frames, sigma=2.0, seed=3), synth.synth_stream(n, frames, sigma=2.0, seed=3))
    for snr in (8, 14):
        s2, t2 = synth.fleet_at(snr, 50, 1)
        s24, t24 = synth.fleet_at_rate(snr, 50, 1, sample_rate=2_000_000)
        assert t2 == t24 and np.array_equal(s2, s24)
    s24, t24 = synth.fleet_at_rate(12, 50, 1)
    assert t24 == t2 and s24.size == 2 * -(-(200 + 50 * 400 + 400) * 6 // 5)


def _df17(msgs, truth):
    got = [bytes(m.msg[:14]).hex() for m in msgs if m.msgtype == 17 and m.msgbits == 112]
    true = sum(1 for h in got if h in truth)
    return true, len(got) - true


# From the sweep in DESIGN §6 (T = 6, 1.1 MHz; 300 frames x seeds 0-2): 412 true frames at 14 dB, 547 at
# 18 dB, none false at any SNR.  The floors leave about 15 % of margin.
QUALITY_FLOOR = {14: 350, 18: 465}


@pytest.mark.parametrize("snr", sorted(QUALITY_FLOOR))
def test_quality_through_oracle(checker_libs, snr):
    true = false = 0
    for seed in range(3):
        s24, truth = synth.fleet_at_rate(snr, 300, seed)
        t, f = _df17(C.oracle_decode(RM.resample(s24))[0], truth)
        true += t
        false += f
    assert false == 0
    assert true >= QUALITY_FLOOR[snr], true


def test_no_false_frames_at_low_snr(checker_libs):
    for snr in (6, 8, 10):
        s24, truth = synth.fleet_at_rate(snr, 300, 7)
        assert _df17(C.oracle_decode(RM.resample(s24))[0], truth)[1] == 0, snr


def upsampled_modes1() -> np.ndarray:
    """modes1() upsampled 6:5 in floating point and quantised to u8: a 2.4 MS/s capture."""
    from scipy.signal import resample_poly
    x = C.modes1().astype(np.float64).reshape(-1, 2) - 127.0
    y = resample_poly(x, 6, 5, axis=0)
    return np.clip(np.rint(y + 127.0), 0, 255).astype(np.uint8).reshape(-1)


def test_modes1_round_trip(checker_libs):
    base = {bytes(m.msg[: m.msgbits // 8]).hex() for m in C.oracle_decode(C.modes1())[0]}
    got = {bytes(m.msg[: m.msgbits // 8]).hex() for m in C.oracle_decode(RM.resample(upsampled_modes1()))[0]}
    assert len(base) == 75 and base <= got


# ---------------------------------------------------------------- GPU


def traffic24(n_samples: int, nframes: int, seed: int) -> np.ndarray:
    """A random_traffic-style stream at 2.4 MS/s: random_traffic's frames (with their flipped bits) at its
    positions, amplitudes, phases and fractional delays drawn like random_traffic's."""
    _, truth = synth.random_traffic(n_samples * 5 // 6, nframes, seed, return_truth=True)
    rng = synth.Counter(seed + 1000)
    frames = []
    for pos, frame, flips in truth:
        amp = 12.0 + 98.0 * rng.uniform()
        frac = 0.15 + 0.7 * rng.uniform() if rng.below(2) else 0.0
        frames.append((pos, synth.flip_bits(frame, flips), amp, 2 * np.pi * rng.uniform(), frac))
    return synth.synth_stream_at(n_samples, frames, sigma=1.5, seed=seed, sample_rate=2_400_000)


_inputs = {}


def inputs():
    if not _inputs:
        _inputs["traffic"] = traffic24(500_000, 500, 3)
        _inputs["fleet10"] = synth.fleet_at_rate(10, 1200, 1)[0]
        _inputs["fleet16"] = synth.fleet_at_rate(16, 1200, 2)[0]
        _inputs["modes1"] = upsampled_modes1()
    return _inputs


def fields(m) -> tuple:
    return tuple(bytes(getattr(m, f)) if f in ("msg", "flight", "pad1") else getattr(m, f) for f, _ in api.Message._fields_)


def assert_same(got, want, what):
    assert len(got) == len(want), (what, len(got), len(want))
    for k, (g, w) in enumerate(zip(got, want)):
        assert fields(g) == fields(w), (what, k, g.raw_line(), w.raw_line(), g.sample_pos, w.sample_pos)


def _decode(dec, data, chunk):
    msgs = dec.decode(data, chunk=chunk)
    return msgs, dec.stats()


@pytest.mark.gpu
def test_resample_device_equals_model(gpu_decoder_factory):
    import torch
    rng = np.random.default_rng(8)
    x = np.concatenate([traffic24(400_000, 300, 5), rng.integers(0, 256, 1001, dtype=np.uint8)])
    n_total = RM.n_out((x.size + 1) // 2)
    dec = gpu_decoder_factory()
    d_x = torch.from_numpy(x).cuda()
    for first, nb in [(0, 1), (0, 2), (1, 1), (1, 2), (2, 1), (0, 3)]:
        out = torch.zeros(nb * BUF, dtype=torch.uint8, device="cuda")
        o0 = first * B
        lo, hi = RM.input_span(o0 - 238, nb * B + 238)
        lo = max(lo, 0)
        hi = min(hi, (x.size + 1) // 2)
        # a span with its history only: the bytes before it are not given
        span = torch.zeros(2 * (hi - lo) + 16, dtype=torch.uint8, device="cuda")
        span[: min(2 * hi, x.size) - 2 * lo] = d_x[2 * lo: 2 * hi]
        carry = dec.resample_device(span.data_ptr(), min(2 * hi, x.size) - 2 * lo, lo, first, nb, out.data_ptr(),
                                    out_end=n_total)
        want = RM.resample_range(x, o0 - 238, nb * B + 238, limit=n_total)
        assert carry == want[:476].tobytes(), (first, nb)
        got = out.cpu().numpy()
        assert np.array_equal(got, want[476:]), (first, nb, np.flatnonzero(got != want[476:])[:5])
        if first == 0:
            assert carry == bytes([127]) * 476
    # the whole input without a carry request, no limit
    out = torch.zeros(2 * BUF, dtype=torch.uint8, device="cuda")
    launches = dec.launch_count()
    assert dec.resample_device(d_x.data_ptr(), x.size, 0, 1, 2, out.data_ptr(), want_carry=False) is None
    torch.cuda.synchronize()
    assert dec.launch_count() - launches == 1
    assert np.array_equal(out.cpu().numpy(), RM.resample_range(x, B, 2 * B))
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        dec.resample_device(d_x.data_ptr() + 2, 100, 0, 0, 1, out.data_ptr())


@pytest.mark.gpu
@pytest.mark.parametrize("fix,aggressive,check_crc", FLAGS)
def test_contract(gpu_decoder_factory, checker_libs, fix, aggressive, check_crc):
    """Decoder(input_rate=2_400_000) == Decoder() on the model's resampled bytes == the oracle on them."""
    cfg = dict(fix_errors=fix, aggressive=aggressive, check_crc=check_crc)
    for drop in (0, 1):
        d24 = gpu_decoder_factory(input_rate=2_400_000, drop_eof_buffer=drop, **cfg)
        d20 = gpu_decoder_factory(drop_eof_buffer=drop, **cfg)
        for name, x in inputs().items():
            y = RM.resample(x)
            want, want_st = _decode(d20, y, None)
            ora, ora_st = C.oracle_decode(y, fix=fix, aggressive=aggressive, check_crc=check_crc, drop_eof=drop)
            assert [m.raw_line() for m in want] == [m.hexline() for m in ora], name
            assert [m.sample_pos for m in want] == [m.sample_pos for m in ora], name
            assert list(want_st.values()) == ora_st, name
            for chunk in (None, 100003, 3 << 19):
                got, st = _decode(d24, x, chunk)
                assert_same(got, want, (name, drop, chunk))
                assert st == want_st, (name, drop, chunk)
        # one-byte calls on a short stream (an EOF buffer only) and odd call sizes
        x = inputs()["traffic"][:40001]
        want = _decode(d20, RM.resample(x), None)
        got, st = _decode(d24, x, 1)
        assert_same(got, want[0], ("bytes", drop))
        assert st == want[1]


@pytest.mark.gpu
def test_contract_one_byte_calls_over_a_buffer(gpu_decoder_factory):
    """One-byte calls across whole buffers, and call sizes that straddle the batches."""
    x = inputs()["traffic"][: 2 * 330_000 + 1]
    want = gpu_decoder_factory().decode(RM.resample(x))
    d24 = gpu_decoder_factory(input_rate=2_400_000, max_batch_bytes=2 * BUF)
    assert_same(d24.decode(x, chunk=1), want, "one byte")
    rng = np.random.default_rng(1)
    d24.reset()
    off = 0
    while off < x.size:
        n = int(rng.integers(1, 300_000))
        d24.process(x[off: off + n])
        off += n
    d24.finish()
    assert_same(d24.take_messages(), want, "random calls")


def _switch_case(factory, x, **kw):
    y = RM.resample(x)
    d24 = factory(input_rate=2_400_000, **kw)
    d20 = factory(**kw)
    out = {}
    for name, dec, data in (("24", d24, x), ("20", d20, y)):
        msgs = []
        for chunk in ((None, 100003) if name == "24" else (None,)):
            msgs.append(dec.decode(data, chunk=chunk))
            res = dict(stats=dec.stats())
            if kw.get("levels"):
                res["levels"] = dec.take_levels()
            if kw.get("recover"):
                res["recovery"] = dec.recovery_stats()
                res["weak"] = dec.weak_recovery_stats()
            out.setdefault(name, []).append((msgs[-1], res))
    (want, wres), = out["20"]
    for got, res in out["24"]:
        assert_same(got, want, kw)
        for k, v in wres.items():
            if k == "levels":
                assert np.array_equal(res[k], v), kw
            else:
                assert res[k] == v, (kw, k)
    return want


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(signal=True), dict(arrival=True, signal=True), dict(levels=True),
                                dict(levels=True, drop_eof_buffer=1), dict(recover=True),
                                dict(recover=True, weak_preambles=True), dict(gpu_resolve=1),
                                dict(n_gpus=2, max_batch_bytes=BUF), dict(n_gpus=2, levels=True, recover=True)],
                         ids=["signal", "arrival", "levels", "levels_drop", "recover", "weak", "gpu_resolve", "gpus2",
                              "gpus2_passes"])
def test_contract_with_switches(gpu_decoder_factory, kw):
    for name in ("traffic", "fleet10", "modes1"):
        want = _switch_case(gpu_decoder_factory, inputs()[name], **kw)
        if kw.get("signal"):
            assert any(m.signal for m in want)
        if kw.get("arrival"):
            assert any(m.arrival for m in want)


@pytest.mark.gpu
def test_setter(gpu_decoder_factory):
    dec = gpu_decoder_factory()
    with pytest.raises(RuntimeError, match="not supported"):
        dec.set_input_rate(2_400_001)
    x = inputs()["traffic"][:300_000]
    dec.reset()
    dec.process(x[:1000])
    with pytest.raises(RuntimeError, match="in progress"):
        dec.set_input_rate(2_400_000)
    dec.finish()
    dec.set_input_rate(2_400_000)                                           # between streams
    assert_same(dec.decode(x), gpu_decoder_factory().decode(RM.resample(x)), "after finish")
    dec.reset()
    dec.process(x[:10])
    with pytest.raises(RuntimeError, match="in progress"):
        dec.set_input_rate(2_000_000)
    d_default = gpu_decoder_factory()
    d_explicit = gpu_decoder_factory(input_rate=2_000_000)
    d_explicit.set_input_rate(2_000_000)
    y = inputs()["modes1"]
    assert_same(d_explicit.decode(y), d_default.decode(y), "explicit 2 MHz")
    assert d_explicit.launch_count() == d_default.launch_count()


@pytest.mark.gpu
def test_cli(tmp_path):
    x = inputs()["traffic"]
    p24, p20 = tmp_path / "x24.bin", tmp_path / "x20.bin"
    x.tofile(p24)
    RM.resample(x).tofile(p20)
    exe = str(ROOT / "dump1090-b200")
    for mode in (["--raw"], ["--beast"], ["--beast", "--arrival", "--levels"]):
        a = subprocess.run([exe, "--ifile", str(p24), "--sample-rate", "2400000", *mode, "--chunk", "100003"],
                           capture_output=True, check=True)
        b = subprocess.run([exe, "--ifile", str(p20), *mode], capture_output=True, check=True)
        assert a.stdout == b.stdout and len(a.stdout) > 0, mode
        assert a.stderr == b.stderr, mode
    r = subprocess.run([exe, "--ifile", str(p24), "--sample-rate", "2400001"], capture_output=True)
    assert r.returncode != 0 and b"2400000" in r.stderr
