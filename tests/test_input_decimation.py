"""4, 6, 8 and 10 MS/s input (modes_set_input_rate, modes_resample_device_at): integer decimation by M = 2..5
in front of the 2 MHz pipeline.

The contract: decoding a stream at 2 M MS/s gives exactly what the 2 MHz decoder gives on the stream's
decimated bytes, defined by tests/decimate_model.py (a 16-bit stream converted first, as
tests/input_format_model.py defines).  CPU tests check the arithmetic (host build of modes_resample_core.cuh
against the model), the rate descriptor, the streaming of the model and the decode quality of the decimated
stream through the oracle; GPU tests check the kernel byte for byte and the contract on every decode path."""
import ctypes
import subprocess

import numpy as np
import pytest

import checker as C
import decimate_model as DM
import input_format_model as IF
import resample_model as RM
from dump1090_b200 import api, synth

ROOT = C.ROOT
SHIM = ROOT / "tests" / "_build" / "libdecimate_core_host.so"
BUF = api.BUFFER_BYTES
B = api.BUFFER_SAMPLES
NO_LIMIT = 2 ** 63 - 1
MS = (2, 3, 4, 5)
FLAGS = [(0, 0, 0), (0, 0, 1), (1, 0, 0), (1, 0, 1), (1, 1, 0), (1, 1, 1)]   # fix_errors, aggressive, check_crc
FORMATS = {"uc8": (-1, 1.0), "sc16": (8, 256.0), "sc16q11": (4, 16.0)}      # default shift, synth scale

# ---------------------------------------------------------------- CPU: arithmetic


@pytest.fixture(scope="module")
def shim():
    subprocess.run(["make", "-s", "shim"], cwd=ROOT, check=True)
    lib = ctypes.CDLL(str(SHIM))
    lib.shim_decimate.restype = ctypes.c_int
    lib.shim_decimate.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int64, ctypes.c_int64,
                                  ctypes.c_size_t, ctypes.c_int64, ctypes.c_int, ctypes.c_void_p]
    lib.shim_decimate_taps.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
    lib.shim_input_rate.argtypes = [ctypes.c_uint32, ctypes.c_void_p]
    lib.shim_input_reach.argtypes = [ctypes.c_uint32, ctypes.c_int64, ctypes.c_int64, ctypes.c_void_p]
    return lib


def _shim_range(shim, m, span, in_first, out_first, count, limit=NO_LIMIT, shift=-1):
    span = np.ascontiguousarray(span, dtype=np.uint8)
    out = np.zeros(2 * count, dtype=np.uint8)
    assert shim.shim_decimate(m, span.ctypes.data if span.size else None, span.size, in_first, out_first, count, limit,
                              shift, out.ctypes.data) == 0
    return out


def test_tap_tables_are_the_derivation(shim):
    for m in MS:
        h = np.zeros(32, np.int16)
        t = shim.shim_decimate_taps(m, h.ctypes.data, h.size)
        e, fc = DM.FILTER[m]
        assert t == m + 2 * e == DM.taps(m).size, m
        assert np.array_equal(h[:t], DM.derive_taps(m, e, fc)), m
        assert int(h[:t].astype(np.int64).sum()) == 16384 and np.array_equal(h[:t], h[:t][::-1]), m
    # the box: 1 / M in Q14, the remainder on the middle tap
    assert DM.derive_taps(3).tolist() == [5461, 5462, 5461]
    assert DM.derive_taps(5).tolist() == [3277, 3277, 3276, 3277, 3277]


def test_rate_descriptor(shim):
    v = np.zeros(6, np.int32)
    r = np.zeros(3, np.int64)
    for hz in (3_000_000, 12_000_000, 2_400_001, 0):
        assert shim.shim_input_rate(hz, v.ctypes.data) == -1, hz
    for hz, m in DM.RATES.items():
        assert shim.shim_input_rate(hz, v.ctypes.data) == 0
        e = DM.extent(DM.taps(m), m)
        assert v.tolist() == [1, m, e, m + 2 * e, 240, m], hz
        for n in (-240, -1, 0, 7, B - 1, 2 ** 32 // m + 3, 2 ** 40 + 5):
            for n_in in (0, 1, m - 1, m, m + 1, 2 ** 33 + 1):
                assert shim.shim_input_reach(hz, n, n_in, r.ctypes.data) == 0
                assert r.tolist() == [*DM.input_span(n, 1, m), DM.n_out(n_in, m)], (hz, n, n_in)
    for n in (-238, 0, 5, 2 ** 35 + 1):                                      # 2.4 MS/s as K9 defines it
        assert shim.shim_input_reach(2_400_000, n, 1001, r.ctypes.data) == 0
        assert r.tolist() == [*RM.input_span(n, 1), RM.n_out(1001)]
    assert shim.shim_input_reach(2_000_000, 9, 1001, r.ctypes.data) == 0 and r.tolist() == [9, 10, 1001]


def _cases(rng, m):
    yield "random", rng.integers(0, 256, 4000 * m + 6, dtype=np.uint8)
    yield "random_odd", rng.integers(0, 256, 1001 * m, dtype=np.uint8)
    for v in (0, 127, 255):
        yield f"const{v}", np.full(800 * m, v, np.uint8)
    for k in (1, 2, 3):                                                     # full scale, runs of k samples
        ch = np.tile(np.r_[np.zeros(k), np.full(k, 255)], 300).astype(np.uint8)
        yield f"alternation{k}", np.stack([ch, 255 - ch], 1).reshape(-1)
    for n in (1, 2, 3, 2 * m - 1, 2 * m + 1, 16 * m + 3):
        yield f"len{n}", rng.integers(0, 256, n, dtype=np.uint8)


@pytest.mark.parametrize("m", MS)
def test_host_build_equals_model(shim, m):
    rng = np.random.default_rng(m)
    for name, data in _cases(rng, m):
        n = DM.n_out((data.size + 1) // 2, m)
        assert np.array_equal(_shim_range(shim, m, data, 0, 0, n), DM.decimate(data, m)), (m, name)
    assert (DM.decimate(np.full(6000, 127, np.uint8), m) == 127).all()


@pytest.mark.parametrize("m", MS)
def test_host_build_spans_limits_and_positions(shim, m):
    """Output ranges anywhere in the stream (negative ones: the first batch's carry, and positions past 2^32
    input samples and past 2^32 int16 bytes) from an input span, every other input no signal, with the EOF
    limit; UC8 and int16 at several shifts."""
    rng = np.random.default_rng(20 + m)
    x = rng.integers(0, 256, 2 * 3000 * m + 1, dtype=np.uint8)
    x16 = rng.integers(-2 ** 15, 2 ** 15, 2 * 3000 * m, dtype=np.int64).astype("<i2").view(np.uint8)
    bases = [0, 2 ** 30 // m + 5, 2 ** 32 // m - 700, 2 ** 32 // m + 9, 2 ** 40 // m]    # output samples
    for base in bases:
        for first, count in [(-240, 240), (-7, 50), (0, 2000), (13, 1003), (2500, 600)]:
            o = base + first
            lo, hi = DM.input_span(o, count, m)
            b0 = m * base                                                   # the data's first input sample
            for shift, data, bps in ((-1, x, 2), (8, x16, 4), (4, x16, 4), (0, x16, 4)):
                conv = data if shift < 0 else IF.convert(data, shift)
                want = DM.decimate_range(conv, m, o, count, in_first=b0)
                slo = max(lo, b0)
                span = data[bps * (slo - b0): bps * (hi - b0)]
                assert np.array_equal(_shim_range(shim, m, span, slo, o, count, shift=shift), want), (m, base, first, shift)
            limit = o + 17
            assert np.array_equal(_shim_range(shim, m, x, b0, o, count, limit),
                                  DM.decimate_range(x, m, o, count, limit=limit, in_first=b0)), (m, base, first)
    assert (DM.decimate_range(x, m, -240, 240)[: 2 * 230] == 127).all()     # the stream start's carry


@pytest.mark.parametrize("m", MS)
def test_impulse_at_every_phase(shim, m):
    """A single full-scale sample at every input phase: each output sees the tap at its offset."""
    h = DM.taps(m)
    e = DM.extent(h, m)
    for pos in range(40, 40 + 2 * m + 1):
        for val in (0, 255):
            data = np.full(2 * 40 * m, 127, np.uint8)
            data[2 * pos] = val
            data[2 * pos + 1] = 255 - val
            got = _shim_range(shim, m, data, 0, 0, 40)
            assert np.array_equal(got, DM.decimate(data, m)), (m, pos, val)
            y = got.reshape(-1, 2).astype(np.int64)
            k = pos - (m * np.arange(40) - e)
            ok = (k >= 0) & (k < h.size)
            want = np.zeros(40, np.int64)
            want[ok] = (h[k[ok]].astype(np.int64) * (val - 127) + 8192) >> 14
            assert np.array_equal(y[:, 0] - 127, want), (m, pos, val)
            assert np.array_equal(y[:, 1] - 127, (h[np.clip(k, 0, h.size - 1)].astype(np.int64) * (128 - val) + 8192 >> 14)
                                  * ok), (m, pos, val)


@pytest.mark.parametrize("m", MS)
def test_streaming_model_equals_whole(m):
    rng = np.random.default_rng(4 + m)
    x = rng.integers(0, 256, 40 * m + 1, dtype=np.uint8)
    whole = DM.decimate(x, m)
    for cut in range(x.size + 1):
        s = DM.Streaming(m)
        got = np.concatenate([s.feed(x[:cut]), s.feed(x[cut:]), s.finish()])
        assert np.array_equal(got, whole), (m, cut)
    s = DM.Streaming(m)
    got = np.concatenate([s.feed(x[k: k + 1]) for k in range(x.size)] + [s.finish()])
    assert np.array_equal(got, whole)
    assert s.hist.size <= 2 * (DM.taps(m).size + 1) + 1                     # only the history is kept


def test_tone_is_opt_in():
    frames = [(100, synth.make_frame(17, 5, bytes(range(10))), 30.0, 1.0, 0.25)]
    base = synth.synth_stream_at(2000, frames, sigma=2.0, seed=3, sample_rate=8_000_000)
    assert np.array_equal(synth.synth_stream_at(2000, frames, sigma=2.0, seed=3, sample_rate=8_000_000, tone=None), base)
    assert not np.array_equal(synth.synth_stream_at(2000, frames, sigma=2.0, seed=3, sample_rate=8_000_000,
                                                    tone=(2.5e6, 20.0)), base)


def _df17(msgs, truth):
    got = [bytes(m.msg[:14]).hex() for m in msgs if m.msgtype == 17 and m.msgbits == 112]
    true = sum(1 for h in got if h in truth)
    return true, len(got) - true


TONE = (2.5e6, 20.0)
# From the sweep in DESIGN §6 (scripts/decimate_quality.py, 300 frames x seeds 0-1, density-matched noise):
# the chosen filter's true frames at 12 and 18 dB, clean and with the 2.5 MHz tone; the floors are 85 % of them.
SWEEP = {2: {12: (261, 226), 18: (436, 381)}, 3: {12: (338, 341), 18: (508, 505)},
         4: {12: (338, 334), 18: (483, 485)}, 5: {12: (342, 340), 18: (508, 505)}}


@pytest.mark.parametrize("m", MS)
@pytest.mark.parametrize("snr", (12, 18))
def test_quality_through_oracle(checker_libs, m, snr):
    for case, tone in ((0, None), (1, TONE)):
        true = false = 0
        for seed in range(2):
            x, truth = synth.fleet_at_rate(snr - 10 * np.log10(m), 300, seed, sample_rate=2_000_000 * m, tone=tone)
            t, f = _df17(C.oracle_decode(DM.decimate(x, m))[0], truth)
            true += t
            false += f
        assert false == 0, (m, snr, tone)
        assert true >= int(0.85 * SWEEP[m][snr][case]), (m, snr, tone, true)


@pytest.mark.parametrize("m", MS)
def test_no_false_frames_at_low_snr(checker_libs, m):
    for snr in (6, 8, 10):
        for tone in (None, TONE):
            x, truth = synth.fleet_at_rate(snr - 10 * np.log10(m), 300, 7, sample_rate=2_000_000 * m, tone=tone)
            assert _df17(C.oracle_decode(DM.decimate(x, m))[0], truth)[1] == 0, (m, snr, tone)


@pytest.mark.parametrize("m", MS)
def test_modes1_round_trip(checker_libs, m):
    """modes1 with each sample repeated M times: the box gives modes1 back byte for byte; the product's filter
    decodes every one of its frames."""
    y = C.modes1()
    up = DM.upsample(y, m)
    assert np.array_equal(DM.decimate(up, m, DM.derive_taps(m)), y)
    base = {bytes(x.msg[: x.msgbits // 8]).hex() for x in C.oracle_decode(y)[0]}
    got = {bytes(x.msg[: x.msgbits // 8]).hex() for x in C.oracle_decode(DM.decimate(up, m))[0]}
    assert len(base) == 75 and base <= got


def test_python_rates():
    assert api.INPUT_RATES == (2_000_000, 2_400_000, 4_000_000, 6_000_000, 8_000_000, 10_000_000)
    for nbytes in (0, 1, 2, 39, 40, 41, 10 ** 9 + 1):
        assert api.resampled_samples(nbytes) == RM.n_out((nbytes + 1) // 2)
        for hz, m in DM.RATES.items():
            assert api.resampled_samples(nbytes, hz) == DM.n_out((nbytes + 1) // 2, m)
    with pytest.raises(ValueError):
        api.resampled_samples(10, 3_000_000)


# ---------------------------------------------------------------- GPU

_inputs = {}


def traffic_at(m: int, fmt: str, n_samples: int = 600_000, seed: int = 3) -> np.ndarray:
    """random_traffic's frames at 2 M MS/s in the format: positions, amplitudes, phases and fractional
    delays drawn like random_traffic's."""
    key = (m, fmt, n_samples, seed)
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
                                             scale=FORMATS[fmt][1])
    return _inputs[key]


def fleet(m: int, fmt: str) -> np.ndarray:
    key = ("fleet", m, fmt)
    if key not in _inputs:
        _inputs[key] = synth.fleet_at_rate(12 - 10 * np.log10(m), 1000, 1, sample_rate=2_000_000 * m,
                                           dtype="uc8" if fmt == "uc8" else "sc16", scale=FORMATS[fmt][1])[0]
    return _inputs[key]


def modes1_at(m: int, fmt: str) -> np.ndarray:
    y = DM.upsample(C.modes1(), m)
    return y if fmt == "uc8" else IF.to_sc16(y, FORMATS[fmt][0])


def decimated(x, m, fmt) -> np.ndarray:
    return DM.decimate(x if fmt == "uc8" else IF.convert(x, FORMATS[fmt][0]), m)


def fields(m) -> tuple:
    return tuple(bytes(getattr(m, f)) if f in ("msg", "flight", "pad1") else getattr(m, f) for f, _ in api.Message._fields_)


def assert_same(got, want, what):
    assert len(got) == len(want), (what, len(got), len(want))
    for k, (g, w) in enumerate(zip(got, want)):
        assert fields(g) == fields(w), (what, k, g.raw_line(), w.raw_line(), g.sample_pos, w.sample_pos)


def _dec(m, fmt, **kw):
    return api.Decoder(input_rate=2_000_000 * m, input_format=fmt, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("m", MS)
def test_resample_device_at_equals_model(m):
    import torch
    rng = np.random.default_rng(8 + m)
    hz = 2_000_000 * m
    x = np.concatenate([traffic_at(m, "uc8", 2 * B * m), rng.integers(0, 256, 1001, dtype=np.uint8)])
    n_total = DM.n_out((x.size + 1) // 2, m)
    with api.Decoder() as dec:
        d_x = torch.from_numpy(x).cuda()
        for first, nb, base in [(0, 1, 0), (0, 2, 0), (1, 1, 0), (0, 3, 0), (1, 1, 2 ** 32 // (m * B) + 1),
                                (0, 2, 2 ** 34 // (m * B))]:
            out = torch.zeros(nb * BUF, dtype=torch.uint8, device="cuda")
            o0 = first * B
            lo, hi = DM.input_span(o0 - 240, nb * B + 240, m)
            lo = max(lo, 0)
            hi = min(hi, (x.size + 1) // 2)
            # a span with its history only, the stream moved base buffers later (input m B base samples)
            span = torch.zeros(2 * (hi - lo) + 16, dtype=torch.uint8, device="cuda")
            span[: min(2 * hi, x.size) - 2 * lo] = d_x[2 * lo: 2 * hi]
            sb = base * B
            carry = dec.resample_device_at(hz, span.data_ptr(), min(2 * hi, x.size) - 2 * lo, lo + m * sb, first + base,
                                           nb, out.data_ptr(), out_end=n_total + sb)
            want = DM.decimate_range(x, m, o0 - 238, nb * B + 238, limit=n_total)
            assert carry == want[:476].tobytes(), (m, first, nb, base)
            got = out.cpu().numpy()
            assert np.array_equal(got, want[476:]), (m, first, nb, base, np.flatnonzero(got != want[476:])[:5])
        out = torch.zeros(2 * BUF, dtype=torch.uint8, device="cuda")
        launches = dec.launch_count()
        assert dec.resample_device_at(hz, d_x.data_ptr(), x.size, 0, 1, 2, out.data_ptr(), want_carry=False) is None
        torch.cuda.synchronize()
        assert dec.launch_count() - launches == 1
        assert np.array_equal(out.cpu().numpy(), DM.decimate_range(x, m, B, 2 * B))
        with pytest.raises(RuntimeError, match="16-byte aligned"):
            dec.resample_device_at(hz, d_x.data_ptr() + 2, 100, 0, 0, 1, out.data_ptr())
        for bad in (2_000_000, 3_000_000, 12_000_000):
            with pytest.raises(RuntimeError, match="not supported"):
                dec.resample_device_at(bad, d_x.data_ptr(), 100, 0, 0, 1, out.data_ptr())
        # modes_resample_device is modes_resample_device_at(2400000)
        a = dec.resample_device(d_x.data_ptr(), x.size, 0, 1, 1, out.data_ptr())
        b = dec.resample_device_at(2_400_000, d_x.data_ptr(), x.size, 0, 1, 1, out.data_ptr() + BUF)
        torch.cuda.synchronize()
        assert a == b and torch.equal(out[:BUF], out[BUF:])


def _oracle_check(y, want, want_st, fix, aggressive, check_crc, drop, what):
    ora, ora_st = C.oracle_decode(y, fix=fix, aggressive=aggressive, check_crc=check_crc, drop_eof=drop)
    assert [m.raw_line() for m in want] == [m.hexline() for m in ora], what
    assert [m.sample_pos for m in want] == [m.sample_pos for m in ora], what
    assert list(want_st.values()) == ora_st, what


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", list(FORMATS))
@pytest.mark.parametrize("m", MS)
def test_contract(checker_libs, m, fmt):
    """Decoder(input_rate=2 M MHz, input_format=fmt) == Decoder() on the model's decimated bytes == the
    oracle on them, with every FLAGS set, both EOF modes, whole, odd-sized and one-byte calls."""
    data = {"traffic": traffic_at(m, fmt), "fleet": fleet(m, fmt), "modes1": modes1_at(m, fmt)}
    for fix, aggressive, check_crc in FLAGS:
        cfg = dict(fix_errors=fix, aggressive=aggressive, check_crc=check_crc)
        for drop in (0, 1):
            with _dec(m, fmt, drop_eof_buffer=drop, **cfg) as dm, api.Decoder(drop_eof_buffer=drop, **cfg) as d2:
                for name, x in data.items():
                    y = decimated(x, m, fmt)
                    want = d2.decode(y)
                    want_st = d2.stats()
                    _oracle_check(y, want, want_st, fix, aggressive, check_crc, drop, (m, fmt, name))
                    for chunk in ((None, 100003) if (fix, aggressive, check_crc) != (1, 0, 1) else (None, 100003, 3 << 19)):
                        got = dm.decode(x, chunk=chunk)
                        assert_same(got, want, (m, fmt, name, drop, chunk))
                        assert dm.stats() == want_st, (m, fmt, name, drop, chunk)
                if (fix, aggressive, check_crc) == (1, 0, 1):                   # an EOF buffer only, one-byte calls
                    x = data["traffic"][: 40001 * (2 if fmt == "uc8" else 4)]
                    want = d2.decode(decimated(x, m, fmt))
                    assert_same(dm.decode(x, chunk=1), want, (m, fmt, "bytes", drop))


@pytest.mark.gpu
@pytest.mark.parametrize("m,fmt", [(2, "uc8"), (5, "sc16")])
def test_contract_calls_across_buffers(m, fmt):
    """One-byte calls across a whole buffer, and random call sizes that straddle the batches."""
    bps = 2 if fmt == "uc8" else 4
    x = traffic_at(m, fmt, 2 * m * B + 777, 5)
    x = x[: x.size - (x.size % bps) + (1 if fmt == "uc8" else 3)]             # and a partial last sample
    with api.Decoder() as d2:
        want = d2.decode(decimated(x, m, fmt))
    with _dec(m, fmt, max_batch_bytes=2 * BUF) as dm:
        n1 = (m * B + 5000) * bps
        dm.reset()
        for k in range(n1):
            dm.process(x[k: k + 1])
        dm.process(x[n1:])
        dm.finish()
        assert_same(dm.take_messages(), want, "one byte")
        rng = np.random.default_rng(1)
        dm.reset()
        off = 0
        while off < x.size:
            n = int(rng.integers(1, 700_000))
            dm.process(x[off: off + n])
            off += n
        dm.finish()
        assert_same(dm.take_messages(), want, "random calls")


SWITCHES = [dict(signal=True), dict(arrival=True, signal=True), dict(levels=True), dict(levels=True, drop_eof_buffer=1),
            dict(recover=True), dict(recover=True, weak_preambles=True), dict(gpu_resolve=1),
            dict(n_gpus=2, max_batch_bytes=BUF), dict(n_gpus=2, levels=True, recover=True)]


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", list(FORMATS))
@pytest.mark.parametrize("m", MS)
def test_contract_with_switches(m, fmt):
    for kw in SWITCHES:
        for name, x in (("traffic", traffic_at(m, fmt)), ("fleet", fleet(m, fmt))):
            y = decimated(x, m, fmt)
            with _dec(m, fmt, **kw) as dm, api.Decoder(**kw) as d2:
                want = d2.decode(y)
                wres = dict(stats=d2.stats())
                if kw.get("levels"):
                    wres["levels"] = d2.take_levels()
                if kw.get("recover"):
                    wres["recovery"] = d2.recovery_stats()
                    wres["weak"] = d2.weak_recovery_stats()
                for chunk in (None, 100003):
                    got = dm.decode(x, chunk=chunk)
                    assert_same(got, want, (m, fmt, kw, name, chunk))
                    assert dm.stats() == wres["stats"], (m, fmt, kw, name)
                    if kw.get("levels"):
                        assert np.array_equal(dm.take_levels(), wres["levels"]), (m, fmt, kw, name)
                    if kw.get("recover"):
                        assert dm.recovery_stats() == wres["recovery"] and dm.weak_recovery_stats() == wres["weak"]
                if kw.get("signal") and name == "traffic":
                    assert any(x.signal for x in want)
                if kw.get("arrival") and name == "traffic":
                    assert any(x.arrival for x in want)


@pytest.mark.gpu
def test_setter():
    with api.Decoder() as dec:
        for bad in (3_000_000, 12_000_000, 2_400_001):
            with pytest.raises(RuntimeError, match="not supported"):
                dec.set_input_rate(bad)
        x = traffic_at(4, "uc8")
        for hz in (4_000_000, 6_000_000, 8_000_000, 10_000_000):
            dec.reset()
            dec.process(x[:1000])
            with pytest.raises(RuntimeError, match="in progress"):
                dec.set_input_rate(hz)
            dec.finish()
        dec.set_input_rate(8_000_000)                                       # between streams
        with api.Decoder() as d2:
            assert_same(dec.decode(x), d2.decode(decimated(x, 4, "uc8")), "after finish")
    with api.ReceiverPool(2) as pool:
        with pytest.raises(RuntimeError, match="not supported"):
            pool.set_input_rate(0, 8_000_000)


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", list(FORMATS))
def test_cli(tmp_path, fmt):
    x = traffic_at(4, fmt)
    px, p2 = tmp_path / "x8.bin", tmp_path / "x2.bin"
    x.tofile(px)
    decimated(x, 4, fmt).tofile(p2)
    exe = str(ROOT / "dump1090-b200")
    for mode in (["--raw"], ["--beast"], ["--beast", "--arrival", "--levels"]):
        a = subprocess.run([exe, "--ifile", str(px), "--sample-rate", "8000000", "--iformat", fmt.upper(), *mode,
                            "--chunk", "100003"], capture_output=True, check=True)
        b = subprocess.run([exe, "--ifile", str(p2), *mode], capture_output=True, check=True)
        assert a.stdout == b.stdout and len(a.stdout) > 0, (fmt, mode)
        assert a.stderr == b.stderr, (fmt, mode)
    r = subprocess.run([exe, "--ifile", str(px), "--sample-rate", "12000000"], capture_output=True)
    assert r.returncode != 0 and b"2400000" in r.stderr


# ---------------------------------------------------------------- GPU: past 2^32 input samples

PINNED = 192 << 20
SILENCE = {"uc8": 127, "sc16": 0, "sc16q11": 0}


def _shifted(msgs, base):
    out = []
    for x in msgs:
        c = x.copy()
        c.sample_pos += base * B
        out.append(c)
    return out


def _run_prefixed(m, fmt, prefix_buffers, **kw):
    bps = 2 if fmt == "uc8" else 4
    x = fleet(m, fmt)
    res = {}
    for with_prefix in (False, True):
        with _dec(m, fmt, **kw) as dec:
            if with_prefix:
                buf = api.PinnedBuffer(PINNED)
                try:
                    buf.array[:] = SILENCE[fmt]
                    left = prefix_buffers * B * m * bps
                    first = True
                    while left:
                        n = min(12_345_679 * bps if first else PINNED, left)
                        dec.process_ptr(buf.ptr, n)
                        left -= n
                        first = False
                finally:
                    buf.free()
                assert not dec.take_messages() and not any(dec.stats().values())
                prefix_levels = dec.take_levels()
                assert prefix_levels.size >= prefix_buffers - 1
            for off in range(0, x.size, 100003):
                dec.process(x[off: off + 100003])
            dec.finish()
            res[with_prefix] = dict(msgs=dec.take_messages(), stats=dec.stats())
            res[with_prefix]["levels"] = dec.take_levels()
            if with_prefix:
                res[with_prefix]["levels"] = np.concatenate([prefix_levels, res[with_prefix]["levels"]])
            if kw.get("recover"):
                res[with_prefix]["recovery"] = dec.recovery_stats()
    return res[False], res[True]


@pytest.mark.gpu
@pytest.mark.parametrize("m,fmt", [(2, "uc8"), (5, "sc16"), (3, "sc16q11")])
def test_decoder_after_silent_prefix(m, fmt):
    """A silent prefix that carries the input past 2^32 samples (and the int16 byte offset past 2^34), then
    traffic: the traffic's own decode, shifted by the prefix."""
    prefix = 2 ** 32 // (m * B) + 2                         # 2 MHz buffers
    want, got = _run_prefixed(m, fmt, prefix, signal=True, arrival=True, levels=True, recover=True)
    assert len(got["msgs"]) == len(want["msgs"]) > 20
    for k, (g, w) in enumerate(zip(got["msgs"], _shifted(want["msgs"], prefix))):
        assert fields(g) == fields(w), (m, fmt, k, g.sample_pos, w.sample_pos)
        assert g.beast() == w.beast(), (m, fmt, k)
    assert got["stats"] == want["stats"] and got["recovery"] == want["recovery"]
    lv, wl = got["levels"], want["levels"].copy()
    assert lv.size == prefix + wl.size
    # the prefix's last buffer reads E input samples of the traffic through the filter, so it need not be silent
    assert list(lv["buffer"][:prefix]) == list(range(prefix)) and (lv["peak"][:prefix - 1] == 0).all()
    wl["buffer"] += prefix
    assert np.array_equal(lv[prefix:], wl)
