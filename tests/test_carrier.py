"""Carrier frequency of each message (modes_set_carrier).

The reference computation is tests/carrier_model.py, a restatement of the definition in include/modes_b200.h
from the 2 MHz bytes a stream is decoded from: the pulse samples of the delivered frame's bits, the pairs two
samples apart, the sum of z_later conj(z_earlier) and its code.  CPU tests cover the arithmetic (host build of
modes_carrier_core.cuh), the conversion to the code, the accuracy on synthetic fleets of known offsets, the
summary and the layout; GPU tests the kernel on constructed corpora and every decode path."""
import ctypes
import math
import subprocess

import numpy as np
import pytest

import carrier_model as CM
import checker as C
import decimate_model as DM
import input_format_model as IM
import resample_model as RM
import shift_model as SM
import test_arrival as TA
import test_kernel_edges as KE
import test_signal as TS
from dump1090_b200 import api, synth
from test_pool_input_format import FULL_CALLS, FULL_RX, _pool, _want_buffers, full_world  # noqa: F401

ROOT = C.ROOT
SHIM = ROOT / "tests" / "_build" / "libcarrier_core_host.so"
DSHIM = ROOT / "tests" / "_build" / "libcarrier_device.so"
BUF = api.BUFFER_BYTES
NS = BUF // 2
CAR_DTYPE = np.dtype([("re", "<i4", 2), ("im", "<i4", 2)])


def _accuracy():
    import importlib.util
    spec = importlib.util.spec_from_file_location("carrier_accuracy", ROOT / "scripts" / "carrier_accuracy.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def zero_carrier(m) -> bytes:
    b = bytearray(bytes(m))
    b[106:108] = b"\0\0"
    return bytes(b)


# ---------------------------------------------------------------- CPU: arithmetic


@pytest.fixture(scope="module")
def shim():
    subprocess.run(["make", "-s", "shim"], cwd=ROOT, check=True)
    lib = ctypes.CDLL(str(SHIM))
    lib.shim_carrier_window.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_void_p]
    lib.shim_carrier_code.restype = ctypes.c_int32
    lib.shim_carrier_code.argtypes = [ctypes.c_int32, ctypes.c_int32]
    return lib


N_WIN = 17 + 2 * 112                                     # window samples 0 .. 16+2*112


def _heads(rng, n):
    return rng.integers(0, 256, size=(n, 16), dtype=np.uint8)


def carrier_windows(rng):
    """(name, windows as I/Q bytes of samples 0 .. 16+2*112, attempt heads)."""
    yield "random", rng.integers(0, 256, size=(300, 2 * N_WIN), dtype=np.uint8), _heads(rng, 300)
    yield "saturated", rng.choice(np.array([0, 255], dtype=np.uint8), size=(150, 2 * N_WIN)), _heads(rng, 150)
    yield "extremes", np.tile(np.array([0, 255, 255, 0], np.uint8), (4, N_WIN // 2 + 1))[:, : 2 * N_WIN], _heads(rng, 4)
    for fill, name in ((0x00, "all_zero_bits"), (0xFF, "all_one_bits"), (0x55, "alternating"), (0xAA, "alternating2")):
        h = _heads(rng, 40)
        h[:, :14] = fill
        yield name, rng.integers(0, 256, size=(40, 2 * N_WIN), dtype=np.uint8), h
    # frames of the pulse model at known offsets, with noise
    h = _heads(rng, 200)
    wins = []
    for k in range(200):
        frame = bytes(h[k, :14])
        env = synth.frame_envelope(frame, frac=float(rng.uniform()))
        amp = float(rng.choice([6.0, 12.0, 40.0, 120.0]))
        f = float(rng.uniform(-450e3, 450e3))
        ph = float(rng.uniform(0, 2 * np.pi)) + 2 * np.pi * f / 2e6 * np.arange(N_WIN)
        x = np.zeros(N_WIN)
        x[: min(env.size, N_WIN)] = env[:N_WIN] * amp
        i = np.clip(np.rint(127 + x * np.cos(ph) + rng.normal(0, 1.5, N_WIN)), 0, 255)
        q = np.clip(np.rint(127 + x * np.sin(ph) + rng.normal(0, 1.5, N_WIN)), 0, 255)
        wins.append(np.stack([i, q], 1).reshape(-1).astype(np.uint8))
    yield "frames", np.array(wins), h


def model_record(win, head, bits):
    return CM.record(win, 0, bytes(head[:14]), bits)


@pytest.mark.parametrize("bits", [56, 112])
def test_shim_window_equals_model(shim, bits):
    rng = np.random.default_rng(bits)
    out = np.zeros(2, np.int32)
    n = 0
    for name, wins, heads in carrier_windows(rng):
        for w, h in zip(wins, heads):
            w, h = np.ascontiguousarray(w), np.ascontiguousarray(h)
            shim.shim_carrier_window(w.ctypes.data, h.ctypes.data, bits, out.ctypes.data)
            assert tuple(int(v) for v in out) == model_record(w, h, bits), (name, bits)
            n += 1
    assert n > 800


@pytest.mark.parametrize("bits", [56, 112])
def test_pair_counts(bits):
    assert len(CM.pairs(CM.frame_bits(bytes(14), bits))) == 2 + bits - 1          # all equal: the most pairs
    assert len(CM.pairs(CM.frame_bits(b"\xff" * 14, bits))) == 2 + bits - 1
    assert len(CM.pairs(CM.frame_bits(b"\x55" * 14, bits))) == 2                   # alternating: the preamble's
    # the largest record: every term 2 * 128^2 at saturation, far inside int32
    w = np.tile(np.array([255, 255], np.uint8), N_WIN)
    re, im = CM.record(w, 0, bytes(14), bits)
    assert re == (2 + bits - 1) * 2 * 128 * 128 and im == 0


def test_window_reaching_into_the_next_buffer():
    """j = 131069: the frame's window runs past the buffer into the next one's samples (the carry)."""
    rng = np.random.default_rng(3)
    stream = rng.integers(0, 256, size=2 * 2 * NS, dtype=np.uint8)
    head = _heads(rng, 1)[0]
    j = 131069
    for bits in (56, 112):
        win = stream[2 * j: 2 * (j + N_WIN)]
        assert CM.record(stream, j, bytes(head[:14]), bits) == model_record(win, head, bits)
    # past the end of the stream every sample reads as no signal
    tail = np.full(2 * N_WIN, 127, np.uint8)
    tail[:20] = stream[-20:]
    assert CM.record(stream, 2 * NS - 10, bytes(head[:14]), 112) == model_record(tail, head, 112)


def _code_cases():
    out = [(1, 0), (0, 1), (-1, 0), (0, -1), (1000, 0), (0, 1000), (-1000, 0), (0, -1000), (-1000, 1), (-1000, -1),
           (5, 5), (-5, 5), (-5, -5), (5, -5), (2 ** 22, 1), (-(2 ** 22), 1), (-(2 ** 22), -1), (1, 2 ** 22)]
    rng = np.random.default_rng(11)
    for _ in range(4000):
        a = float(rng.uniform(-np.pi, np.pi))
        r = float(rng.choice([3.0, 100.0, 1e5, 3e6]))
        out.append((int(round(r * math.cos(a))), int(round(r * math.sin(a)))))
    return [(re, im) for re, im in out if (re, im) != (0, 0)]


def test_code_conversion(shim):
    assert shim.shim_carrier_code(0, 0) == 0 == CM.code_of(0, 0)
    for re, im in _code_cases():
        got, want = shim.shim_carrier_code(re, im), CM.code_of(re, im)
        assert abs(got - want) <= 1 and got != 0, (re, im, got, want)
        assert 16384 - 5000 <= got <= 16384 + 5000
    # the axes and the wrap, exactly: +-250 kHz, 0 Hz, +500 kHz on the negative real axis, -500 kHz just below it
    assert [shim.shim_carrier_code(*z) for z in ((1, 0), (0, 1), (0, -1), (-1, 0))] == [16384, 18884, 13884, 21384]
    assert shim.shim_carrier_code(-(2 ** 22), -1) == 16384 - 5000
    # the sign: a frame above the centre turns its phase forward, im > 0, f > 0
    assert shim.shim_carrier_code(1000, 10) > 16384 > shim.shim_carrier_code(1000, -10)


def test_sign_on_a_synthetic_frame():
    """A frame synthesised 100 kHz above the centre of the bytes measures as +100 kHz."""
    frame = synth.make_frame(17, 5, (0x4840D6).to_bytes(3, "big") + bytes(7))
    for f in (100e3, -100e3, 420e3, -420e3):
        x = synth.synth_stream(1000, [(100, frame, 60.0, 0.3, 0.0, f)], sigma=0.0, seed=1)
        hz = CM.hz_of(CM.code_of(*CM.record(x, 100, frame, 112)))
        assert abs(hz - f) <= 2000, (f, hz)


def test_message_field_and_layout():
    assert api.Message.pad1.size == 3 and api.Message.pad1.offset == 105 and api.C.sizeof(api.Message) == 200
    m = api.Message()
    assert m.carrier_code == 0 and m.carrier_hz() is None
    raw = bytearray(bytes(m))
    raw[106:108] = (16384 - 1234).to_bytes(2, "little", signed=True)
    m2 = api.Message.from_buffer_copy(bytes(raw))
    assert m2.carrier_code == 16384 - 1234 and m2.carrier_hz() == -123400
    assert zero_carrier(m2) == bytes(m)


def test_carrier_summary():
    def msg(addr, code):
        m = api.Message()
        m.aa1, m.aa2, m.aa3 = addr >> 16, (addr >> 8) & 0xFF, addr & 0xFF
        api.C.c_int16.from_address(api.C.addressof(m) + 106).value = code
        return m

    s = api.carrier_summary([])
    assert s["messages"] == 0 and s["aircraft"] == 0 and s["receiver_hz"] is None and s["receiver_ppm"] is None
    msgs = [msg(0xA1, 16384 + 100), msg(0xA1, 16384 + 120), msg(0xA1, 16384 + 500), msg(0xB2, 16384 - 40),
            msg(0xC3, 16384 + 60), msg(0xC3, 16384 + 80), msg(0xD4, 0)]
    s = api.carrier_summary(msgs)
    assert s["messages"] == 6 and s["aircraft"] == 3
    assert s["per_aircraft"] == {0xA1: 12000.0, 0xB2: -4000.0, 0xC3: 7000.0}
    assert s["receiver_hz"] == 7000.0 and s["receiver_ppm"] == pytest.approx(7000.0 / 1090.0)


def test_setters_and_exports():
    assert "modes_set_carrier" in api.EXPORTS and "modes_pool_set_carrier" in api.EXPORTS
    L = api.lib()
    assert L.modes_set_carrier(None, 1) == -1 and L.modes_pool_set_carrier(None, 1) == -1


def test_c_host_refuses_carrier_with_gpu_resolve(tmp_path):
    subprocess.run(["make", "-s", "all"], cwd=ROOT, check=True)
    f = tmp_path / "x.bin"
    f.write_bytes(bytes(1000))
    r = subprocess.run([str(ROOT / "dump1090-b200"), "--ifile", str(f), "--carrier", "--gpu-resolve"], capture_output=True, text=True)
    assert r.returncode == 1 and "--carrier cannot be combined with --gpu-resolve" in r.stderr


# ---------------------------------------------------------------- CPU: accuracy on fleets of known offsets

# Measured with scripts/carrier_accuracy.py (1500 frames a case, DESIGN.md §6 has the table): median / p95
# absolute error and receiver estimate error in Hz.  At 2 MHz the error falls with the amplitude (3200 / 10300 Hz
# at 8 LSB, 500 / 1500 at 60); through the resampler and the decimator it stays near 3500 / 11000 Hz at every
# amplitude.  The limits are those numbers with a margin of about a third.
ACCURACY_LIMITS = {
    2_000_000: {8.0: (4500, 14000, 2500), 12.0: (3000, 9000, 2500), 20.0: (2000, 6000, 2000), 60.0: (700, 2000, 1000)},
    2_400_000: {8.0: (7000, 18000, 5500), 12.0: (4500, 14000, 2500), 20.0: (4500, 14000, 2500), 60.0: (4500, 15000, 2500)},
    8_000_000: {8.0: (5500, 16500, 3000), 12.0: (5000, 15000, 2500), 20.0: (5000, 15000, 2500), 60.0: (5000, 16500, 2500)},
}


@pytest.mark.parametrize("rate,offset", [(2_000_000, 0), (2_400_000, 0), (8_000_000, 0), (8_000_000, 2_000_000)],
                         ids=["2M", "2.4M", "8M", "8M-offset"])
@pytest.mark.parametrize("amp", [8.0, 12.0, 20.0, 60.0])
def test_accuracy_on_fleets(rate, offset, amp, checker_libs):
    r = _accuracy().measure(rate, offset, amp, n_frames=1500)
    med, p95, rx = ACCURACY_LIMITS[rate][amp]
    assert r["messages"] > 100 and r["aircraft"] >= 20, r
    assert r["median_hz"] <= med and r["p95_hz"] <= p95 and abs(r["receiver_err_hz"]) <= rx, r
    assert abs(r["bias_hz"]) <= 1500, r                    # the sign: a wrong one would put the bias near 2 x 400 kHz


# ---------------------------------------------------------------- GPU: every decode path


def _assert_codes(msgs, y):
    bad = [(int(m.sample_pos), m.carrier_code, CM.expected_code(y, m)) for m in msgs if m.carrier_code != CM.expected_code(y, m)]
    assert not bad, f"{len(bad)} of {len(msgs)} differ, first (pos, got, want): {bad[0]}"
    assert all(m.carrier_code != 0 for m in msgs if not m.recovered)


def _fleet(rate, seed, offset=0, fmt="uc8", n_frames=900):
    """A fleet of known offsets at `rate` (frames moved by `offset`) and the 2 MHz bytes the decoder decodes."""
    acc = _accuracy()
    sigma = 1.5 * np.sqrt(rate / 2_000_000)
    x, _ = synth.fleet_at_rate(20 * np.log10(30.0 / (np.sqrt(2.0) * sigma)), n_frames, seed, sample_rate=rate, amp=30.0,
                               n_aircraft=24, carrier_hz=float(offset), carrier_of=acc.true_hz)
    y = x
    if fmt != "uc8":
        shift = IM.DEFAULT_SHIFT[fmt]
        x = IM.to_sc16(x, shift)
        y = IM.convert(x, shift)
    if rate == 2_400_000:
        y = RM.resample(y)
    elif rate > 2_400_000:
        m = rate // 2_000_000
        y = SM.shift_decimate(y, m, offset) if offset else DM.decimate(y, m)
    return x, y


def _on_off(factory, x, chunk=None, **kw):
    off = factory(**kw).decode(x, chunk=chunk) if chunk else factory(**kw).decode(x)
    dec = factory(carrier=True, **kw)
    on = dec.decode(x, chunk=chunk) if chunk else dec.decode(x)
    assert [zero_carrier(m) for m in on] == [bytes(m) for m in off]
    assert all(m.carrier_code == 0 for m in off)
    return on, dec


PATHS = [dict(rate=2_000_000), dict(rate=2_400_000), dict(rate=4_000_000), dict(rate=8_000_000),
         dict(rate=8_000_000, offset=2_000_000), dict(rate=10_000_000, offset=-3_000_000), dict(rate=6_000_000, offset=1_000_000),
         dict(rate=2_000_000, fmt="sc16"), dict(rate=2_000_000, fmt="sc16q11"), dict(rate=2_400_000, fmt="sc16"),
         dict(rate=8_000_000, offset=2_000_000, fmt="sc16q11")]


def _pid(p):
    return f"{p['rate'] / 1e6:g}M" + (f"{p['offset'] / 1e6:+g}" if p.get("offset") else "") + (f"-{p['fmt']}" if p.get("fmt") else "")


def _decoder_kw(p):
    kw = dict(input_rate=p["rate"])
    if p.get("offset"):
        kw["input_offset"] = p["offset"]
    if p.get("fmt"):
        kw["input_format"] = p["fmt"]
    return kw


@pytest.mark.gpu
@pytest.mark.parametrize("p", PATHS, ids=_pid)
def test_every_rate_and_format_equals_model(p, gpu_decoder_factory, checker_libs):
    x, y = _fleet(p["rate"], 40 + len(PATHS) + p["rate"] // 1_000_000, p.get("offset", 0), p.get("fmt", "uc8"))
    kw = _decoder_kw(p)
    got, _ = _on_off(gpu_decoder_factory, x, **kw)
    assert len(got) > 300
    _assert_codes(got, y)
    s = api.carrier_summary(got)
    assert s["aircraft"] >= 20 and abs(s["receiver_hz"] - _accuracy().receiver_truth_hz(s)) < 3000, s
    # odd call sizes and small batches: the same messages
    dec = gpu_decoder_factory(carrier=True, max_batch_bytes=2 * BUF, **kw)
    assert [bytes(m) for m in dec.decode(x, chunk=300001)] == [bytes(m) for m in got]


@pytest.mark.gpu
@pytest.mark.parametrize("kw", TS.FLAGS, ids=TS._kid)
def test_streaming_paths_equal_model(kw, gpu_decoder_factory, checker_libs):
    """Host-fed in odd call sizes, device-fed (modes_process_device), two GPU shards: every message's code is
    the model's, and every other field and the statistics equal the switch-off decode."""
    import torch
    data = np.concatenate([synth.random_traffic(131072 * 6 + 4321, 1800, 95, n_aircraft=16), TS._seam_and_eof_stream(3, 5)])
    cfg = TS._cfg(kw)
    ref, dec = _on_off(gpu_decoder_factory, data, **cfg)
    off = gpu_decoder_factory(**cfg)
    off.decode(data)
    assert dec.stats() == off.stats()
    assert len(ref) > 200
    _assert_codes(ref, data)
    want = [bytes(m) for m in ref]
    for chunk in (1000, 262145, 300001):
        d = gpu_decoder_factory(carrier=True, max_batch_bytes=2 * BUF, **cfg)
        assert [bytes(m) for m in d.decode(data, chunk=chunk)] == want, chunk
    for batch in (1, 3):
        multi = gpu_decoder_factory(carrier=True, n_gpus=2, max_batch_bytes=batch * BUF, **cfg)
        assert [bytes(m) for m in multi.decode(data, chunk=300001)] == want
    t = torch.from_numpy(data).cuda()
    dev = gpu_decoder_factory(carrier=True, max_batch_bytes=2 * BUF, **cfg)
    assert [bytes(m) for m in dev.decode(t)] == want
    for variant in ("fused", "warp"):
        import os
        os.environ["MODES_EVAL_VARIANT"] = variant
        try:
            assert [bytes(m) for m in gpu_decoder_factory(carrier=True, **cfg).decode(data)] == want
        finally:
            del os.environ["MODES_EVAL_VARIANT"]


@pytest.mark.gpu
def test_device_fed_offset_stream_equals_model(gpu_decoder_factory, checker_libs):
    import torch
    x, y = _fleet(10_000_000, 77, 3_000_000, "sc16")
    kw = dict(input_rate=10_000_000, input_offset=3_000_000, input_format="sc16")
    host, _ = _on_off(gpu_decoder_factory, x, **kw)
    _assert_codes(host, y)
    dev = gpu_decoder_factory(carrier=True, max_batch_bytes=3 * BUF, **kw)
    t = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    got = []
    for lo in range(0, x.size, 777777):
        dev.process(t[lo: lo + 777777])
    dev.finish()
    got = dev.take_messages()
    assert [bytes(m) for m in got] == [bytes(m) for m in host]


@pytest.mark.gpu
def test_other_records_unchanged(gpu_decoder_factory, checker_libs):
    """With every other measurement on, the carrier changes no message field but its own, no statistic,
    level or spectrum record; it adds no launch when the signal pass already runs and one when it does not."""
    x, y = _fleet(8_000_000, 5, 2_000_000)
    kw = dict(input_rate=8_000_000, input_offset=2_000_000, signal=True, arrival=True, levels=True, spectrum=True,
              recover=True, max_batch_bytes=2 * BUF)
    a = gpu_decoder_factory(**kw)
    b = gpu_decoder_factory(carrier=True, **kw)
    ma, mb = a.decode(x), b.decode(x)
    assert [zero_carrier(m) for m in mb] == [bytes(m) for m in ma]
    _assert_codes([m for m in mb if not m.recovered], y)
    assert all(m.carrier_code == 0 for m in mb if m.recovered)
    assert any(m.signal for m in mb) and any(m.arrival for m in mb)
    assert a.stats() == b.stats() and a.recovery_stats() == b.recovery_stats()
    assert np.array_equal(a.take_levels(), b.take_levels()) and np.array_equal(a.take_spectra(), b.take_spectra())
    assert a.launch_count() == b.launch_count()
    plain, car = gpu_decoder_factory(max_batch_bytes=2 * BUF), gpu_decoder_factory(carrier=True, max_batch_bytes=2 * BUF)
    plain.decode(y)
    car.decode(y)
    batches = -(-(y.size // BUF + 1) // 2)
    assert car.launch_count() == plain.launch_count() + batches


@pytest.mark.gpu
def test_refused_with_gpu_resolve(gpu_decoder_factory):
    dec = gpu_decoder_factory(gpu_resolve=1)
    with pytest.raises(RuntimeError, match="gpu_resolve"):
        dec.set_carrier(True)
    dec.set_carrier(False)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["ingest", "pipelined"])
def test_full_pool_equals_model(mode, full_world, gpu_decoder_factory):
    """Every receiver of a full-size pool of mixed rates and formats, two batches in flight: the messages
    are the switch-off pool's with the model's codes on the bytes each receiver decodes."""
    rxs, calls = full_world["rxs"], full_world["calls"]
    out = {}
    for on in (False, True):
        nxt = [0] * FULL_RX
        with _pool(rxs, max_batch=FULL_RX, carrier=on) as pool:
            pending = 0
            for ids in calls:
                bufs = [rxs[r].buf(nxt[r]) for r in ids]
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
            out[on] = [(pool.take(r), pool.stats(r), pool.buffers(r)) for r in range(FULL_RX)]
    n = 0
    for r, rx in enumerate(rxs):
        (m_off, s_off, k), (m_on, s_on, k2) = out[False][r], out[True][r]
        assert k == k2 == _want_buffers(rx.rate, FULL_CALLS) and s_off == s_on
        assert [zero_carrier(m) for m in m_on] == [bytes(m) for m in m_off], r
        _assert_codes(m_on, rx.decoded(k))
        n += len(m_on)
    assert n > 1000


@pytest.mark.gpu
def test_c_host_carrier_line(gpu_decoder_factory, checker_libs, tmp_path):
    """--carrier: one stderr line, the same through --chunk sizes and rates, equal to carrier_summary; stdout
    unchanged."""
    subprocess.run(["make", "-s", "all"], cwd=ROOT, check=True)
    lines = {}
    for rate, offset in ((2_000_000, 0), (8_000_000, 2_000_000)):
        x, y = _fleet(rate, 91, offset)
        f = tmp_path / f"{rate}.bin"
        f.write_bytes(x.tobytes())
        base = [str(ROOT / "dump1090-b200"), "--ifile", str(f), "--raw", "--sample-rate", str(rate)]
        if offset:
            base += ["--input-offset", str(offset)]
        plain = subprocess.run(base, capture_output=True, text=True, check=True)
        for chunk in (4096, 262145, 16 << 20):
            r = subprocess.run(base + ["--carrier", "--chunk", str(chunk)], capture_output=True, text=True, check=True)
            assert r.stdout == plain.stdout
            line = [ln for ln in r.stderr.splitlines() if ln.startswith("carrier:")]
            assert len(line) == 1
            lines.setdefault(rate, set()).add(line[0])
        assert len(lines[rate]) == 1
        s = api.carrier_summary(gpu_decoder_factory(carrier=True, **_decoder_kw(dict(rate=rate, offset=offset))).decode(x))
        want = (f"carrier: {s['messages']} messages, {s['aircraft']} aircraft, receiver offset {s['receiver_hz']:+.0f} Hz "
                f"({s['receiver_ppm']:+.3f} ppm of 1090 MHz)")
        assert lines[rate] == {want}


# ---------------------------------------------------------------- GPU: the device harness


@pytest.fixture(scope="module")
def dshim():
    subprocess.run(["make", "-s", "dshim"], cwd=ROOT, check=True)
    lib = ctypes.CDLL(str(DSHIM))
    u32, p, i = ctypes.c_uint32, ctypes.c_void_p, ctypes.c_int
    lib.car_error.restype = ctypes.c_char_p
    lib.car_sm_count.restype = ctypes.c_int
    lib.car_signal_pass.argtypes = [p, u32, p, p, p, u32, u32, u32, i, i, i]
    assert lib.car_sm_count() > 0, lib.car_error()
    return lib


@pytest.fixture(scope="module")
def corpus():
    rng = np.random.default_rng(123)
    wins, heads = [], []
    for _, w, h in carrier_windows(rng):
        wins.append(w)
        heads.append(h)
    return np.concatenate(wins), np.concatenate(heads)


SENTINEL = np.frombuffer(b"\xa5" * 16, dtype=CAR_DTYPE)[0]


def expected_carrier(wins, heads, combos, limit):
    want = np.full(len(combos), SENTINEL, dtype=CAR_DTYPE)
    for i in range(min(limit, len(combos))):
        if not combos[i].any():
            continue
        for k in (0, 1):
            bits = int(combos[i, k])
            re, im = model_record(wins[i], heads[i, k], bits) if bits else (0, 0)
            want[i]["re"][k], want[i]["im"][k] = re, im
    return want


def run_dev(lib, batch, recs, switches, capacity=None, counter=None):
    recs = np.ascontiguousarray(recs).copy()
    car = np.full(recs.size, SENTINEL, dtype=CAR_DTYPE)
    body, carry = batch.args()
    rc = lib.car_signal_pass(body.ctypes.data, batch.n_buffers, carry.ctypes.data, recs.ctypes.data, car.ctypes.data, recs.size,
                             recs.size if capacity is None else capacity, recs.size if counter is None else counter,
                             *[int(s) for s in switches])
    assert rc == 0, lib.car_error()
    return recs, car


SWITCH_SETS = [(False, False, True), (True, False, True), (False, True, True), (True, True, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("placement", ["even", "odd", "carry", "last_j"])
def test_carrier_records_on_constructed_corpora(placement, dshim, corpus):
    wins, heads = corpus
    rng = np.random.default_rng(len(placement) + 17)
    n_dec = 0
    for nb, idx, t in TA.arrival_placements(len(wins), placement):
        batch = KE.Batch(nb)
        for i, ti in zip(idx, t):
            TA._put(batch, ti, wins[i])
        combos = TA.COMBOS[rng.integers(0, len(TA.COMBOS), idx.size)]
        hd = np.stack([heads[idx], heads[rng.permutation(idx)]], axis=1)
        recs = TA.arrival_records(rng, t, hd, combos)
        want = expected_carrier(wins[idx], hd, combos, idx.size)
        for sw in SWITCH_SETS:
            got_recs, got = run_dev(dshim, batch, recs, sw)
            # the records are what the same pass writes without the carrier
            ref_recs, ref = run_dev(dshim, batch, recs, (sw[0], sw[1], False))
            KE.assert_records_equal(got_recs, ref_recs, (placement, sw))
            assert (ref.view(np.uint8) == 0xA5).all()
            assert got.tobytes() == want.tobytes(), (placement, sw)
        n_dec += int((combos > 0).sum())
    assert n_dec > 0


@pytest.mark.gpu
def test_carrier_capacity_and_second_trip(dshim, corpus):
    wins, heads = corpus
    rng = np.random.default_rng(8)
    wins, heads = wins[:200], heads[:200]
    (nb, idx, t), = TA.arrival_placements(len(wins), "odd")
    batch = KE.Batch(nb)
    for i, ti in zip(idx, t):
        TA._put(batch, ti, wins[i])
    n = 600
    widx = rng.integers(0, len(wins), n)
    combos = TA.COMBOS[rng.integers(0, len(TA.COMBOS), n)]
    hd = np.stack([heads[widx], heads[widx]], axis=1)
    recs = TA.arrival_records(rng, t[widx], hd, combos)
    for capacity, counter in ((n // 3, n + 5), (n // 3, 2 ** 32 - 1), (n, 100), (n, 0), (0, n)):
        _, got = run_dev(dshim, batch, recs, (True, True, True), capacity, counter)
        want = expected_carrier(wins[widx], hd, combos, min(capacity, counter))
        assert got.tobytes() == want.tobytes(), (capacity, counter)
    # more records than 32 per warp of a full wave: the grid-stride loop comes back
    n = 32 * KE.MAX_WARPS_PER_SM * dshim.car_sm_count() * 5 // 2
    widx = rng.integers(0, len(wins), n)
    combos = TA.COMBOS[rng.integers(0, len(TA.COMBOS), n)]
    hd = np.stack([heads[widx], heads[widx]], axis=1)
    recs = TA.arrival_records(rng, t[widx], hd, combos)
    _, got = run_dev(dshim, batch, recs, (False, False, True))
    rec = {b: np.array([model_record(w, h, b) for w, h in zip(wins, heads)]) for b in (56, 112)}
    want = np.full(n, SENTINEL, dtype=CAR_DTYPE)
    dec = combos.any(axis=1)
    for k in (0, 1):
        bits = combos[:, k]
        v = np.where((bits == 112)[:, None], rec[112][widx], rec[56][widx])
        v[bits == 0] = 0
        want["re"][dec, k] = v[dec, 0]
        want["im"][dec, k] = v[dec, 1]
    assert got.tobytes() == want.tobytes()
    assert not dec.all() and dec.sum() > n // 2
