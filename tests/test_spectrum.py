"""The input spectrum pass (modes_set_spectrum, modes_pool_set_spectrum, K13): every record equals the numpy
restatement (tests/spectrum_model.py) from the raw stream bytes, on every decode path and per pool receiver,
and the switch changes no message, statistic or level record.

CPU tests cover the arithmetic (host build of modes_spectrum_core.cuh), the frame geometry, spectrum_summary
and the setters' refusals; GPU tests the kernel on every decode path, the pool and the C host."""
import ctypes
import re
import subprocess

import numpy as np
import pytest

import checker as C
import spectrum_model as SPM
from dump1090_b200 import api, synth

ROOT = C.ROOT
SHIM = ROOT / "tests" / "_build" / "libspectrum_core_host.so"
BUF = api.BUFFER_BYTES
B = api.BUFFER_BYTES // 2
N = SPM.N

# ---------------------------------------------------------------- CPU: arithmetic


@pytest.fixture(scope="module")
def shim():
    subprocess.run(["make", "-s", "shim"], cwd=ROOT, check=True)
    lib = ctypes.CDLL(str(SHIM))
    lib.shim_frame_power.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    lib.shim_geometry.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p,
                                  ctypes.c_void_p]
    return lib


def _host_power(shim, iq):
    iq = np.ascontiguousarray(iq, dtype=np.uint8).reshape(-1)
    n = iq.size // (2 * N)
    out = np.zeros(n * N, dtype=np.uint32)
    assert shim.shim_frame_power(iq.ctypes.data, n, out.ctypes.data) == 0
    return out.reshape(n, N).astype(np.uint64)


def _model_power(iq):
    return SPM.frame_power(np.asarray(iq, dtype=np.int64).reshape(-1, N, 2) - 127)


def _tone(k, amp=128.0, phase=0.0):
    """A full-scale complex tone at FFT bin k (natural index), as UC8 bytes."""
    n = np.arange(N)
    i = np.clip(np.rint(127 + amp * np.cos(2 * np.pi * k * n / N + phase)), 0, 255)
    q = np.clip(np.rint(127 + amp * np.sin(2 * np.pi * k * n / N + phase)), 0, 255)
    return np.stack([i, q], axis=1).astype(np.uint8).reshape(-1)


def _saturated_frames():
    alt = np.zeros(2 * N, np.uint8)
    alt[0::4] = alt[1::4] = 255                                        # (255, 255), (0, 0), ...
    alt_iq = np.tile(np.array([255, 0], np.uint8), N)                   # I at the top rail, Q at the bottom
    frames = [np.zeros(2 * N, np.uint8), np.full(2 * N, 255, np.uint8), alt, alt_iq,
              np.tile(np.array([0, 255], np.uint8), N)]
    frames += [_tone(k) for k in (0, 1, 17, 64, 127, 128, 200, 255)]
    frames += [_tone(k, amp=181.0, phase=0.3) for k in (5, 100)]      # clipped to the rails
    return np.concatenate(frames)


def test_host_build_equals_model(shim):
    rng = np.random.default_rng(13)
    for iq in (rng.integers(0, 256, 2 * N * 300, dtype=np.uint8), _saturated_frames(),
               np.clip(rng.normal(127, 40, 2 * N * 50), 0, 255).astype(np.uint8)):
        got, want = _host_power(shim, iq), _model_power(iq)
        assert np.array_equal(got, want)
    # no overflow at the extremes: every power under 2^32, as the bound says
    assert _model_power(_saturated_frames()).max() < 2 ** 32


def test_tone_lands_in_its_bin_and_silence_is_zero(shim):
    for k in (1, 17, 64, 100, 128, 200, 255):
        p = _host_power(shim, _tone(k, amp=100.0))[0]
        assert int(np.argmax(p)) == (k + N // 2) % N, k                  # record order: bin 128 is DC
        assert p[(k + N // 2) % N] > 1000 * np.sort(p)[-4]              # the Hann window's two neighbours aside
    assert not _host_power(shim, np.full(2 * N * 4, 127, np.uint8)).any()


@pytest.mark.parametrize("rate", list(SPM.RATIOS))
def test_frame_geometry(shim, rate):
    out, inp = SPM.RATIOS[rate]
    first, frames, most = ctypes.c_int64(), ctypes.c_uint32(), ctypes.c_uint32()
    big = (1 << 32) // (inp * B // out) + 3                           # a buffer past 2^32 input samples
    for b in (0, 1, 4, big, big + 1):
        assert shim.shim_geometry(out, inp, b, ctypes.byref(first), ctypes.byref(frames), ctypes.byref(most)) == 0
        assert first.value == inp * b * B // out == SPM.first_sample(rate, b)
        assert frames.value == SPM.frames(rate, b) == {1: 512, 2: 1024, 3: 1536, 4: 2048, 5: 2560, 6: 614}[inp]
        assert most.value >= frames.value
    assert SPM.first_sample(rate, big) >= 1 << 32


def test_record_restatement():
    """SPM.record: the frames start at s_b, the remainder is not read, samples past the end are 0."""
    x = np.zeros((3 * 157287, 2), np.int64)
    b = 1
    s0 = SPM.first_sample(2_400_000, b)
    x[s0: s0 + N] = np.stack([np.full(N, 50), np.zeros(N)], axis=1)     # frame 0 of buffer 1 only
    r = SPM.record(x, 2_400_000, b)
    assert r["frames"] == 614 and r["buffer"] == 1
    assert np.array_equal(r["power"], SPM.frame_power(x[s0: s0 + N][None])[0])
    x[s0 + 614 * N: SPM.first_sample(2_400_000, b + 1)] = 90           # the unmeasured remainder
    assert np.array_equal(SPM.record(x, 2_400_000, b)["power"], r["power"])
    assert not SPM.record(x[:10], 2_000_000, 0)["power"].any()        # past the end: zero


def _records(power_by_bin, frames=512, n=1):
    r = np.zeros(n, dtype=api.SPECTRUM_DTYPE)
    r["frames"] = frames
    r["power"][:] = power_by_bin
    return r


def test_spectrum_summary():
    flat = np.full(N, 1000, np.uint64)
    s = api.spectrum_summary(_records(flat, n=2), 10_000_000)
    assert s["buffers"] == 2 and s["frames"] == 1024
    assert s["freq_hz"][128] == 0 and s["freq_hz"][0] == -5_000_000 and s["freq_hz"][1] == -5_000_000 + 39062.5
    assert s["floor_db"] == pytest.approx(10 * np.log10(2000 / 1024)) and s["dc_excess_db"] == 0.0
    p = flat.copy()
    p[128] = 1000 * 100                                                 # a DC spike, 20 dB: reported, not a band
    p[128 + 51: 128 + 51 + 20] = 10 ** 6                                # energy around +2 MHz at 10 MS/s
    s = api.spectrum_summary(_records(p), 10_000_000)
    assert s["dc_excess_db"] == pytest.approx(20.0)
    w = 256 * 2_000_000 // 10_000_000
    assert abs(s["band_offset_hz"] - 2_000_000) <= 10_000_000 / 256 * (w / 2)
    assert s["band_offset_hz"] == (128 + 51 + 20 - w + (w - 1) / 2 - 128) * 10_000_000 / 256   # the lowest best band
    # 2 MHz: the band is the whole spectrum; no frames: nothing derived
    assert api.spectrum_summary(_records(p), 2_000_000)["band_offset_hz"] == -0.5 * 2_000_000 / 256
    e = api.spectrum_summary(np.zeros(0, dtype=api.SPECTRUM_DTYPE), 2_400_000)
    assert e["frames"] == 0 and e["power_db"] is None and e["band_offset_hz"] is None
    with pytest.raises(ValueError):
        api.spectrum_summary(_records(p), 3_000_000)


def _dc_capture(seed=3, n_aircraft=12):
    """10 MS/s SC16 traffic sent 2 MHz above the baseband's 0 Hz with a DC spike."""
    x, _ = synth.fleet_at_rate(30, 700, seed, sample_rate=10_000_000, n_aircraft=n_aircraft, dtype="sc16",
                               scale=256.0, carrier_hz=2_000_000, dc=(9.0, -6.0), period=600)
    return x


def test_summary_of_an_off_centre_capture():
    """The model's records of the CLI's capture: the DC bin stands out and the channel is found at +2 MHz."""
    x = _dc_capture()
    recs = SPM.expected(x, 10_000_000, "sc16")
    s = api.spectrum_summary(recs, 10_000_000)
    assert s["dc_excess_db"] > 10
    assert abs(s["band_offset_hz"] - 2_000_000) <= 10_000_000 / 256


def test_setters_refuse_without_a_device():
    L = api.lib()
    assert L.modes_set_spectrum(None, 1) == -1
    assert L.modes_take_spectra(None, None, 0) == 0
    assert L.modes_pool_set_spectrum(None, 1) == -1
    assert L.modes_pool_take_spectra(None, 0, None, 0) == 0
    assert "modes_set_spectrum" in api.EXPORTS and "modes_pool_take_spectra" in api.EXPORTS


# ---------------------------------------------------------------- GPU


def assert_spectra(got, want, what=""):
    assert got.dtype == api.SPECTRUM_DTYPE
    assert got.size == want.size, (what, got.size, want.size)
    assert np.array_equal(got["buffer"], want["buffer"]), what
    assert np.array_equal(got["frames"], want["frames"]), what
    bad = np.flatnonzero((got["power"] != want["power"]).any(axis=1))
    assert bad.size == 0, f"{what}: power differs in buffers {bad[:5].tolist()}"


def _stream(rate, fmt, n_buffers=2.6, seed=5, carrier=0.0, dc=None):
    """Traffic at the rate and format, n_buffers 2 MHz buffers long (a partial last one)."""
    period = 400
    nframes = int(n_buffers * B / period)
    x, _ = synth.fleet_at_rate(25, nframes, seed, sample_rate=rate, n_aircraft=10, dtype="uc8" if fmt == "uc8" else "sc16",
                               scale={"uc8": 1.0, "sc16": 256.0, "sc16q11": 16.0}[fmt], carrier_hz=carrier, dc=dc,
                               period=period)
    return x


PATHS = [(2_000_000, "uc8", 0), (2_000_000, "sc16", 0), (2_000_000, "sc16q11", 0), (2_400_000, "uc8", 0),
         (2_400_000, "sc16", 0)] + [(2_000_000 * m, fmt, o) for m, fmt in ((2, "uc8"), (3, "sc16q11"), (4, "sc16"), (5, "uc8"))
                                    for o in (0, (m - 1) * 1_000_000 - 123_457)]


@pytest.mark.gpu
@pytest.mark.parametrize("rate,fmt,offset", PATHS)
def test_decode_paths_equal_model(rate, fmt, offset, gpu_decoder_factory):
    """Every rate and format, with and without an input offset: whole, in chunks that cut buffers, both EOF
    modes, and small batches over both slots; the EOF buffer has a record iff it has a level record."""
    x = _stream(rate, fmt, carrier=offset / 2, dc=(3.0, -2.0))
    for drop in (0, 1):
        want = SPM.expected(x, rate, fmt, drop_eof=drop)
        for chunk, mbb in ((None, 0), (100003, BUF), (777777, 2 * BUF)):
            dec = gpu_decoder_factory(spectrum=True, levels=True, input_rate=rate, input_format=fmt, input_offset=offset,
                                      drop_eof_buffer=drop, max_batch_bytes=mbb)
            dec.decode(x, chunk=chunk)
            got = dec.take_spectra()
            assert_spectra(got, want, f"{rate} {fmt} {offset} drop={drop} chunk={chunk}")
            assert np.array_equal(dec.take_levels()["buffer"], got["buffer"])
            assert dec.take_spectra().size == 0


@pytest.mark.gpu
def test_switch_leaves_the_decode_alone(gpu_decoder_factory, checker_libs):
    """Messages, statistics and level records with the switch on equal those with it off, on every path;
    exactly one more launch per batch with it on, and the plain two launches per batch with it off."""
    data = np.concatenate([synth.random_traffic(B * 5 + 777, 1500, 41, n_aircraft=14), np.full(300001, 255, np.uint8)])
    want = SPM.expected(data)
    for extra in (dict(), dict(signal=True), dict(gpu_resolve=1), dict(n_gpus=2), dict(check_crc=0, aggressive=1),
                  dict(recover=True, weak_preambles=True)):
        off = gpu_decoder_factory(levels=True, max_batch_bytes=BUF, **extra)
        on = gpu_decoder_factory(levels=True, spectrum=True, max_batch_bytes=BUF, **extra)
        m_off, m_on = off.decode(data), on.decode(data)
        assert len(m_off) > 100
        assert [bytes(m.copy()) for m in m_on] == [bytes(m.copy()) for m in m_off], extra
        assert on.stats() == off.stats(), extra
        assert np.array_equal(on.take_levels(), off.take_levels()), extra
        assert on.launch_count() - off.launch_count() == want.size, extra      # one batch per buffer here
        assert_spectra(on.take_spectra(), want, str(extra))
        assert off.take_spectra().size == 0
    plain = gpu_decoder_factory(max_batch_bytes=BUF)
    plain.decode(data)
    assert plain.launch_count() == 2 * want.size


@pytest.mark.gpu
def test_spectra_on_every_path(gpu_decoder_factory):
    """Two GPU shards (one GPU reused) at 2 MHz and 10 MS/s SC16, a reset mid-stream, the switch turned on
    between batches, and partial takes."""
    x = _stream(10_000_000, "sc16", n_buffers=3.3, seed=8)
    want = SPM.expected(x, 10_000_000, "sc16")
    for batch in (1, 2):
        d = gpu_decoder_factory(spectrum=True, n_gpus=2, max_batch_bytes=batch * BUF, input_rate=10_000_000,
                                input_format="sc16")
        d.decode(x, chunk=1_000_003)
        assert_spectra(d.take_spectra(), want, f"n_gpus=2 batch={batch}")
    data = synth.random_traffic(B * 4 + 99, 900, 31)
    w2 = SPM.expected(data)
    d = gpu_decoder_factory(spectrum=True, max_batch_bytes=BUF)
    d.process(data[: 2 * BUF])
    d.reset()
    assert d.take_spectra().size == 0
    d.decode(data, chunk=300001)
    assert_spectra(d.take_spectra(), w2, "after reset")
    d = gpu_decoder_factory(max_batch_bytes=BUF)
    d.reset()
    d.process(data[: 2 * BUF])
    d.set_spectrum(True)
    d.process(data[2 * BUF:])
    d.finish()
    assert_spectra(d.take_spectra(), w2[2:], "switched on")
    d = gpu_decoder_factory(spectrum=True)
    d.decode(data)
    first = np.zeros(2, dtype=api.SPECTRUM_DTYPE)
    assert api.lib().modes_take_spectra(d._h, first.ctypes.data, 2) == 2
    assert_spectra(np.concatenate([first, d.take_spectra()]), w2, "partial takes")


PINNED = 64 << 20


@pytest.mark.gpu
@pytest.mark.parametrize("rate,fmt", [(2_000_000, "uc8"), (10_000_000, "sc16")])
def test_after_silent_prefix(rate, fmt):
    """A silent prefix that carries the input past 2^32 samples, then traffic: the prefix's records are silent,
    and the traffic's are its own, re-indexed."""
    m = rate // 2_000_000
    bps = 2 if fmt == "uc8" else 4
    x = _stream(rate, fmt, n_buffers=2.2, seed=12)
    own = SPM.expected(x, rate, fmt)
    prefix = 2 ** 32 // (m * B) + 2                                      # 2 MHz buffers
    with api.Decoder(spectrum=True, input_rate=rate, input_format=fmt) as dec:
        dec.reset()
        buf = api.PinnedBuffer(PINNED)
        try:
            buf.array[:] = 127 if fmt == "uc8" else 0
            left = prefix * B * m * bps
            while left:
                n = min(PINNED, left)
                dec.process_ptr(buf.ptr, n)
                left -= n
        finally:
            buf.free()
        for off in range(0, x.size, 1_000_003):
            dec.process(x[off: off + 1_000_003])
        dec.finish()
        got = dec.take_spectra()
    assert got.size == prefix + own.size
    assert list(got["buffer"][:prefix]) == list(range(prefix)) and not got["power"][:prefix].any()
    assert (got["frames"][:prefix] == 512 * m).all()
    own["buffer"] += prefix
    assert_spectra(got[prefix:], own, f"{rate} {fmt} after the prefix")


def _schedule(rng, n_rx, n_buf, max_batch):
    left, calls = [n_buf] * n_rx, []
    while any(left):
        ids = [r for r in range(n_rx) if left[r] and rng.random() < 0.7]
        rng.shuffle(ids)
        ids = ids[:max_batch]
        for r in ids:
            left[r] -= 1
        if ids:
            calls.append(ids)
    return calls


@pytest.mark.gpu
def test_pool_spectra(gpu_decoder_factory):
    """2 MHz, 2.4 MS/s and 16-bit receivers out of lock step, through ingest and with two batches in flight,
    an idle call (a 2.4 MS/s receiver alone in its first call) and a reset: each receiver's records equal
    the single-stream decoder's for its first buffers(r) buffers.  Messages equal the pool's without spectra."""
    kinds = [(2_000_000, "uc8"), (2_400_000, "uc8"), (2_000_000, "sc16"), (2_400_000, "sc16q11"), (2_000_000, "uc8")]
    n_buf = 4
    streams = []
    for r, (rate, fmt) in enumerate(kinds):
        x = _stream(rate, fmt, n_buffers=n_buf * 1.3, seed=40 + r)
        nb = BUF * (1 if fmt == "uc8" else 2)
        streams.append(np.resize(x, n_buf * nb))
    single = []
    for (rate, fmt), x in zip(kinds, streams):
        d = gpu_decoder_factory(spectrum=True, input_rate=rate, input_format=fmt)
        d.decode(x)
        single.append(d.take_spectra())
    msgs_plain = {}
    for spectrum in (False, True):
        with api.ReceiverPool(len(kinds), max_batch=3, spectrum=spectrum) as pool:
            for r, (rate, fmt) in enumerate(kinds):
                pool.set_input_rate(r, rate)
                pool.set_input_format(r, fmt)
            for overlap in (False, True):
                nxt = [0] * len(kinds)
                in_flight = 0
                calls = [[1]] + _schedule(np.random.default_rng(3 + overlap), len(kinds), n_buf, 3)
                left = [n_buf] * len(kinds)
                for ids in calls:
                    ids = [r for r in ids if left[r]]
                    if not ids:
                        continue
                    for r in ids:
                        left[r] -= 1
                    bufs = []
                    for r in ids:
                        nb = BUF * (1 if kinds[r][1] == "uc8" else 2)
                        bufs.append(streams[r][nxt[r] * nb: (nxt[r] + 1) * nb])
                        nxt[r] += 1
                    if not overlap:
                        pool.ingest(ids, bufs)
                        continue
                    pool.submit(ids, bufs)
                    in_flight += 1
                    if in_flight == 2:
                        pool.collect()
                        in_flight -= 1
                if in_flight:
                    pool.collect()
                for r in range(len(kinds)):
                    msgs = [bytes(m.copy()) for m in pool.take(r)]
                    got = pool.take_spectra(r)
                    if spectrum:
                        assert msgs == msgs_plain[(overlap, r)]
                        nb = pool.buffers(r)
                        assert nb >= 2
                        assert_spectra(got, single[r][:nb], f"overlap={overlap} receiver {r} {kinds[r]}")
                    else:
                        msgs_plain[(overlap, r)] = msgs
                        assert got.size == 0
                    if r == 4 and spectrum and not overlap:
                        pool.reset(r)
                        assert pool.take_spectra(r).size == 0
                    pool.reset(r)


def _parse(err: str) -> dict:
    m = re.search(r"spectrum: (\d+) buffers, (\d+) frames, floor (\S+) dB, DC (\S+) dB over its neighbours, "
                  r"strongest 2 MHz band at (\S+) Hz", err)
    assert m, err
    return dict(buffers=int(m[1]), frames=int(m[2]), floor_db=float(m[3]), dc_excess_db=float(m[4]),
                band_offset_hz=float(m[5]))


@pytest.mark.gpu
def test_c_host_spectrum(tmp_path):
    """./dump1090-b200 --spectrum on a 10 MS/s SC16 capture tuned 2 MHz off 1090 MHz with a DC spike reports
    the DC spike and the channel at +2 MHz, as spectrum_summary of the model's records says; stdout equals
    the run without the flag, with and without the offset that decodes it."""
    x = _dc_capture()
    f = tmp_path / "off_centre.sc16"
    f.write_bytes(x.tobytes())
    s = api.spectrum_summary(SPM.expected(x, 10_000_000, "sc16"), 10_000_000)
    exe = str(ROOT / "dump1090-b200")
    base = [exe, "--ifile", str(f), "--sample-rate", "10000000", "--iformat", "SC16"]
    for extra in ((), ("--input-offset", "2000000"), ("--raw", "--input-offset", "2000000")):
        plain = subprocess.run(base + list(extra), capture_output=True, check=True)
        sp = subprocess.run(base + list(extra) + ["--spectrum"], capture_output=True, check=True)
        assert sp.stdout == plain.stdout, extra
        assert b"spectrum: " not in plain.stderr
        got = _parse(sp.stderr.decode())
        assert (got["buffers"], got["frames"]) == (s["buffers"], s["frames"])
        assert abs(got["floor_db"] - s["floor_db"]) <= 0.0051 and abs(got["dc_excess_db"] - s["dc_excess_db"]) <= 0.0051
        assert got["band_offset_hz"] == pytest.approx(s["band_offset_hz"], abs=0.51)
        assert got["dc_excess_db"] > 10
        assert abs(got["band_offset_hz"] - 2_000_000) <= 10_000_000 / 256
    assert len(subprocess.run(base + ["--input-offset", "2000000"], capture_output=True, check=True).stdout) > 0
