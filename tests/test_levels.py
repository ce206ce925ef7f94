"""Receiver levels per buffer (modes_set_levels, modes_levels_device, modes_pool_set_levels): noise,
peak and clipping sums of every decoded reference buffer.

The reference computation is a numpy restatement of the definition, from the raw stream bytes: for
each buffer the decode processes, over its own samples (the 238 it carries over belong to the buffer
before it; the EOF buffer's 127-padding has magnitude 0 and is never clipped),
    n_samples = stream samples in it (a trailing odd byte counts), clipped = samples with an I or Q
    byte of 0 or 255, sum_mag = sum m, sum_power = sum m^2, peak = max m
with m = the reference's magnitude round(360 * sqrt((I-127)^2 + (Q-127)^2)) (dump1090.c:359-364).
CPU tests cover the arithmetic (host build of modes_levels_core.cuh) and level_summary; GPU tests the
kernel on every decode path, the pool and the C host."""
import ctypes
import math
import re
import subprocess

import numpy as np
import pytest

import checker as C
import edge_corpora as E
import streams as S
from dump1090_b200 import api, synth

ROOT = C.ROOT
SHIM = ROOT / "tests" / "_build" / "liblevels_core_host.so"
BUF = api.BUFFER_BYTES
KERNEL_THREADS = 512                      # partial sums per buffer in modes_levels.cu

# ---------------------------------------------------------------- the restatement


def _mag_table():
    """round(360 * sqrt(i*i + q*q)) for i, q in 0..128, as the reference builds it (dump1090.c:359-364)."""
    i, q = np.meshgrid(np.arange(129), np.arange(129), indexing="ij")
    return np.floor(np.sqrt((i * i + q * q).astype(np.float64)) * 360 + 0.5).astype(np.int64)


MAG = _mag_table()


def buffer_sums(iq) -> tuple:
    """(clipped, sum_mag, sum_power, peak) of I/Q bytes."""
    b = np.asarray(iq, dtype=np.uint8).reshape(-1, 2)
    a = np.abs(b.astype(np.int64) - 127)
    m = MAG[a[:, 0], a[:, 1]]
    clipped = int(((b == 0) | (b == 255)).any(axis=1).sum())
    return clipped, int(m.sum()), int((m * m).sum()), int(m.max()) if m.size else 0


def expected_levels(data, drop_eof=0) -> np.ndarray:
    """The records a streaming decode of `data` gives: one per whole buffer, then the EOF buffer
    (the rest of the stream, 127-padded) unless it is dropped."""
    data = np.asarray(data, dtype=np.uint8)
    whole = data.size // BUF
    n = whole + (0 if drop_eof else 1)
    out = np.zeros(n, dtype=api.LEVEL_DTYPE)
    for k in range(n):
        chunk = data[k * BUF: (k + 1) * BUF]
        out[k]["buffer"] = k
        out[k]["n_samples"] = (chunk.size + 1) // 2
        padded = np.full(BUF, 127, dtype=np.uint8)
        padded[: chunk.size] = chunk
        out[k]["clipped"], out[k]["sum_mag"], out[k]["sum_power"], out[k]["peak"] = buffer_sums(padded)
    return out


def assert_records(got, want, what=""):
    assert got.dtype == api.LEVEL_DTYPE
    assert got.size == want.size, (what, got.size, want.size)
    for f in ("buffer", "n_samples", "clipped", "sum_mag", "sum_power", "peak", "pad"):
        bad = np.flatnonzero(got[f] != want[f])
        assert bad.size == 0, f"{what}: field {f} differs at buffers {bad[:5].tolist()}: got {got[f][bad[:3]]} want {want[f][bad[:3]]}"


# ---------------------------------------------------------------- CPU: arithmetic


@pytest.fixture(scope="module")
def shim():
    subprocess.run(["make", "-s", "shim"], cwd=ROOT, check=True)
    lib = ctypes.CDLL(str(SHIM))
    lib.shim_levels.restype = ctypes.c_int
    lib.shim_levels.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_uint32, ctypes.c_void_p]
    return lib


_buffers = E.level_buffers


def _shim_sums(shim, buf, threads=KERNEL_THREADS):
    out = np.zeros(4, dtype=np.uint64)
    buf = np.ascontiguousarray(buf)
    assert shim.shim_levels(buf.ctypes.data, buf.size, threads, out.ctypes.data) == 0
    mag, power, peak, clip = (int(x) for x in out)
    return clip, mag, power, peak


def test_shim_equals_restatement(shim):
    rng = np.random.default_rng(5)
    for name, buf in _buffers(rng):
        assert _shim_sums(shim, buf) == buffer_sums(buf), name
    assert _shim_sums(shim, np.full(BUF, 255, np.uint8)) == (131072, 131072 * 65167, 131072 * 65167 ** 2, 65167)
    assert _shim_sums(shim, np.full(BUF, 127, np.uint8)) == (0, 0, 0, 0)
    assert _shim_sums(shim, next(b for n, b in _buffers(rng) if n == "three_clipped"))[0] == 3
    assert _shim_sums(shim, next(b for n, b in _buffers(rng) if n == "rails_254"))[0] == 0


def test_shim_every_byte_pair(shim):
    """All 65536 (I, Q) pairs, each once, through the host build: the magnitude lookup and the clip
    test of every possible sample."""
    lib = shim
    i, q = np.meshgrid(np.arange(256, dtype=np.uint8), np.arange(256, dtype=np.uint8), indexing="ij")
    pairs = np.stack([i.ravel(), q.ravel()], axis=1).reshape(-1)
    out = np.zeros(4, dtype=np.uint64)
    for k in range(0, 65536, 8):                                          # one 16-byte word at a time
        w = np.ascontiguousarray(pairs[2 * k: 2 * k + 16])
        assert lib.shim_levels(w.ctypes.data, 16, 1, out.ctypes.data) == 0
        clip, mag, power, peak = buffer_sums(w)
        assert (int(out[3]), int(out[0]), int(out[1]), int(out[2])) == (clip, mag, power, peak), k


def test_level_summary():
    r = np.zeros(3, dtype=api.LEVEL_DTYPE)
    r["buffer"] = [0, 1, 2]
    r["n_samples"] = [131072, 131072, 1000]
    r["clipped"] = [0, 5, 1]
    r["sum_power"] = [131072 * 400 ** 2, 131072 * 600 ** 2, 1000 * 500 ** 2]
    r["sum_mag"] = [131072 * 400, 131072 * 600, 1000 * 500]
    r["peak"] = [9000, 65167, 300]
    s = api.level_summary(r)
    n = 2 * 131072 + 1000
    power = 131072 * (400 ** 2 + 600 ** 2) + 1000 * 500 ** 2
    assert s["buffers"] == 3 and s["n_samples"] == n and s["clipped"] == 6
    assert s["noise_dbfs"] == pytest.approx(10 * math.log10(power / n / 65535 ** 2), abs=1e-12)
    assert s["peak_dbfs"] == pytest.approx(20 * math.log10(65167 / 65535), abs=1e-12)
    assert s["clipped_fraction"] == pytest.approx(6 / n, rel=1e-15)
    # full scale: a constant magnitude of 65535 would be 0 dBFS; a sum larger than 64 bits holds
    big = np.zeros(40000, dtype=api.LEVEL_DTYPE)
    big["n_samples"] = 131072
    big["sum_power"] = 131072 * 65167 ** 2
    big["peak"] = 65167
    s = api.level_summary(big)
    assert s["noise_dbfs"] == pytest.approx(20 * math.log10(65167 / 65535), abs=1e-9)
    # silence, and no samples at all
    quiet = np.zeros(2, dtype=api.LEVEL_DTYPE)
    quiet["n_samples"] = 131072
    s = api.level_summary(quiet)
    assert s["noise_dbfs"] == -math.inf and s["peak_dbfs"] == -math.inf and s["clipped_fraction"] == 0.0
    for empty in (np.zeros(0, dtype=api.LEVEL_DTYPE), np.zeros(1, dtype=api.LEVEL_DTYPE)):
        s = api.level_summary(empty)
        assert s["n_samples"] == 0 and s["noise_dbfs"] is None and s["peak_dbfs"] is None and s["clipped_fraction"] is None
        assert s["buffers"] == empty.size


def test_restatement_of_a_stream():
    """expected_levels itself: buffer split, EOF padding, a trailing odd byte."""
    data = np.full(BUF + 5, 200, dtype=np.uint8)
    data[-1] = 0
    e = expected_levels(data)
    assert e["buffer"].tolist() == [0, 1] and e["n_samples"].tolist() == [131072, 3]
    assert e["clipped"].tolist() == [0, 1]
    m = int(MAG[73, 73])
    assert e["sum_mag"][1] == 2 * m + int(MAG[127, 0]) and e["peak"][1] == max(m, int(MAG[127, 0]))
    assert expected_levels(data, drop_eof=1).size == 1
    assert expected_levels(data[:BUF])["n_samples"].tolist() == [131072, 0]


# ---------------------------------------------------------------- GPU


def _saturated(seed=4):
    """Traffic at far too much gain: I and Q scaled 8x around 127 and clipped to the rails."""
    d = synth.random_traffic(131072 * 3 + 999, 500, seed).astype(np.int64)
    return np.clip((d - 127) * 8 + 127, 0, 255).astype(np.uint8)


def _gpu_streams():
    yield "modes1_head", C.modes1()
    yield "traffic", synth.random_traffic(131072 * 4 + 12345, 900, 31)
    yield "ties", S.tie_rich(11)
    yield "saturated", _saturated()
    for k, (case, levels, data) in enumerate(S.random_alphabet_cases(n_cases=3)):
        yield f"alphabet{k}", data
    yield "silent", np.full(BUF * 2 + 7, 127, dtype=np.uint8)
    yield "odd_tail", synth.random_traffic(131072 * 2, 300, 8)[: 2 * BUF + 1]
    yield "whole_buffers", synth.random_traffic(131072 * 2, 300, 9)                     # all-padding EOF buffer


GPU_STREAMS = dict(_gpu_streams())


def raw_bytes(m) -> bytes:
    return bytes(m.copy())


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(GPU_STREAMS))
def test_decode_levels_equal_restatement(name, gpu_decoder_factory, checker_libs):
    data = GPU_STREAMS[name]
    for drop in (0, 1):
        want = expected_levels(data, drop)
        for mbb in (0, BUF, 3 * BUF):                                    # one batch, and many batches over both slots
            dec = gpu_decoder_factory(levels=True, drop_eof_buffer=drop, max_batch_bytes=mbb)
            dec.decode(data)
            assert_records(dec.take_levels(), want, f"{name} drop={drop} batch={mbb}")
            assert dec.take_levels().size == 0                            # taken means gone
        for chunk in (4097, 262145, 100001):                              # ragged feeding, odd sizes
            dec = gpu_decoder_factory(levels=True, drop_eof_buffer=drop, max_batch_bytes=2 * BUF)
            dec.decode(data, chunk=chunk)
            assert_records(dec.take_levels(), want, f"{name} drop={drop} chunk={chunk}")
    if name == "saturated":
        assert want["clipped"].sum() > 10000
    if name == "silent":
        assert not want["sum_power"].any()


@pytest.mark.gpu
def test_levels_leave_messages_and_statistics_alone(gpu_decoder_factory, checker_libs):
    """Messages (raw bytes, signal included) and statistics with levels on equal those with levels
    off, with the signal pass on and off, on every decode path; one more launch per batch."""
    # traffic, then a block stuck at the rails (clipped, and no preamble in it)
    data = np.concatenate([synth.random_traffic(131072 * 5 + 777, 1500, 41, n_aircraft=14), np.full(300001, 255, np.uint8)])
    want = expected_levels(data)
    for extra in (dict(), dict(signal=True), dict(gpu_resolve=1), dict(signal=True, gpu_resolve=1),
                  dict(n_gpus=2), dict(signal=True, n_gpus=2), dict(check_crc=0, aggressive=1)):
        off = gpu_decoder_factory(max_batch_bytes=BUF, **extra)
        on = gpu_decoder_factory(levels=True, max_batch_bytes=BUF, **extra)
        m_off, m_on = off.decode(data), on.decode(data)
        assert len(m_off) > 100
        assert [raw_bytes(m) for m in m_on] == [raw_bytes(m) for m in m_off], extra
        assert on.stats() == off.stats(), extra
        assert on.launch_count() - off.launch_count() == want.size, extra    # one batch per buffer here
        assert_records(on.take_levels(), want, str(extra))
        assert off.take_levels().size == 0


@pytest.mark.gpu
def test_levels_on_every_path(gpu_decoder_factory, checker_libs):
    """n_gpus = 2 (one GPU reused round-robin) with batches of 1 and 3 buffers, the device resolve,
    a reset in the middle of a stream, and the switch changed between batches."""
    data = np.concatenate([synth.random_traffic(131072 * 6 + 4321, 1800, 93, n_aircraft=16), _saturated(7)])
    want = expected_levels(data)
    for drop in (0, 1):
        for batch in (1, 3):
            multi = gpu_decoder_factory(levels=True, n_gpus=2, max_batch_bytes=batch * BUF, drop_eof_buffer=drop)
            multi.decode(data, chunk=300001)
            assert_records(multi.take_levels(), expected_levels(data, drop), f"n_gpus=2 batch={batch} drop={drop}")
        gres = gpu_decoder_factory(levels=True, gpu_resolve=1, max_batch_bytes=2 * BUF, drop_eof_buffer=drop)
        gres.decode(data)
        assert_records(gres.take_levels(), expected_levels(data, drop), f"gpu_resolve drop={drop}")
    # reset mid-stream: the queued records go, the new stream counts from buffer 0
    dec = gpu_decoder_factory(levels=True, max_batch_bytes=BUF)
    dec.reset()
    dec.process(_saturated(8))
    assert dec.take_levels().size == 3
    dec.process(_saturated(8))
    dec.reset()
    assert dec.take_levels().size == 0
    dec.decode(data, chunk=777777)
    assert_records(dec.take_levels(), want, "after reset")
    # switched on after two buffers: records from the third buffer on
    dec = gpu_decoder_factory(max_batch_bytes=BUF)
    dec.reset()
    dec.process(data[: 2 * BUF])
    dec.set_levels(True)
    dec.process(data[2 * BUF:])
    dec.finish()
    assert_records(dec.take_levels(), want[2:], "switched on")
    # partial takes drain oldest first
    dec = gpu_decoder_factory(levels=True)
    dec.decode(data)
    n = int(api.lib().modes_take_levels(dec._h, None, 0))
    assert n == want.size
    first = np.zeros(3, dtype=api.LEVEL_DTYPE)
    assert api.lib().modes_take_levels(dec._h, first.ctypes.data, 3) == 3
    assert_records(np.concatenate([first, dec.take_levels()]), want, "partial takes")


def _periodic(period_pattern, nsamples, amp=100):
    """I/Q stream whose magnitude repeats `period_pattern` (1 = pulse, 0 = silence)."""
    pat = np.array(period_pattern, dtype=np.uint8)
    hi = np.tile(pat, -(-nsamples // pat.size))[:nsamples]
    out = np.full(2 * nsamples, 127, dtype=np.uint8)
    out[0::2] = 127 + amp * hi
    return out


@pytest.mark.gpu
def test_levels_after_a_repeated_batch(gpu_decoder_factory, checker_libs):
    """A stream dense enough to overflow the candidate buffers (more than one candidate per 64
    samples) makes the decode repeat the batch with larger buffers; the records stay the same."""
    data = np.concatenate([_periodic([1, 0, 1, 0, 0, 0, 0, 1, 0, 1, 0, 0, 0, 0, 0], 131072 * 2 + 5000),
                           synth.random_traffic(131072 + 3, 200, 12)])
    want = expected_levels(data)
    plain = gpu_decoder_factory(check_crc=0, max_batch_bytes=BUF)
    on = gpu_decoder_factory(check_crc=0, levels=True, max_batch_bytes=BUF)
    m_plain, m_on = plain.decode(data), on.decode(data)
    assert [raw_bytes(m) for m in m_on] == [raw_bytes(m) for m in m_plain]
    # every batch is one buffer: 2 launches each, 3 with levels, and the repeats on top
    assert plain.launch_count() > 2 * want.size, "no batch was repeated"
    assert on.launch_count() - plain.launch_count() > want.size
    assert_records(on.take_levels(), want, "repeated batch")


@pytest.mark.gpu
def test_levels_device_stage_level(gpu_decoder_factory, checker_libs):
    """modes_levels_device over buffers in HBM, contiguous and at a stride (the pool's layout)."""
    import torch
    rng = np.random.default_rng(3)
    bufs = [rng.integers(0, 256, BUF, dtype=np.uint8), np.full(BUF, 255, np.uint8), np.full(BUF, 127, np.uint8),
            synth.random_traffic(131072, 200, 5), _saturated(9)[:BUF]]
    want = np.zeros(len(bufs), dtype=api.LEVEL_DTYPE)
    for k, b in enumerate(bufs):
        want[k]["buffer"], want[k]["n_samples"] = k, 131072
        want[k]["clipped"], want[k]["sum_mag"], want[k]["sum_power"], want[k]["peak"] = buffer_sums(b)
    dec = gpu_decoder_factory(levels=True)                                # the streaming switch does not matter here
    flat = torch.from_numpy(np.concatenate(bufs)).cuda()
    launches = dec.launch_count()
    dec.levels_device(flat.data_ptr(), len(bufs))
    assert_records(dec.levels_fetch(), want, "contiguous")
    assert dec.launch_count() - launches == 1
    strided = np.full(2 * len(bufs) * BUF, 0, dtype=np.uint8)             # pads on the rail: would count as clipped
    for k, b in enumerate(bufs):
        strided[(2 * k + 1) * BUF: (2 * k + 2) * BUF] = b
    d = torch.from_numpy(strided).cuda()
    dec.levels_device(d.data_ptr() + BUF, len(bufs), 2 * BUF)
    assert_records(dec.levels_fetch(), want, "stride 2")
    dec.levels_device(d.data_ptr() + 3 * BUF, 2, 4 * BUF)
    assert_records(dec.levels_fetch(), np.array([(0, *want[1].tolist()[1:]), (1, *want[3].tolist()[1:])],
                                                dtype=api.LEVEL_DTYPE), "stride 4")
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        dec.levels_device(d.data_ptr() + 8, 1)
    assert dec.take_levels().size == 0                                    # the stage level queues nothing


def _schedule(rng, n_rx, n_buf, max_batch):
    """Which receivers deliver a buffer in which call: every receiver n_buf times, not in lock step."""
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
def test_pool_levels(gpu_decoder_factory, checker_libs):
    """Five receivers, not in lock step, through ingest and through submit/collect with two batches in
    flight: each receiver's records equal the restatement of its own buffers (own buffer indices; the
    pad buffers, which hold the carries, are never counted).  Messages equal the pool's without levels."""
    n_rx, n_buf = 5, 3
    streams = [synth.random_traffic(n_buf * 131072, 120 * n_buf + 37 * r, seed=500 + r) for r in range(n_rx)]
    streams[1] = _saturated(10)[: n_buf * BUF]                           # overloaded
    streams[2] = np.full(n_buf * BUF, 127, dtype=np.uint8)                # dead
    streams[3] = np.full(n_buf * BUF, 255, dtype=np.uint8)                # stuck at the rail
    want = [expected_levels(s, drop_eof=1) for s in streams]
    msgs_plain = {}
    for levels in (False, True):
        with api.ReceiverPool(n_rx, max_batch=4, levels=levels) as pool:
            for overlap in (False, True):
                nxt = [0] * n_rx
                in_flight = 0
                for ids in _schedule(np.random.default_rng(8 + overlap), n_rx, n_buf, 4):
                    bufs = [streams[r][nxt[r] * BUF: (nxt[r] + 1) * BUF] for r in ids]
                    for r in ids:
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
                for r in range(n_rx):
                    msgs = [raw_bytes(m) for m in pool.take(r)]
                    if levels:
                        assert msgs == msgs_plain[(overlap, r)]
                        if r == 4 and not overlap:
                            pool.reset(r)                                  # clears its queue
                            assert pool.take_levels(r).size == 0
                        else:
                            assert_records(pool.take_levels(r), want[r], f"overlap={overlap} receiver {r}")
                    else:
                        msgs_plain[(overlap, r)] = msgs
                        assert pool.take_levels(r).size == 0
                    pool.reset(r)
    assert want[1]["clipped"].sum() > 1000 and want[3]["clipped"].sum() == n_buf * 131072


def _parse_levels_line(err: str) -> dict:
    m = re.search(r"levels: (\d+) buffers, (\d+) samples, noise (\S+) dBFS, peak (\S+) dBFS, clipped (\d+) \((\S+)\)", err)
    assert m, err
    return dict(buffers=int(m[1]), n_samples=int(m[2]), noise_dbfs=float(m[3]), peak_dbfs=float(m[4]),
                clipped=int(m[5]), clipped_fraction=float(m[6]))


@pytest.mark.gpu
def test_c_host_levels(gpu_decoder_factory, checker_libs, tmp_path):
    """./dump1090-b200 --levels prints on stderr what level_summary gives for the same file, and its
    stdout equals the run without the flag in every output mode."""
    exe = ROOT / "dump1090-b200"
    files = {"modes1": str(C.modes1_path())}
    sat = tmp_path / "saturated.bin"
    sat.write_bytes(_saturated(11).tobytes())
    files["saturated"] = str(sat)
    for name, f in files.items():
        data = np.fromfile(f, dtype=np.uint8)
        for flags in ((), ("--drop-eof-buffer",), ("--gpus", "2", "--chunk", "300000")):
            dec = gpu_decoder_factory(levels=True, drop_eof_buffer=int("--drop-eof-buffer" in flags))
            dec.decode(data)
            recs = dec.take_levels()
            assert_records(recs, expected_levels(data, int("--drop-eof-buffer" in flags)), name)
            s = api.level_summary(recs)
            r = subprocess.run([str(exe), "--ifile", f, "--levels", *flags], capture_output=True, check=True, text=True)
            got = _parse_levels_line(r.stderr)
            assert (got["buffers"], got["n_samples"], got["clipped"]) == (s["buffers"], s["n_samples"], s["clipped"])
            for k in ("noise_dbfs", "peak_dbfs"):
                assert abs(got[k] - s[k]) <= 0.0051, (k, got[k], s[k])
            assert abs(got["clipped_fraction"] - s["clipped_fraction"]) <= 5.1e-7
        for mode in ((), ("--raw",), ("--beast",), ("--stats",), ("--onlyaddr",), ("--sbs",)):
            plain = subprocess.run([str(exe), "--ifile", f, *mode], capture_output=True, check=True)
            lv = subprocess.run([str(exe), "--ifile", f, "--levels", *mode], capture_output=True, check=True)
            assert lv.stdout == plain.stdout, (name, mode)
            assert b"levels: " not in plain.stderr and lv.stderr.decode().count("levels: ") == 1
    assert api.level_summary(expected_levels(_saturated(11)))["clipped"] > 1000
