"""Signal level per message (modes_set_signal) and the Beast binary feed (modes_format_beast).

The reference computation is a numpy restatement of the definition, from the raw stream bytes:
    S = sum_{i < b} max(m[p+16+2i], m[p+17+2i])^2,   signal = isqrt(S // b)
with p = the message's sample_pos, b = its msgbits, m = the reference's magnitudes
(dump1090.c:359-364), and samples outside the stream (before its start, in the EOF padding) of
magnitude 0.  CPU tests cover the arithmetic (host build of modes_signal_core.cuh), the Beast
writer and the host resolve's hand-over of the field; GPU tests the kernel and every decode path."""
import ctypes
import math
import subprocess

import numpy as np
import pytest

import checker as C
import edge_corpora as E
import streams as S
from dump1090_b200 import api, synth

ROOT = C.ROOT
SHIM = ROOT / "tests" / "_build" / "libsignal_core_host.so"
BUF = api.BUFFER_BYTES

# ---------------------------------------------------------------- the restatement


def _mag_table():
    """round(360 * sqrt(i*i + q*q)) for i, q in 0..128, as the reference builds it (dump1090.c:359-364)."""
    i, q = np.meshgrid(np.arange(129), np.arange(129), indexing="ij")
    return np.floor(np.sqrt((i * i + q * q).astype(np.float64)) * 360 + 0.5).astype(np.int64)


MAG = _mag_table()


def magnitudes(iq) -> np.ndarray:
    a = np.abs(np.asarray(iq, dtype=np.uint8).reshape(-1, 2).astype(np.int64) - 127)
    return MAG[a[:, 0], a[:, 1]]


def expected_signal(mag, pos, bits) -> np.ndarray:
    """Signal of frames of `bits` bits whose preamble starts at stream sample `pos` (arrays)."""
    pos = np.asarray(pos, dtype=np.int64)
    bits = np.asarray(bits, dtype=np.int64)
    out = np.zeros(pos.size, dtype=np.int64)
    for b in (56, 112):
        sel = np.flatnonzero(bits == b)
        if not sel.size:
            continue
        idx = pos[sel, None] + 16 + 2 * np.arange(b)[None, :]

        def take(ix):
            ok = (ix >= 0) & (ix < mag.size)
            return np.where(ok, mag[np.clip(ix, 0, mag.size - 1)], 0)

        s = (np.maximum(take(idx), take(idx + 1)) ** 2).sum(axis=1)
        out[sel] = [math.isqrt(int(v) // b) for v in s]
    return out


def beast_level(signal: int) -> int:
    return min(255, (signal * 255 + 32767) // 65535)


def parse_beast(buf: bytes):
    """A small Beast reader: [(type, timestamp, signal byte, frame bytes)]."""
    frames, i = [], 0
    while i < len(buf):
        assert buf[i] == 0x1A, f"no frame start at {i}"
        typ = buf[i + 1]
        i += 2
        n = {0x32: 7, 0x33: 14}[typ]
        payload = bytearray()
        while len(payload) < 7 + n:
            b = buf[i]
            i += 1
            if b == 0x1A:
                assert buf[i] == 0x1A, f"lone 0x1a inside a frame at {i - 1}"
                i += 1
            payload.append(b)
        frames.append((chr(typ), int.from_bytes(payload[:6], "big"), payload[6], bytes(payload[7:])))
    return frames


def raw_bytes(m, zero_signal=False) -> bytes:
    c = m.copy()
    if zero_signal:
        c.signal = 0
    return bytes(c)


# ---------------------------------------------------------------- CPU: arithmetic


@pytest.fixture(scope="module")
def shim():
    subprocess.run(["make", "-s", "shim"], cwd=ROOT, check=True)
    lib = ctypes.CDLL(str(SHIM))
    lib.shim_signal_window.restype = ctypes.c_uint32
    lib.shim_signal_window.argtypes = [ctypes.c_void_p, ctypes.c_uint32]
    lib.shim_signal_of.restype = ctypes.c_uint32
    lib.shim_signal_of.argtypes = [ctypes.c_uint64, ctypes.c_uint32]
    return lib


@pytest.mark.parametrize("bits", [56, 112])
def test_shim_window_equals_restatement(shim, bits):
    rng = np.random.default_rng(bits)
    for name, wins in E.signal_windows(rng):
        for w in wins:
            w = np.ascontiguousarray(w)
            want = expected_signal(magnitudes(w), [-16], [bits])[0]
            assert shim.shim_signal_window(w.ctypes.data, bits) == want, name
    assert shim.shim_signal_window(np.full(448, 127, np.uint8).ctypes.data, bits) == 0
    top = np.full(448, 255, np.uint8)
    assert shim.shim_signal_window(top.ctypes.data, bits) == int(MAG[128, 128]) == 65167


@pytest.mark.parametrize("bits", [56, 112])
def test_shim_isqrt_at_perfect_squares(shim, bits):
    """floor(S / b) at k^2 - 1, k^2, k^2 + 1 for k over the whole range (single-precision estimate
    plus correction), with every remainder S mod b at a few k."""
    ks = np.unique(np.concatenate([np.arange(0, 4096), np.arange(4096, 65168, 7), [46340, 46341, 65535, 65167, 65166]]))
    for k in ks.tolist():
        for x in (k * k - 1, k * k, k * k + 1):
            if x < 0 or x >= 1 << 32:
                continue
            s = x * bits + (k % bits)
            assert shim.shim_signal_of(s, bits) == math.isqrt(x), (k, x)
    for k in (1, 255, 40000, 65167):
        for r in range(bits):
            assert shim.shim_signal_of(k * k * bits + r, bits) == k
            assert shim.shim_signal_of((k * k - 1) * bits + r, bits) == k - 1


# ---------------------------------------------------------------- CPU: Beast writer


def _msg(frame: bytes, sample_pos: int, signal: int) -> api.Message:
    m = api.Message()
    m.msgbits = 8 * len(frame)
    for i, b in enumerate(frame):
        m.msg[i] = b
    m.sample_pos = sample_pos
    m.signal = signal
    return m


def _beast_by_hand(frame, sample_pos, signal):
    ts = 0 if sample_pos < 0 else (6 * sample_pos) % (1 << 48)
    body = bytes([0x33 if len(frame) == 14 else 0x32]) + ts.to_bytes(6, "big") + bytes([beast_level(signal)]) + frame
    return b"\x1a" + body.replace(b"\x1a", b"\x1a\x1a")


BEAST_CASES = [
    ("short", bytes.fromhex("5d4840d6202cc3"), 1000, 30000),
    ("long", bytes.fromhex("8d4840d6202cc371c32ce0576098"), 123456789, 65535),
    ("ts_1a", bytes.fromhex("5d4840d6202cc3"), 47, 100),                              # timestamp 0x00000000011a
    ("ts_all_1a", bytes.fromhex("5d4840d6202cc3"), 0x1A1A1A1A1A1A // 6, 100),           # timestamp 0x1a1a1a1a1a1a
    ("signal_26", bytes.fromhex("5d4840d6202cc3"), 7, 6682),                          # signal byte = 26 = 0x1a
    ("body_1a", bytes.fromhex("8d1a1a1a1a2cc371c32ce057601a"), 99, 4000),
    ("all_1a", bytes([0x1A] * 14), 0x1A1A1A1A1A1A // 6, 6682),
    ("wrap_2_48", bytes.fromhex("5d4840d6202cc3"), (1 << 48) // 6 + 5, 1),            # 6 * pos passes 2^48
    ("wrap_big", bytes.fromhex("8d4840d6202cc371c32ce0576098"), (1 << 50) + 3, 2),
    ("hex_door", bytes.fromhex("5d4840d6202cc3"), -1, 0),
    ("clamped", bytes.fromhex("5d4840d6202cc3"), 5, 70000),
]


@pytest.mark.parametrize("name,frame,pos,signal", BEAST_CASES, ids=[c[0] for c in BEAST_CASES])
def test_format_beast(name, frame, pos, signal):
    m = _msg(frame, pos, signal)
    want = _beast_by_hand(frame, pos, signal)
    got = m.beast()
    assert got == want
    assert len(got) <= 44
    (typ, ts, lvl, body), = parse_beast(got)
    assert typ == ("3" if len(frame) == 14 else "2") and body == frame and lvl == beast_level(signal)
    assert ts == (0 if pos < 0 else (6 * pos) % (1 << 48))
    if name == "signal_26":
        assert lvl == 0x1A
    if name.startswith("ts_"):
        assert b"\x1a" in ts.to_bytes(6, "big")
    if name == "all_1a":
        assert ts == 0x1A1A1A1A1A1A and len(got) == 44
    # length needed / truncation: never more than capacity bytes, no terminator
    L = api.lib()
    for cap in range(len(want) + 2):
        buf = (ctypes.c_uint8 * 64)(*([0xEE] * 64))
        n = L.modes_format_beast(ctypes.byref(m), buf, cap)
        assert n == len(want)
        assert bytes(buf[:min(cap, n)]) == want[:cap] and all(b == 0xEE for b in buf[min(cap, n):])
    assert L.modes_format_beast(ctypes.byref(m), None, 0) == len(want)


def test_beast_round_trip_of_many_frames():
    rng = np.random.default_rng(7)
    msgs, blob = [], b""
    for k in range(500):
        n = 14 if k % 3 else 7
        frame = bytes(rng.choice(np.array([0x1A, 0x00, 0xFF, 0x8D, 0x5D], np.uint8), size=n)) if k % 2 else bytes(rng.integers(0, 256, n, dtype=np.uint8))
        pos = int(rng.integers(-1, 1 << 47))
        sig = int(rng.integers(0, 65536))
        msgs.append((frame, pos, sig))
        blob += _msg(frame, pos, sig).beast()
    got = parse_beast(blob)
    assert [(f[3], f[1], f[2]) for f in got] == [(fr, 0 if p < 0 else (6 * p) % (1 << 48), beast_level(s)) for fr, p, s in msgs]


def test_rssi_dbfs():
    assert _msg(bytes(7), 0, 0).rssi_dbfs() is None
    assert _msg(bytes(7), 0, 65535).rssi_dbfs() == 0.0
    assert abs(_msg(bytes(7), 0, 6554).rssi_dbfs() - 20 * math.log10(6554 / 65535)) < 1e-12


def test_c_host_refuses_beast_with_other_stdout_outputs(tmp_path):
    exe = ROOT / "dump1090-b200"
    assert exe.exists(), "build the C host with `make`"
    f = tmp_path / "empty.bin"
    f.write_bytes(b"")
    for other in ("--raw", "--onlyaddr", "--sbs", "--aircraft-json"):
        r = subprocess.run([str(exe), "--ifile", str(f), "--beast", other], capture_output=True, text=True)
        assert r.returncode == 1 and "--beast" in r.stderr and r.stdout == "", other


# ---------------------------------------------------------------- CPU: host resolve carries the field

FLAGS = [dict(), dict(aggressive=1), dict(fix=0), dict(check_crc=0)]


def _kid(k):
    return "-".join(f"{a}{b}" for a, b in k.items()) or "default"


def _cfg(kw):
    return dict(fix_errors=kw.get("fix", 1), aggressive=kw.get("aggressive", 0), check_crc=kw.get("check_crc", 1))


def _tiled(sel, n_buffers):
    g = (sel["t"] + 2) // api.TILE_SAMPLES
    nt = api.tiles_for(n_buffers)
    cnt = np.bincount(g, minlength=nt).astype(np.uint32)
    t = np.zeros(nt, dtype=api.TILE_DTYPE)
    t["count"] = cnt
    t["offset"] = np.concatenate([[0], np.cumsum(cnt)[:-1]])
    return t


def _records(data, kw):
    recs = C.oracle_scan_candidates(data, fix=kw.get("fix", 1), aggressive=kw.get("aggressive", 0), cap=400000)
    arr = np.frombuffer(b"".join(bytes(c) for c in recs), dtype=api.CANDIDATE_DTYPE).copy()
    # hand-set signals, distinct per candidate and attempt
    rng = np.random.default_rng(arr.size)
    arr["p"]["signal"] = rng.integers(1, 65536, size=(arr.size, 2))
    return arr


def _check_attempts(msgs, index_of, arr, check_crc):
    """Every message carries the signal of the attempt it was delivered from: the retry (pass[1]) for a
    phase-corrected message and for the second message at one position; the first attempt otherwise,
    unless that was not decoded."""
    seen = {}
    counts = {"p0": 0, "p1": 0, "both": 0}
    for m in msgs:
        i = index_of(m)
        c = arr[i]
        nth = seen.get(i, 0)
        seen[i] = nth + 1
        assert nth < 2 and (nth == 0 or check_crc == 0)
        p0_decoded = bool(c["p"]["flags"][0] & api.EVAL_DECODED)
        k = 1 if (nth == 1 or m.phase_corrected or not p0_decoded) else 0
        assert m.signal == int(c["p"]["signal"][k]), (m.sample_pos, nth, k)
        counts["p1" if k else "p0"] += 1
        counts["both"] += nth == 1
    return counts


def _stream():
    return np.concatenate([synth.random_traffic(131072 * 5 + 777, 1600, 41, n_aircraft=14), S.tie_rich(5, n_frames=300)])


@pytest.mark.parametrize("kw", FLAGS, ids=_kid)
def test_host_resolve_delivers_the_attempts_signal(kw, checker_libs):
    data = _stream()
    nbuf = data.size // BUF + 1
    arr = _records(data, kw)
    tiles = _tiled(arr, nbuf)
    pos_to_idx = {int(t) - 238: i for i, t in enumerate(arr["t"])}
    index_of = lambda m: pos_to_idx[int(m.sample_pos)]                          # noqa: E731
    plain = arr.copy()
    plain["p"]["signal"] = 0

    res = api.Resolver(**_cfg(kw))
    res.run(plain, tiles)
    base = res.take_messages()
    res = api.Resolver(**_cfg(kw))
    res.run(arr, tiles)
    one = res.take_messages()
    assert len(one) == len(base) > 100
    assert [raw_bytes(m, True) for m in one] == [raw_bytes(m) for m in base]
    counts = _check_attempts(one, index_of, arr, kw.get("check_crc", 1))
    assert counts["p0"] > 50 and counts["p1"] > 5
    if kw.get("check_crc", 1) == 0:
        assert counts["both"] > 5

    # shards resolved together, and one tentative run + commit per shard: the same messages
    cut = [0, 2, 4, nbuf]
    shards = []
    for a, b in zip(cut[:-1], cut[1:]):
        sel = arr[((arr["t"] >> 17) >= a) & ((arr["t"] >> 17) < b)].copy()
        sel["t"] -= a << 17
        shards.append((sel, _tiled(sel, b - a), a))
    res = api.Resolver(**_cfg(kw))
    res.run_shards(shards)
    assert [raw_bytes(m) for m in res.take_messages()] == [raw_bytes(m) for m in one]
    res = api.Resolver(**_cfg(kw))
    for c, t, b in shards:
        res.run_tentative(c, t, b)
        res.commit()
    assert [raw_bytes(m) for m in res.take_messages()] == [raw_bytes(m) for m in one]


@pytest.mark.parametrize("kw", [dict(), dict(check_crc=0)], ids=_kid)
def test_pool_resolve_delivers_the_attempts_signal(kw, checker_libs):
    n_rx = 4
    streams = [synth.random_traffic(131072, 160 + 20 * r, seed=300 + r) for r in range(n_rx)]
    batch = np.full(2 * n_rx * BUF, 127, dtype=np.uint8)
    for i in range(n_rx):
        batch[(2 * i + 1) * BUF: (2 * i + 2) * BUF] = streams[i]
    arr = _records(batch, kw)
    tiles = _tiled(arr, 2 * n_rx)
    with api.ReceiverPool(n_rx, **_cfg(kw)) as pool:
        pool.resolve(list(range(n_rx)), arr, tiles)
        total = 0
        for r in range(n_rx):
            t0 = 131072 * (2 * r + 1)
            pos_to_idx = {int(t) - t0 - 238: i for i, t in enumerate(arr["t"]) if t0 <= t < t0 + 131072}
            msgs = pool.take(r)
            exp, _ = C.oracle_decode(streams[r], drop_eof=1, **kw)
            assert [m.raw_line() for m in msgs] == [m.hexline() for m in exp]
            counts = _check_attempts(msgs, lambda m: pos_to_idx[int(m.sample_pos)], arr, kw.get("check_crc", 1))
            total += counts["p0"] + counts["p1"]
        assert total > 100


# ---------------------------------------------------------------- GPU


def _seam_and_eof_stream(n_buffers=10, seed=21):
    """Frames whose preamble lies among the 238 samples a buffer carries over from the previous one
    (read from the carry block when a batch starts at that buffer), frames needing the phase-corrected
    retry, frames in the buffer that hits EOF, and frames cut off by EOF (their last bits are padding)."""
    rng = synth.Counter(seed)
    js = [0, 1, 2, 60, 150, 221, 222, 223, 237]
    frames = []
    for k in range(1, n_buffers):
        icao = 0x400000 + rng.below(0x3FFFFF)
        long_frame = synth.make_frame(17, 5, icao.to_bytes(3, "big") + bytes(rng.below(256) for _ in range(7)))
        short_frame = synth.make_frame(11, 5, icao.to_bytes(3, "big"))
        frames.append((131072 * k - 238 + js[(k - 1) % len(js)], long_frame if k % 2 else short_frame, 60.0 + 5 * k, 0.3 * k, 0.0))
        frames.append((131072 * k + 50000, long_frame, 50.0, 0.2 * k, 0.35))
    nsamples = 131072 * n_buffers + 3000
    for k, p in enumerate((131072 * n_buffers + 400, 131072 * n_buffers + 1500, nsamples - 150, nsamples - 40)):
        frames.append((p, synth.make_frame(17, 5, (0x500000 + k).to_bytes(3, "big") + bytes(7)), 70.0, 0.5, 0.0))
    return synth.synth_stream(nsamples, frames, sigma=1.2, seed=seed)


def _gpu_streams():
    yield "modes1", C.modes1()
    for seed in (1, 2, 3):
        yield f"traffic{seed}", synth.random_traffic(300000, 400, seed)
    yield "ties", S.tie_rich(11)
    yield "ties_weak", S.tie_rich(12, levels=(0, 0, 1, 3, 30))
    yield "retry_at_j0", S.retry_at_buffer_start()
    yield "seam_and_eof", _seam_and_eof_stream()


GPU_STREAMS = dict(_gpu_streams())


def _assert_signals(msgs, data):
    mag = magnitudes(data)
    want = expected_signal(mag, [m.sample_pos for m in msgs], [m.msgbits for m in msgs])
    got = np.array([m.signal for m in msgs], dtype=np.int64)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{bad.size} of {got.size} differ, first: pos {msgs[bad[0]].sample_pos} got {got[bad[0]]} want {want[bad[0]]}"
    assert np.all(got > 0)


def _decode_on_off(data, kw, factory, **extra):
    off = factory(**_cfg(kw), **extra)
    on = factory(signal=True, **_cfg(kw), **extra)
    got_off, got_on = off.decode(data), on.decode(data)
    assert [raw_bytes(m, True) for m in got_on] == [raw_bytes(m) for m in got_off]
    assert all(m.signal == 0 for m in got_off)
    assert on.stats() == off.stats()
    return got_on


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(GPU_STREAMS))
@pytest.mark.parametrize("kw", FLAGS, ids=_kid)
def test_decode_signal_equals_restatement(name, kw, gpu_decoder_factory, checker_libs):
    data = GPU_STREAMS[name]
    got = _decode_on_off(data, kw, gpu_decoder_factory)
    # the tie-rich streams are demodulator stress: only without the CRC check do they deliver messages
    assert got or (name.startswith("ties") and kw.get("check_crc", 1))
    _assert_signals(got, data)
    # one buffer per batch: every buffer's first positions read the carry block
    small = _decode_on_off(data, kw, gpu_decoder_factory, max_batch_bytes=BUF)
    assert [raw_bytes(m) for m in small] == [raw_bytes(m) for m in got]


@pytest.mark.gpu
def test_decode_signal_random_alphabets(gpu_decoder_factory, checker_libs):
    """Random amplitude alphabets with noise and saturated samples (tests/streams.py)."""
    n = 0
    for case, levels, data in S.random_alphabet_cases():
        for kw in (dict(), dict(check_crc=0, aggressive=1)):
            got = _decode_on_off(data, kw, gpu_decoder_factory)
            if got:
                _assert_signals(got, data)
            n += len(got)
    assert n > 500


def _padded(data):
    nbuf = data.size // BUF + 1
    p = np.full(nbuf * BUF, 127, dtype=np.uint8)
    p[: data.size] = data
    return p, nbuf


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["fused", "warp"])
@pytest.mark.parametrize("name", ["modes1", "traffic1", "ties", "seam_and_eof"])
def test_records_signal_fields(variant, name, gpu_decoder_factory, checker_libs, monkeypatch):
    """detect_host + fetch with the pass on: the records equal those without it except the two signal
    fields, which equal the restatement for decoded attempts and are 0 otherwise."""
    monkeypatch.setenv("MODES_EVAL_VARIANT", variant)
    data = GPU_STREAMS[name]
    padded, nbuf = _padded(data)
    recs = {}
    for on in (False, True):
        dec = gpu_decoder_factory(aggressive=1, signal=on)
        launches = dec.launch_count()
        dec.detect_host(padded.ctypes.data, nbuf, None)
        cands, tiles = dec.detect_fetch(nbuf)
        assert dec.launch_count() - launches == (3 if on else 2)
        order = np.concatenate([np.arange(o, o + c) for o, c in tiles]).astype(int)
        recs[on] = cands.view(np.uint8).reshape(-1, 56)[order].copy()          # in stream order, bytes kept
    b_off, b_on = recs[False], recs[True]
    assert b_off.shape == b_on.shape and b_on.shape[0] > 0
    off, on = b_off.reshape(-1).view(api.CANDIDATE_DTYPE), b_on.reshape(-1).view(api.CANDIDATE_DTYPE)
    assert np.all(off["p"]["signal"] == 0)
    b_on = b_on.copy()
    b_on[:, [26, 27, 50, 51]] = 0
    assert np.array_equal(b_on, b_off)
    mag = magnitudes(data)
    for k in (0, 1):
        p = on["p"][:, k]
        decoded = (p["flags"] & api.EVAL_DECODED) != 0
        bits = np.where((p["msgtype"] >= 16) & (p["msgtype"] <= 21), 112, 56)
        want = np.where(decoded, expected_signal(mag, on["t"] - 238, bits), 0)
        assert np.array_equal(p["signal"].astype(np.int64), want), k
        assert decoded.sum() > 0


@pytest.mark.gpu
def test_every_path_delivers_the_same_signals(gpu_decoder_factory, checker_libs):
    """Chunked feeding, two GPUs (devices reused round-robin), the device resolve and the stage-level
    entry points all deliver exactly the single-context messages, signal included."""
    import torch
    data = np.concatenate([synth.random_traffic(131072 * 6 + 4321, 1800, 93, n_aircraft=16), _seam_and_eof_stream(3, 5)])
    for kw in (dict(), dict(aggressive=1, check_crc=0)):
        ref = gpu_decoder_factory(signal=True, **_cfg(kw)).decode(data)
        want = [raw_bytes(m) for m in ref]
        assert len(want) > 200
        _assert_signals(ref, data)
        dec = gpu_decoder_factory(signal=True, max_batch_bytes=2 * BUF, **_cfg(kw))
        for chunk in (1000, 262145, 300001):
            assert [raw_bytes(m) for m in dec.decode(data, chunk=chunk)] == want, chunk
        for batch in (1, 3):
            multi = gpu_decoder_factory(signal=True, n_gpus=2, max_batch_bytes=batch * BUF, **_cfg(kw))
            assert [raw_bytes(m) for m in multi.decode(data, chunk=300001)] == want
        gres = gpu_decoder_factory(signal=True, gpu_resolve=1, max_batch_bytes=2 * BUF, **_cfg(kw))
        assert [raw_bytes(m) for m in gres.decode(data)] == want
        # stage level: detect_device over the stream in HBM, then the host resolver
        padded, nbuf = _padded(data)
        d = torch.from_numpy(padded).cuda()
        st = gpu_decoder_factory(signal=True, **_cfg(kw))
        st.detect_device(d.data_ptr(), nbuf)
        cands, tiles = st.detect_fetch(nbuf)
        res = api.Resolver(**_cfg(kw))
        res.run(cands, tiles)
        assert [raw_bytes(m) for m in res.take_messages()] == want
    # a setting changed between batches applies to the batches after it
    dec = gpu_decoder_factory(max_batch_bytes=BUF, **_cfg(kw))
    dec.reset()
    dec.process(data[: 2 * BUF])
    dec.set_signal(True)
    dec.process(data[2 * BUF:])
    dec.finish()
    msgs = dec.take_messages()
    assert [raw_bytes(m, True) for m in msgs] == [raw_bytes(m, True) for m in ref]
    assert [m.signal == 0 for m in msgs] == [m.sample_pos < 2 * 131072 - 238 for m in msgs]


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(), dict(check_crc=0)], ids=_kid)
def test_pool_delivers_the_single_stream_signals(kw, gpu_decoder_factory, checker_libs):
    """Five receivers, not in lock step, through ingest and through submit/collect: each receiver's
    messages equal a signal-on decode of its stream alone (no EOF buffer: a live receiver has none)."""
    n_rx, n_buf = 5, 3
    streams = [synth.random_traffic(n_buf * 131072, 120 * n_buf + 37 * r, seed=500 + r) for r in range(n_rx)]
    streams[-1] = S.address_chain(n_buf, "df4", seed=3)
    want = [[raw_bytes(m) for m in gpu_decoder_factory(signal=True, drop_eof_buffer=1, **_cfg(kw)).decode(s)] for s in streams]
    with api.ReceiverPool(n_rx, max_batch=4, signal=True, **_cfg(kw)) as pool:
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
                pool.submit(ids, bufs)                               # two batches in flight
                in_flight += 1
                if in_flight == 2:
                    pool.collect()
                    in_flight -= 1
            if in_flight:
                pool.collect()
            for r in range(n_rx):
                assert [raw_bytes(m) for m in pool.take(r)] == want[r], (overlap, r)
                pool.reset(r)


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
def test_signal_tracks_pulse_amplitude(gpu_decoder_factory, checker_libs):
    """DF17 frames of one amplitude A over noise of sigma = 1.5 (I and Q), no phase offset.  The pulse
    of a bit is |A + n| with n the I/Q noise plus the rounding to integers (variance 1.5^2 + 1/12 per
    component), so E[pulse^2] = A^2 + 2 * 2.33 and the RMS is 360 * sqrt(A^2 + 4.67): +0.6 % at A = 20.
    Over the 112 bits of a frame the RMS scatters by about sigma / (A * sqrt(112)) = 0.7 % at A = 20;
    the median over hundreds of frames scatters far less.  So the median lies within 2 % of 360 * A."""
    med = []
    for amp in (20.0, 40.0, 80.0):
        data = synth.df17_grid(280000, 700, 5, amp=amp, flips_cycle=(0,))
        msgs = gpu_decoder_factory(signal=True).decode(data)
        assert len(msgs) > 350
        _assert_signals(msgs, data)
        m = float(np.median([x.signal for x in msgs]))
        assert abs(m / (360 * amp) - 1) < 0.02, (amp, m)
        med.append(m)
    assert med[0] < med[1] < med[2]


@pytest.mark.gpu
def test_c_host_beast(gpu_decoder_factory, checker_libs):
    """./dump1090-b200 --beast (one and two GPUs): one frame per --raw line, same frame bytes, 12 MHz
    timestamps = 6 * sample_pos, signal bytes from the measured signal, and byte for byte what
    Message.beast() gives for a Python decode of the same file."""
    exe = ROOT / "dump1090-b200"
    f = str(C.modes1_path())
    msgs = gpu_decoder_factory(signal=True).decode(C.modes1())
    want = b"".join(m.beast() for m in msgs)
    for flags in ((), ("--gpus", "2", "--chunk", "300000")):
        raw = subprocess.run([str(exe), "--ifile", f, "--raw", *flags], capture_output=True, check=True, text=True).stdout.split()
        out = subprocess.run([str(exe), "--ifile", f, "--beast", *flags], capture_output=True, check=True).stdout
        frames = parse_beast(out)
        assert len(frames) == len(raw) == len(msgs) == 147
        assert ["*" + fr[3].hex() + ";" for fr in frames] == raw
        assert [fr[1] for fr in frames] == [6 * m.sample_pos for m in msgs]
        assert [fr[2] for fr in frames] == [beast_level(m.signal) for m in msgs]
        assert out == want, flags
    for flags in (("--no-crc-check", "--aggressive"), ("--no-fix",)):
        kw = dict(check_crc=0, aggressive=1) if flags[0] == "--no-crc-check" else dict(fix_errors=0)
        py = b"".join(m.beast() for m in gpu_decoder_factory(signal=True, **kw).decode(C.modes1()))
        out = subprocess.run([str(exe), "--ifile", f, "--beast", *flags], capture_output=True, check=True).stdout
        assert out == py, flags
