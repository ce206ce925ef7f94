"""Arrival time to a sixth of a sample (modes_set_arrival) and the refined Beast timestamp.

The reference computation is tests/arrival_model.py, a restatement of the definition in
include/modes_b200.h from the raw stream bytes: the nominal pulse pattern of the delivered frame's
bits, the main / late / early / quiet classes read from it sample by sample, and the offset rounded
from exact rationals.  CPU tests cover the arithmetic (host build of modes_arrival_core.cuh), the
accuracy against synthetic frames of known arrival, the Beast writer and the host resolve's
hand-over of the code; GPU tests the kernel and every decode path."""
import ctypes
import subprocess
from fractions import Fraction

import numpy as np
import pytest

import arrival_model as AM
import checker as C
import streams as S
import test_kernel_edges as KE
import test_signal as TS
from dump1090_b200 import api, synth

ROOT = C.ROOT
SHIM = ROOT / "tests" / "_build" / "libarrival_core_host.so"
DSHIM = ROOT / "tests" / "_build" / "libarrival_device.so"
BUF = api.BUFFER_BYTES
NS = BUF // 2
SHIFT = api.EVAL_ARRIVAL_SHIFT


def level_iq(levels) -> np.ndarray:
    """I/Q bytes of samples whose magnitude is 360 * level (I = 127 + level, Q = 127)."""
    out = np.full((len(levels), 2), 127, dtype=np.uint8)
    out[:, 0] = 127 + np.asarray(levels, dtype=np.int64)
    return out.reshape(-1)


def arrival_of(m) -> int:
    return int(m.arrival)


def zero_arrival(m) -> bytes:
    c = m.copy()
    c.arrival = 0
    return bytes(c)


# ---------------------------------------------------------------- corpora of windows


def _msgs(rng, n):
    """n random 16-byte attempt heads: 14 frame bytes, then the msgtype and flags bytes of the record."""
    return rng.integers(0, 256, size=(n, 16), dtype=np.uint8)


def _class_levels(msg, bits, level_of):
    """Window samples 0 .. 16+2b with a level per class (level_of: class -> level)."""
    cls = AM.classes(AM.frame_bits(msg, bits))
    lv = np.array([level_of[c] for c in cls], dtype=np.int64)
    return level_iq(np.concatenate([[level_of[AM.UNUSED]], lv]))


def arrival_windows(rng, bits):
    """(name, windows as I/Q bytes of samples 0 .. 16+2*112, attempt heads)."""
    n_s = 17 + 2 * 112
    yield "random", rng.integers(0, 256, size=(300, 2 * n_s), dtype=np.uint8), _msgs(rng, 300)
    yield "saturated", rng.choice(np.array([0, 255], dtype=np.uint8), size=(150, 2 * n_s)), _msgs(rng, 150)
    yield "all_127", np.full((4, 2 * n_s), 127, dtype=np.uint8), _msgs(rng, 4)
    yield "all_equal", np.tile(level_iq(np.full(n_s, 73)), (4, 1)), _msgs(rng, 4)
    yield "all_max", np.full((2, 2 * n_s), 255, dtype=np.uint8), _msgs(rng, 2)
    yield "ties", rng.choice(np.array([0, 1, 126, 127, 128, 200, 254, 255], dtype=np.uint8), size=(200, 2 * n_s)), _msgs(rng, 200)
    yield "weak", np.clip(rng.normal(127, 4, size=(200, 2 * n_s)).round(), 0, 255).astype(np.uint8), _msgs(rng, 200)
    # frames of the leak model at known fractions, with noise
    msgs = _msgs(rng, 200)
    wins = []
    for k, msg in enumerate(msgs):
        env = synth.frame_envelope(bytes(msg[: bits // 8]), frac=float(rng.uniform()))
        amp = float(rng.choice([6.0, 12.0, 40.0, 120.0]))
        x = np.zeros(n_s)
        x[: env.size] = env * amp
        x += rng.normal(0, 1.5, n_s)
        w = np.full((n_s, 2), 127, dtype=np.uint8)
        w[:, 0] = np.clip(np.rint(127 + x), 0, 255).astype(np.uint8)
        w[:, 1] = np.clip(np.rint(127 + rng.normal(0, 1.5, n_s)), 0, 255).astype(np.uint8)
        wins.append(w.reshape(-1))
    yield "leak_model", np.stack(wins), msgs
    # both ends of the clamp: main below the quiet level, a strong late (or early) class; exact halves
    cases, heads = [], []
    for k in range(120):
        msg = _msgs(rng, 1)[0]
        q, d, big = int(rng.integers(2, 40)), int(rng.integers(1, 30)), int(rng.integers(1, 60))
        late = k % 2 == 0
        level_of = {AM.QUIET: q + d, AM.MAIN: q, AM.LATE: q + d + (big if late else 0),
                    AM.EARLY: q + d + (0 if late else big), AM.UNUSED: int(rng.integers(0, 128))}
        cases.append(np.resize(_class_levels(msg, bits, level_of), 2 * n_s))
        heads.append(msg)
    for k in range(60):                                  # 6 L / (A + L) = 2.5 or 3.5: halves
        msg = _msgs(rng, 1)[0]
        a, l = [(7, 5), (5, 7)][k % 2]
        s = int(rng.integers(1, 9))
        level_of = {AM.QUIET: 0, AM.MAIN: a * s, AM.LATE: l * s if k % 4 < 2 else 0,
                    AM.EARLY: 0 if k % 4 < 2 else l * s, AM.UNUSED: 99}
        cases.append(np.resize(_class_levels(msg, bits, level_of), 2 * n_s))
        heads.append(msg)
    yield "clamp_and_halves", np.stack(cases), np.stack(heads)


def model_code(win, msg, bits):
    return AM.code_of_window(TS.magnitudes(win), msg, bits)


# ---------------------------------------------------------------- CPU: arithmetic


@pytest.fixture(scope="module")
def shim():
    subprocess.run(["make", "-s", "shim"], cwd=ROOT, check=True)
    lib = ctypes.CDLL(str(SHIM))
    lib.shim_arrival_window.restype = ctypes.c_uint32
    lib.shim_arrival_window.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32]
    lib.shim_code_of.restype = ctypes.c_uint32
    lib.shim_code_of.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    lib.shim_class_counts.argtypes = [ctypes.c_void_p, ctypes.c_uint32, ctypes.c_void_p]
    return lib


@pytest.mark.parametrize("bits", [56, 112])
def test_shim_window_equals_restatement(shim, bits):
    rng = np.random.default_rng(bits)
    seen = set()
    for name, wins, msgs in arrival_windows(rng, bits):
        for w, msg in zip(wins, msgs):
            w, msg = np.ascontiguousarray(w), np.ascontiguousarray(msg)
            want = model_code(w, msg, bits)
            assert shim.shim_arrival_window(w.ctypes.data, msg.ctypes.data, bits) == want, name
            seen.add(want)
            if name in ("all_127", "all_equal", "all_max"):
                assert want == 0, name
    assert seen == set(range(16)), sorted(seen)                        # not measured, and both clamp ends


@pytest.mark.parametrize("bits", [56, 112])
def test_shim_class_counts(shim, bits):
    rng = np.random.default_rng(3 + bits)
    for msg in _msgs(rng, 300):
        cls = AM.classes(AM.frame_bits(msg, bits))
        n = np.zeros(4, dtype=np.uint32)
        shim.shim_class_counts(np.ascontiguousarray(msg).ctypes.data, bits, n.ctypes.data)
        assert n.tolist() == [int((cls == c).sum()) for c in range(4)]
        assert n[0] >= 3 and n[1] >= 2 and n[2] >= 1 and n[3] >= 6


def test_shim_code_of_rounding_and_clamp(shim):
    """Every small combination of sums with unit counts (many exact halves and ties), and random large
    sums and counts at the bounds of the definition (counts <= 241, sums <= 241 * 65167)."""
    rng = np.random.default_rng(11)
    grid = np.array(np.meshgrid(*[np.arange(9)] * 4, indexing="ij")).reshape(4, -1).T
    n1 = np.ones(4, dtype=np.uint32)
    halves = 0
    for s in grid:
        s = np.ascontiguousarray(s, dtype=np.uint32)
        assert shim.shim_code_of(s.ctypes.data, n1.ctypes.data) == AM.code_from_sums(s, n1), s.tolist()
        mu = Fraction(int(s[3]))
        L, E = max(int(s[1]) - mu, 0), max(int(s[2]) - mu, 0)
        den = int(s[0]) - mu + L + E
        halves += den > 0 and (12 * (L - E) / den).denominator == 1 and (12 * (L - E) / den) % 2 == 1
    assert halves > 100
    for _ in range(20000):
        n = rng.integers(1, 242, 4).astype(np.uint32)
        s = (rng.integers(0, 65168, 4) * n).astype(np.uint32) if rng.random() < 0.5 else \
            rng.integers(0, 241 * 65167 + 1, 4).astype(np.uint32)
        assert shim.shim_code_of(s.ctypes.data, n.ctypes.data) == AM.code_from_sums(s, n), (s.tolist(), n.tolist())


# ---------------------------------------------------------------- CPU: accuracy on synthetic frames


def _known_arrival_stream(amp, seed, n_frames=2500, period=420):
    """DF17 frames at known positions and fractions (uniform in [0, 1)), sigma = 1.5."""
    rng = synth.Counter(seed)
    frames, truth = [], []
    for k in range(n_frames):
        icao = 0x400000 + rng.below(0x3FFFFF)
        frame = synth.make_frame(17, 5, icao.to_bytes(3, "big") + bytes(rng.below(256) for _ in range(7)))
        pos = 300 + k * period + rng.below(100)
        frac = rng.uniform()
        frames.append((pos, frame, amp, 2 * np.pi * rng.uniform(), frac))
        truth.append((pos, frac, frame))
    return synth.synth_stream(300 + n_frames * period + 500, frames, sigma=1.5, seed=seed), truth


def arrival_errors(data, truth, msgs):
    """(refined error, coarse error) in ticks per delivered message matched to a planted frame, and the
    number of phase-corrected messages among them."""
    pos_true = np.array([t[0] for t in truth])
    mag = TS.magnitudes(data)
    codes = AM.expected_arrival(mag, [m.sample_pos for m in msgs], [bytes(m.msg) for m in msgs], [m.msgbits for m in msgs])
    fine, coarse, retry = [], [], 0
    for m, code in zip(msgs, codes):
        k = int(np.searchsorted(pos_true, m.sample_pos - 1))
        if k >= len(truth) or abs(truth[k][0] - m.sample_pos) > 1 or bytes(m.msg[:14]) != truth[k][2]:
            continue
        true = 6 * (truth[k][0] + truth[k][1])
        fine.append(AM.arrival_ticks(m.sample_pos, code) - true)
        coarse.append(6 * m.sample_pos - true)
        retry += m.phase_corrected
    return np.array(fine), np.array(coarse), retry


@pytest.mark.parametrize("amp", [8.0, 12.0, 20.0, 60.0])
def test_accuracy_on_frames_of_known_arrival(amp, checker_libs):
    data, truth = _known_arrival_stream(amp, seed=int(amp) + 3)
    msgs, _ = C.oracle_decode(data)
    fine, coarse, retry = arrival_errors(data, truth, msgs)
    assert fine.size > 800, fine.size
    assert retry > 20                                        # frames delivered by the phase-corrected retry
    med, p95, bias = np.median(np.abs(fine)), np.percentile(np.abs(fine), 95), abs(fine.mean())
    cmed, cp95 = np.median(np.abs(coarse)), np.percentile(np.abs(coarse), 95)
    assert med < cmed and p95 < cp95, (med, p95, cmed, cp95)
    if amp == 8.0:
        assert med <= 0.8 and p95 <= 2.0 and bias <= 0.5, (med, p95, bias)
    if amp >= 20.0:
        assert med <= 0.5 and p95 <= 1.0, (med, p95)


# ---------------------------------------------------------------- CPU: Beast writer


def _msg(frame: bytes, sample_pos: int, arrival: int, signal=1000) -> api.Message:
    m = TS._msg(frame, sample_pos, signal)
    m.arrival = arrival
    return m


def _beast_by_hand(frame, ts, signal):
    body = bytes([0x33 if len(frame) == 14 else 0x32]) + ts.to_bytes(6, "big") + bytes([TS.beast_level(signal)]) + frame
    return b"\x1a" + body.replace(b"\x1a", b"\x1a\x1a")


SHORT = bytes.fromhex("5d4840d6202cc3")
LONG = bytes.fromhex("8d4840d6202cc371c32ce0576098")
BEAST_CASES = [
    ("code0", LONG, 123456789, 0, 6 * 123456789),
    ("code1", SHORT, 1000, 1, 6000 - 7),
    ("code8", SHORT, 1000, 8, 6000),
    ("code15", LONG, 1000, 15, 6007),
    ("clamped_at_0", SHORT, 0, 1, 0),
    ("clamped_at_0_b", SHORT, 1, 3, 1),
    ("not_clamped", SHORT, 1, 2, 0),
    ("wrap_2_48", SHORT, (1 << 48) // 6, 15, (6 * ((1 << 48) // 6) + 7) % (1 << 48)),
    ("wrap_down", SHORT, (1 << 48) // 6 + 1, 1, (6 * ((1 << 48) // 6 + 1) - 7) % (1 << 48)),
    ("wrap_big", LONG, (1 << 50) + 3, 12, (6 * ((1 << 50) + 3) + 4) % (1 << 48)),
    ("offset_makes_1a", SHORT, 4, 10, 0x1A),                           # 24 + 2 = 26 = 0x1a
    ("offset_makes_1a1a", SHORT, 0x1A1A // 6 + 1, 8 - (6 * (0x1A1A // 6 + 1) - 0x1A1A), 0x1A1A),
    ("hex_door", SHORT, -1, 0, 0),
]


@pytest.mark.parametrize("name,frame,pos,code,ts", BEAST_CASES, ids=[c[0] for c in BEAST_CASES])
def test_format_beast_with_arrival(name, frame, pos, code, ts):
    m = _msg(frame, pos, code)
    assert m.timestamp_12mhz() == ts
    got = m.beast()
    assert got == _beast_by_hand(frame, ts, 1000)
    (_, parsed_ts, _, body), = TS.parse_beast(got)
    assert parsed_ts == ts and body == frame
    if name.startswith("offset_makes_1a"):
        assert (6 * pos) % 256 != 0x1A and b"\x1a\x1a" in got
    L = api.lib()
    for cap in range(len(got) + 2):
        buf = (ctypes.c_uint8 * 64)(*([0xEE] * 64))
        assert L.modes_format_beast(ctypes.byref(m), buf, cap) == len(got)
        assert bytes(buf[:min(cap, len(got))]) == got[:cap]


def test_beast_code0_is_todays_frame():
    """arrival = 0 writes exactly the frame of a message without the field."""
    rng = np.random.default_rng(4)
    for _ in range(300):
        frame = bytes(rng.choice(np.array([0x1A, 0x00, 0xFF, 0x8D], np.uint8), size=14 if rng.random() < 0.5 else 7))
        pos, sig = int(rng.integers(-1, 1 << 49)), int(rng.integers(0, 65536))
        m = _msg(frame, pos, 0, sig)
        assert m.beast() == TS._beast_by_hand(frame, pos, sig)
        assert m.timestamp_12mhz() == (0 if pos < 0 else (6 * pos) % (1 << 48))


def test_c_host_refuses_arrival_without_beast(tmp_path):
    exe = ROOT / "dump1090-b200"
    assert exe.exists(), "build the C host with `make`"
    f = tmp_path / "empty.bin"
    f.write_bytes(b"")
    for other in ((), ("--raw",), ("--sbs",), ("--stats",)):
        r = subprocess.run([str(exe), "--ifile", str(f), "--arrival", *other], capture_output=True, text=True)
        assert r.returncode == 1 and "--arrival" in r.stderr and "--beast" in r.stderr and r.stdout == "", other


# ---------------------------------------------------------------- CPU: host resolve carries the code


def _planted(data, kw):
    """Oracle candidate records with a random code planted in bits 4-7 of every attempt's flags."""
    arr = TS._records(data, kw)
    arr["p"]["signal"] = 0
    rng = np.random.default_rng(arr.size + 1)
    codes = rng.integers(0, 16, size=(arr.size, 2)).astype(np.uint8)
    plain = arr.copy()
    arr["p"]["flags"] = (arr["p"]["flags"] & 0x0F) | (codes << SHIFT)
    return plain, arr


def _check_codes(msgs, index_of, arr, check_crc):
    seen, n = {}, 0
    for m in msgs:
        i = index_of(m)
        nth = seen.get(i, 0)
        seen[i] = nth + 1
        p0_decoded = bool(arr[i]["p"]["flags"][0] & api.EVAL_DECODED)
        k = 1 if (nth == 1 or m.phase_corrected or not p0_decoded) else 0
        assert arrival_of(m) == int(arr[i]["p"]["flags"][k]) >> SHIFT, (m.sample_pos, k)
        n += 1
    return n


@pytest.mark.parametrize("kw", TS.FLAGS, ids=TS._kid)
def test_host_resolve_delivers_the_attempts_code(kw, checker_libs):
    data = TS._stream()
    nbuf = data.size // BUF + 1
    plain, arr = _planted(data, kw)
    tiles = TS._tiled(arr, nbuf)
    pos_to_idx = {int(t) - 238: i for i, t in enumerate(arr["t"])}
    index_of = lambda m: pos_to_idx[int(m.sample_pos)]                          # noqa: E731
    res = api.Resolver(**TS._cfg(kw))
    res.run(plain, tiles)
    base = res.take_messages()
    assert all(m.arrival == 0 for m in base)
    res = api.Resolver(**TS._cfg(kw))
    res.run(arr, tiles)
    one = res.take_messages()
    assert len(one) == len(base) > 100
    assert [zero_arrival(m) for m in one] == [bytes(m) for m in base]
    assert _check_codes(one, index_of, arr, kw.get("check_crc", 1)) == len(one)
    assert len({m.arrival for m in one}) == 16
    cut = [0, 2, 4, nbuf]
    shards = []
    for a, b in zip(cut[:-1], cut[1:]):
        sel = arr[((arr["t"] >> 17) >= a) & ((arr["t"] >> 17) < b)].copy()
        sel["t"] -= a << 17
        shards.append((sel, TS._tiled(sel, b - a), a))
    res = api.Resolver(**TS._cfg(kw))
    res.run_shards(shards)
    assert [bytes(m) for m in res.take_messages()] == [bytes(m) for m in one]
    res = api.Resolver(**TS._cfg(kw))
    for c, t, b in shards:
        res.run_tentative(c, t, b)
        res.commit()
    assert [bytes(m) for m in res.take_messages()] == [bytes(m) for m in one]


@pytest.mark.parametrize("kw", [dict(), dict(check_crc=0)], ids=TS._kid)
def test_pool_resolve_delivers_the_attempts_code(kw, checker_libs):
    n_rx = 4
    streams = [synth.random_traffic(131072, 160 + 20 * r, seed=310 + r) for r in range(n_rx)]
    batch = np.full(2 * n_rx * BUF, 127, dtype=np.uint8)
    for i in range(n_rx):
        batch[(2 * i + 1) * BUF: (2 * i + 2) * BUF] = streams[i]
    _, arr = _planted(batch, kw)
    tiles = TS._tiled(arr, 2 * n_rx)
    with api.ReceiverPool(n_rx, **TS._cfg(kw)) as pool:
        pool.resolve(list(range(n_rx)), arr, tiles)
        total = 0
        for r in range(n_rx):
            t0 = 131072 * (2 * r + 1)
            pos_to_idx = {int(t) - t0 - 238: i for i, t in enumerate(arr["t"]) if t0 <= t < t0 + 131072}
            msgs = pool.take(r)
            exp, _ = C.oracle_decode(streams[r], drop_eof=1, **kw)
            assert [m.raw_line() for m in msgs] == [m.hexline() for m in exp]
            total += _check_codes(msgs, lambda m: pos_to_idx[int(m.sample_pos)], arr, kw.get("check_crc", 1))
        assert total > 100


# ---------------------------------------------------------------- GPU


GPU_STREAMS = TS.GPU_STREAMS


def _assert_codes(msgs, data):
    mag = TS.magnitudes(data)
    want = AM.expected_arrival(mag, [m.sample_pos for m in msgs], [bytes(m.msg) for m in msgs], [m.msgbits for m in msgs])
    got = np.array([m.arrival for m in msgs], dtype=np.int64)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{bad.size} of {got.size} differ, first: pos {msgs[bad[0]].sample_pos} got {got[bad[0]]} want {want[bad[0]]}"


SWITCHES = [dict(signal=False), dict(signal=True)]


def _decode_on_off(data, kw, factory, signal, **extra):
    off = factory(signal=signal, **TS._cfg(kw), **extra)
    on = factory(signal=signal, arrival=True, **TS._cfg(kw), **extra)
    got_off, got_on = off.decode(data), on.decode(data)
    assert [zero_arrival(m) for m in got_on] == [bytes(m) for m in got_off]
    assert all(m.arrival == 0 for m in got_off)
    assert on.stats() == off.stats()
    return got_on


@pytest.mark.gpu
@pytest.mark.parametrize("signal", [False, True], ids=["arrival", "signal_arrival"])
@pytest.mark.parametrize("name", list(GPU_STREAMS))
@pytest.mark.parametrize("kw", TS.FLAGS, ids=TS._kid)
def test_decode_arrival_equals_restatement(name, kw, signal, gpu_decoder_factory, checker_libs):
    data = GPU_STREAMS[name]
    got = _decode_on_off(data, kw, gpu_decoder_factory, signal)
    assert got or (name.startswith("ties") and kw.get("check_crc", 1))
    _assert_codes(got, data)
    if signal:
        TS._assert_signals(got, data)
    small = _decode_on_off(data, kw, gpu_decoder_factory, signal, max_batch_bytes=BUF)
    assert [bytes(m) for m in small] == [bytes(m) for m in got]


@pytest.mark.gpu
def test_decode_arrival_random_alphabets(gpu_decoder_factory, checker_libs):
    n = 0
    for c, (case, levels, data) in enumerate(S.random_alphabet_cases()):
        for kw in (dict(), dict(check_crc=0, aggressive=1)):
            got = _decode_on_off(data, kw, gpu_decoder_factory, c % 2 == 1)
            _assert_codes(got, data)
            n += len(got)
    assert n > 500


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["fused", "warp"])
@pytest.mark.parametrize("name", ["modes1", "traffic1", "ties", "seam_and_eof"])
def test_records_arrival_fields(variant, name, gpu_decoder_factory, checker_libs, monkeypatch):
    """detect_host + fetch under each switch set: the records equal the switch-off records except the
    signal halfwords (signal on) and bits 4-7 of the flags (arrival on), which equal the restatements
    for decoded attempts and are 0 otherwise; the pass is one launch whichever switches are on."""
    monkeypatch.setenv("MODES_EVAL_VARIANT", variant)
    data = GPU_STREAMS[name]
    padded, nbuf = TS._padded(data)
    mag = TS.magnitudes(data)
    recs = {}
    for sig, arr in ((False, False), (True, False), (False, True), (True, True)):
        dec = gpu_decoder_factory(aggressive=1, signal=sig, arrival=arr)
        launches = dec.launch_count()
        dec.detect_host(padded.ctypes.data, nbuf, None)
        cands, tiles = dec.detect_fetch(nbuf)
        assert dec.launch_count() - launches == (3 if sig or arr else 2)
        order = np.concatenate([np.arange(o, o + c) for o, c in tiles]).astype(int)
        recs[sig, arr] = cands.view(np.uint8).reshape(-1, 56)[order].copy()
    base = recs[False, False]
    assert np.all(base[:, [23, 47]] >> 4 == 0)
    for (sig, arr), b in recs.items():
        assert b.shape == base.shape and b.shape[0] > 0
        rest = b.copy()
        rest[:, [26, 27, 50, 51]] = 0
        rest[:, [23, 47]] &= 0x0F
        assert np.array_equal(rest, base), (sig, arr)
        assert np.array_equal(b[:, [26, 27, 50, 51]], recs[True, False][:, [26, 27, 50, 51]] if sig else base[:, [26, 27, 50, 51]])
        on = b.reshape(-1).view(api.CANDIDATE_DTYPE)
        for k in (0, 1):
            p = on["p"][:, k]
            decoded = (p["flags"] & api.EVAL_DECODED) != 0
            got = p["flags"].astype(np.int64) >> SHIFT
            if not arr:
                assert np.all(got == 0)
                continue
            bits = np.where((p["msgtype"] >= 16) & (p["msgtype"] <= 21), 112, 56)
            sel = np.flatnonzero(decoded)
            want = AM.expected_arrival(mag, on["t"][sel] - 238, [bytes(x) for x in p["msg"][sel]], bits[sel])
            assert np.array_equal(got[sel], want), k
            assert np.all(got[~decoded] == 0) and sel.size > 0


@pytest.mark.gpu
def test_every_path_delivers_the_same_codes(gpu_decoder_factory, checker_libs, monkeypatch):
    """Chunked feeding, two GPUs, the device resolve and the stage-level entry points all deliver the
    single-context messages, arrival included, after every evaluation variant."""
    import torch
    data = np.concatenate([synth.random_traffic(131072 * 6 + 4321, 1800, 95, n_aircraft=16), TS._seam_and_eof_stream(3, 5)])
    for kw in (dict(), dict(aggressive=1, check_crc=0)):
        ref = gpu_decoder_factory(arrival=True, **TS._cfg(kw)).decode(data)
        want = [bytes(m) for m in ref]
        assert len(want) > 200 and len({m.arrival for m in ref}) > 5
        _assert_codes(ref, data)
        dec = gpu_decoder_factory(arrival=True, max_batch_bytes=2 * BUF, **TS._cfg(kw))
        for chunk in (1000, 262145, 300001):
            assert [bytes(m) for m in dec.decode(data, chunk=chunk)] == want, chunk
        for batch in (1, 3):
            multi = gpu_decoder_factory(arrival=True, n_gpus=2, max_batch_bytes=batch * BUF, **TS._cfg(kw))
            assert [bytes(m) for m in multi.decode(data, chunk=300001)] == want
        gres = gpu_decoder_factory(arrival=True, gpu_resolve=1, max_batch_bytes=2 * BUF, **TS._cfg(kw))
        assert [bytes(m) for m in gres.decode(data)] == want
        padded, nbuf = TS._padded(data)
        d = torch.from_numpy(padded).cuda()
        st = gpu_decoder_factory(arrival=True, **TS._cfg(kw))
        st.detect_device(d.data_ptr(), nbuf)
        cands, tiles = st.detect_fetch(nbuf)
        res = api.Resolver(**TS._cfg(kw))
        res.run(cands, tiles)
        assert [bytes(m) for m in res.take_messages()] == want
    for variant in ("fused", "warp"):
        monkeypatch.setenv("MODES_EVAL_VARIANT", variant)
        got = gpu_decoder_factory(arrival=True, signal=True).decode(data)
        _assert_codes(got, data)
        TS._assert_signals(got, data)


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(), dict(check_crc=0)], ids=TS._kid)
def test_pool_delivers_the_single_stream_codes(kw, gpu_decoder_factory, checker_libs):
    n_rx, n_buf = 4, 3
    streams = [synth.random_traffic(n_buf * 131072, 120 * n_buf + 37 * r, seed=520 + r) for r in range(n_rx)]
    want = [[bytes(m) for m in gpu_decoder_factory(arrival=True, drop_eof_buffer=1, **TS._cfg(kw)).decode(s)] for s in streams]
    with api.ReceiverPool(n_rx, max_batch=3, arrival=True, **TS._cfg(kw)) as pool:
        nxt = [0] * n_rx
        for ids in TS._schedule(np.random.default_rng(9), n_rx, n_buf, 3):
            pool.ingest(ids, [streams[r][nxt[r] * BUF: (nxt[r] + 1) * BUF] for r in ids])
            for r in ids:
                nxt[r] += 1
        for r in range(n_rx):
            assert [bytes(m) for m in pool.take(r)] == want[r], r


@pytest.mark.gpu
def test_arrival_tracks_known_fraction(gpu_decoder_factory, checker_libs):
    """The GPU decode of a stream of known arrivals: the codes equal the restatement and meet the
    accuracy of the CPU test, and the oracle's messages are delivered unchanged."""
    data, truth = _known_arrival_stream(20.0, seed=77, n_frames=1500)
    msgs = gpu_decoder_factory(arrival=True).decode(data)
    exp, _ = C.oracle_decode(data)
    assert [m.raw_line() for m in msgs] == [m.hexline() for m in exp]
    _assert_codes(msgs, data)
    fine, coarse, _ = arrival_errors(data, truth, msgs)
    assert fine.size > 1000
    assert np.median(np.abs(fine)) <= 0.5 and np.percentile(np.abs(fine), 95) <= 1.0


@pytest.mark.gpu
def test_c_host_beast_arrival(gpu_decoder_factory, checker_libs):
    """./dump1090-b200 --beast --arrival (one and two GPUs) writes what Message.beast() gives for a
    decode with signal and arrival on; without --arrival it writes today's bytes."""
    exe = ROOT / "dump1090-b200"
    f = str(C.modes1_path())
    msgs = gpu_decoder_factory(signal=True, arrival=True).decode(C.modes1())
    want = b"".join(m.beast() for m in msgs)
    plain = b"".join(m.beast() for m in gpu_decoder_factory(signal=True).decode(C.modes1()))
    assert want != plain
    for flags in ((), ("--gpus", "2", "--chunk", "300000")):
        out = subprocess.run([str(exe), "--ifile", f, "--beast", "--arrival", *flags], capture_output=True, check=True).stdout
        frames = TS.parse_beast(out)
        assert len(frames) == len(msgs) == 147
        assert [fr[1] for fr in frames] == [m.timestamp_12mhz() for m in msgs]
        assert out == want, flags
        assert subprocess.run([str(exe), "--ifile", f, "--beast", *flags], capture_output=True, check=True).stdout == plain
    codes = np.array([m.arrival for m in msgs])
    assert (codes > 0).mean() > 0.95 and len(set(codes.tolist())) > 3


# ---------------------------------------------------------------- GPU: the device harness


@pytest.fixture(scope="module")
def dshim():
    subprocess.run(["make", "-s", "dshim"], cwd=ROOT, check=True)
    lib = ctypes.CDLL(str(DSHIM))
    u32, p = ctypes.c_uint32, ctypes.c_void_p
    lib.arr_error.restype = ctypes.c_char_p
    lib.arr_sm_count.restype = ctypes.c_int
    lib.arr_signal_pass.argtypes = [p, u32, p, p, u32, u32, u32, ctypes.c_int, ctypes.c_int]
    assert lib.arr_sm_count() > 0, lib.arr_error()
    return lib


N_WIN = 17 + 2 * 112                                     # window samples 0 .. 16+2*112


@pytest.fixture(scope="module")
def arrival_corpus():
    """Windows of both corpora with their attempt heads, for the 56- and 112-bit attempts."""
    rng = np.random.default_rng(99)
    wins, heads = [], []
    for bits in (56, 112):
        for _, w, h in arrival_windows(rng, bits):
            wins.append(w)
            heads.append(h)
    return np.concatenate(wins), np.concatenate(heads)


def _put(batch, t, win):
    v = 2 * (int(t) + 2)                                 # m[j] of record t is virtual sample t + 2
    batch.virt[v: v + win.size] = win


def arrival_placements(n, placement):
    if placement in ("even", "odd"):
        t = 1000 + (placement == "odd") + 242 * np.arange(n)
        return [(int(t[-1] + 244) // NS + 1, np.arange(n), t)]
    if placement == "carry":
        return [(1, np.array([k]), np.array([(37 * k) % 238])) for k in range(min(n, 300))]
    return KE.placements(min(n, 400), "last_j")


COMBOS = np.array([(56, 112), (112, 56), (0, 112), (56, 0), (112, 112), (56, 56), (0, 0)])


def arrival_records(rng, t, heads, combos):
    """Records at t, random bytes elsewhere; attempt k decoded with heads[:, k] as its msg (and the
    msgtype byte set for its length) or not decoded."""
    recs = KE.signal_records(rng, t, combos)
    b = recs.view(np.uint8).reshape(t.size, 56)
    for k in (0, 1):
        b[:, 8 + 24 * k: 22 + 24 * k] = heads[:, k, :14]
    return recs


def expected(before, wins, heads, combos, signal, arrival, limit=None):
    want = before.copy()
    b = want.view(np.uint8).reshape(-1, 56)
    h = want.view(np.uint16).reshape(-1, 28)
    n = want.size if limit is None else min(limit, want.size)
    for i in range(n):
        mag = TS.magnitudes(wins[i])
        for k in (0, 1):
            bits = int(combos[i, k])
            if not bits:
                continue
            if signal:
                h[i, 13 + 12 * k] = TS.expected_signal(mag, [0], [bits])[0]
            if arrival:
                head = b[i, 8 + 24 * k: 24 + 24 * k]
                b[i, 23 + 24 * k] = (b[i, 23 + 24 * k] & 0x0F) | (AM.code_of_window(mag, head, bits) << SHIFT)
    return want


def run_dev(lib, batch, recs, signal, arrival, capacity=None, counter=None):
    recs = np.ascontiguousarray(recs).copy()
    body, carry = batch.args()
    rc = lib.arr_signal_pass(body.ctypes.data, batch.n_buffers, carry.ctypes.data, recs.ctypes.data, recs.size,
                                recs.size if capacity is None else capacity, recs.size if counter is None else counter,
                                int(signal), int(arrival))
    assert rc == 0, lib.arr_error()
    return recs


@pytest.mark.gpu
@pytest.mark.parametrize("placement", ["even", "odd", "carry", "last_j"])
def test_arrival_fields_on_constructed_corpora(placement, dshim, arrival_corpus):
    wins, heads = arrival_corpus
    rng = np.random.default_rng(len(placement) + 7)
    n_dec = 0
    for nb, idx, t in arrival_placements(len(wins), placement):
        batch = KE.Batch(nb)
        for i, ti in zip(idx, t):
            _put(batch, ti, wins[i])
        combos = COMBOS[rng.integers(0, len(COMBOS), idx.size)]
        hd = np.stack([heads[idx], heads[rng.permutation(idx)]], axis=1)
        hd[:, 1] = np.where((combos[:, 1] == combos[:, 0])[:, None] & (rng.random(idx.size) < 0.5)[:, None], hd[:, 0], hd[:, 1])
        recs = arrival_records(rng, t, hd, combos)
        sel_wins = wins[idx]
        for sig, arr in ((False, True), (True, True), (True, False)):
            got = run_dev(dshim, batch, recs, sig, arr)
            KE.assert_records_equal(got, expected(recs, sel_wins, hd, combos, sig, arr), (placement, sig, arr))
        n_dec += int((combos > 0).sum())
    assert n_dec > 0


@pytest.mark.gpu
def test_arrival_capacity_and_second_trip(dshim, arrival_corpus):
    wins, heads = arrival_corpus
    rng = np.random.default_rng(6)
    wins, heads = wins[:200], heads[:200]
    (nb, idx, t), = arrival_placements(len(wins), "odd")
    batch = KE.Batch(nb)
    for i, ti in zip(idx, t):
        _put(batch, ti, wins[i])
    n = 600
    widx = rng.integers(0, len(wins), n)
    combos = COMBOS[rng.integers(0, len(COMBOS), n)]
    hd = np.stack([heads[widx], heads[widx]], axis=1)
    recs = arrival_records(rng, t[widx], hd, combos)
    for capacity, counter in ((n // 3, n + 5), (n // 3, 2 ** 32 - 1), (n, 100), (n, 0), (0, n)):
        got = run_dev(dshim, batch, recs, True, True, capacity, counter)
        KE.assert_records_equal(got, expected(recs, wins[widx], hd, combos, True, True, min(capacity, counter)), (capacity, counter))
    # more records than 32 per warp of a full wave: the grid-stride loop comes back
    n = 32 * KE.MAX_WARPS_PER_SM * dshim.arr_sm_count() * 5 // 2
    widx = rng.integers(0, len(wins), n)
    combos = COMBOS[rng.integers(0, len(COMBOS), n)]
    hd = np.stack([heads[widx], heads[widx]], axis=1)
    recs = arrival_records(rng, t[widx], hd, combos)
    got = run_dev(dshim, batch, recs, False, True)
    code = {b: np.array([AM.code_of_window(TS.magnitudes(w), h, b) for w, h in zip(wins, heads)]) for b in (56, 112)}
    exp = recs.copy()
    eb = exp.view(np.uint8).reshape(-1, 56)
    for k in (0, 1):
        bits = combos[:, k]
        c = np.where(bits == 112, code[112][widx], code[56][widx]).astype(np.uint8)
        eb[:, 23 + 24 * k] = np.where(bits > 0, (eb[:, 23 + 24 * k] & 0x0F) | (c << SHIFT), eb[:, 23 + 24 * k])
    KE.assert_records_equal(got, exp, "second trip")
    # a record whose arrival window would end outside the batch is refused before anything runs
    edge = recs[:2].copy()
    edge["t"][1] = 240 + nb * NS - 242
    body, carry = batch.args()
    assert dshim.arr_signal_pass(body.ctypes.data, nb, carry.ctypes.data, edge.ctypes.data, 2, 2, 2, 0, 1) != 0

