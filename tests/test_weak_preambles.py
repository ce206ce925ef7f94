"""Recovery at weak preambles (modes_set_weak_preambles, modes_weak_device, modes_resolver_run_weak,
modes_pool_set_weak_preambles).

The reference computations are in tests/weak_model.py: a numpy restatement of the weak-preamble scan
from the raw stream bytes (its records are recover_model's restatement at the weak positions), and a
Python model of the resolve with the weak positions merged into the walk.  CPU tests cover the
arithmetic (host build of modes_weak_core.cuh), the scan's condition 4 against the oracle's candidates
and the host resolve; GPU tests the kernels and every decode path."""
import ctypes
import subprocess

import numpy as np
import pytest

import checker as C
import recover_model as R
import streams as S
import weak_model as W
from dump1090_b200 import api, synth

ROOT = C.ROOT
SHIM = ROOT / "tests" / "_build" / "libweak_core_host.so"
BUF = api.BUFFER_BYTES
FLAGS = [dict(), dict(aggressive=1), dict(fix=0), dict(check_crc=0)]


def _kid(k):
    return "-".join(f"{a}{b}" for a, b in k.items()) or "default"


# ---------------------------------------------------------------- CPU: arithmetic


@pytest.fixture(scope="module")
def shim():
    subprocess.run(["make", "-s", "shim"], cwd=ROOT, check=True)
    lib = ctypes.CDLL(str(SHIM))
    lib.shim_weak.restype = ctypes.c_int
    lib.shim_weak.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    return lib


def _shim_flags(shim, wins):
    wins = np.ascontiguousarray(wins, dtype=np.uint8).reshape(-1, 2 * W.WINDOW)
    out = np.zeros(wins.shape[0], dtype=np.uint8)
    assert shim.shim_weak(wins.ctypes.data, wins.shape[0], out.ctypes.data) == 0
    return out


def _restated_flags(wins):
    weak, sc, ref = W.conditions(W.window_mags(wins))
    return weak.astype(np.uint8) | (sc.astype(np.uint8) << 1) | (ref.astype(np.uint8) << 2)


def _window_cases():
    rng = np.random.default_rng(77)
    n = 40000
    cases = {"random": rng.integers(0, 256, (n, 52), dtype=np.uint8),
             "near127": (127 + rng.integers(-6, 7, (n, 52))).astype(np.uint8),
             "ties": rng.choice(np.array([127, 127, 128, 167, 227], np.uint8), (n, 52)),
             "saturated": rng.choice(np.array([0, 1, 254, 255, 127], np.uint8), (n, 52)),
             "all127": np.full((64, 52), 127, np.uint8)}
    # windows cut from streams with weak frames: many pass conditions 1-3
    data, _ = synth.fleet_at(8, 600, 4321)
    M = data[: (data.size // 104) * 104].reshape(-1, 52)
    cases["fleet8"] = np.concatenate([M, data[2: 2 + ((data.size - 2) // 104) * 104].reshape(-1, 52)])
    return cases


def test_shim_equals_restatement(shim):
    total = 0
    for name, wins in _window_cases().items():
        got, want = _shim_flags(shim, wins), _restated_flags(wins)
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, (name, bad[:5].tolist(), got[bad[:5]].tolist(), want[bad[:5]].tolist())
        total += int((want & 1).sum())
        if name == "all127":
            assert (want == 0).all()
    assert total > 50                                    # the corpora reach the positive side


@pytest.mark.parametrize("name", ["modes1", "traffic_s1", "traffic_lowsnr", "traffic_loud", "tiny"])
def test_condition4_equals_oracle_candidates(name, checker_libs):
    data = _golden_stream(name)
    nbuf = data.size // BUF + 1
    cand = R.oracle_records(data, {})["t"]
    ref = W.reference_positions(data, nbuf)
    assert np.array_equal(np.sort(cand).astype(np.int64), ref.astype(np.int64))
    weak = W.weak_positions(data, nbuf)
    assert np.intersect1d(weak, ref).size == 0


def _golden_stream(name):
    import golden_util as G
    return G.make_input(G.load(name))


# ---------------------------------------------------------------- CPU: the resolve


def _fleet(snr, n=1500):
    return synth.fleet_at(snr, n, 2000 + snr)[0]


def _cpu_streams():
    yield "modes1", C.modes1()
    for seed in (1, 2):
        yield f"traffic{seed}", synth.random_traffic(300000, 400, seed)
    for snr in (7, 9, 12):
        yield f"fleet{snr}", _fleet(snr)


CPU_STREAMS = dict(_cpu_streams())


@pytest.mark.parametrize("name", list(CPU_STREAMS))
@pytest.mark.parametrize("kw", FLAGS, ids=_kid)
def test_resolve_equals_model(name, kw, checker_libs, monkeypatch):
    data = CPU_STREAMS[name]
    msgs, stats, rstats, wstats, arr, rec, wt, wr = W.cpu_decode(data, kw, signal=True)
    tiles = R.tiled(arr, data.size // BUF + 1)
    off = api.Resolver(**R.flag_cfg(kw))
    off.run(arr, tiles)
    off_msgs, off_stats = off.take_messages(), off.stats()
    # the reference's messages and statistics are untouched
    assert [bytes(m) for m in msgs if not m.recovered] == [bytes(m) for m in off_msgs]
    assert stats == off_stats
    want, want_st, want_wst = W.model(off_msgs, arr, rec, wt, wr, kw.get("check_crc", 1))
    assert W.as_rows(msgs) == W.model_rows(want)
    assert rstats == want_st and wstats == want_wst
    assert wstats["considered"] <= wt.size
    if name == "fleet9":
        assert wstats["delivered"] > 5, wstats
    # with no weak positions: exactly the recovery resolve
    plain = api.Resolver(**R.flag_cfg(kw))
    plain.run(arr, tiles, recovered=rec)
    empty = api.Resolver(**R.flag_cfg(kw))
    empty.run(arr, tiles, recovered=rec, weak=(wt[:0], wr[:0]))
    assert [bytes(m) for m in empty.take_messages()] == [bytes(m) for m in plain.take_messages()]
    assert empty.stats() == plain.stats() and empty.recovery_stats() == plain.recovery_stats()
    assert empty.weak_stats() == dict.fromkeys(api.RECOVERY_STAT_NAMES, 0)
    # parts judged concurrently, with a guess that is wrong at least sometimes: the same result
    for parts, part_tiles in (("1", None), ("4", "8"), ("7", "3")):
        monkeypatch.setenv("MODES_RESOLVE_PARTS", parts)
        if part_tiles:
            monkeypatch.setenv("MODES_RESOLVE_PART_TILES", part_tiles)
        res = api.Resolver(**R.flag_cfg(kw))
        res.run(arr, tiles, recovered=rec, weak=(wt, wr))
        assert [bytes(m) for m in res.take_messages()] == [bytes(m) for m in msgs], parts
        assert (res.stats(), res.recovery_stats(), res.weak_stats()) == (stats, rstats, wstats)


def test_ground_truth_fleet_sweep(checker_libs):
    """Every frame recovered at a weak preamble was transmitted, and the weak positions add frames."""
    gain = 0
    for snr in (7, 8, 9, 10):
        data, truth = synth.fleet_at(snr, 1500, 1000 + snr)
        msgs, *_ = W.cpu_decode(data, dict(aggressive=1))
        weak = [m.hex() for m in msgs if m.recovered == 2]
        assert all(h in truth for h in weak), snr
        gain += len(weak)
    assert gain > 40


@pytest.mark.parametrize("kw", [dict(), dict(check_crc=0)], ids=_kid)
def test_shards_equal_the_run_shard_by_shard(kw, checker_libs):
    data = np.concatenate([_fleet(8), _fleet(10), synth.random_traffic(131072 * 3, 600, 5)])
    msgs, stats, rstats, wstats, arr, rec, wt, wr = W.cpu_decode(data, kw, signal=True)
    nbuf = data.size // BUF + 1
    cut = [0, 2, 5, 6, nbuf]
    shards, recs, weaks = [], [], []
    for a, b in zip(cut[:-1], cut[1:]):
        sel = ((arr["t"] >> 17) >= a) & ((arr["t"] >> 17) < b)
        c = arr[sel].copy()
        c["t"] -= a << 17
        shards.append((c, R.tiled(c, b - a), a))
        recs.append(rec[sel].copy())
        ws = ((wt >> 17) >= a) & ((wt >> 17) < b)
        weaks.append(((wt[ws] - (a << 17)).astype(np.uint32), wr[ws].copy()))
    one = api.Resolver(**R.flag_cfg(kw))
    for (c, t, b), r, w in zip(shards, recs, weaks):
        one.run(c, t, b, recovered=r, weak=w)
    together = api.Resolver(**R.flag_cfg(kw))
    together.run_shards(shards, recovered=recs, weak=weaks)
    want = [bytes(m) for m in msgs]
    assert [bytes(m) for m in one.take_messages()] == want
    assert [bytes(m) for m in together.take_messages()] == want
    assert one.weak_stats() == together.weak_stats() == wstats and together.recovery_stats() == rstats
    assert together.stats() == stats and wstats["delivered"] > 5


# ---- the rules on hand-made records

_OK = api.EVAL_GATE_OK | api.EVAL_DECODED
_ADDR = bytes.fromhex("4ca1b2")


def _frame(k):
    return synth.make_frame(17, 5, _ADDR + bytes([(11 << 3), k, 2 * k, 3, 4, 5, k ^ 0x55]))


def _records(rows):
    """rows: (t, attempts, recovery, weak) in stream order; attempts: [(frame, crc)]; recovery: None or
    (status, frame, nflips); weak rows have no attempts."""
    cr = [r for r in rows if not r[3]]
    wk = [r for r in rows if r[3]]
    cands = np.zeros(len(cr), dtype=api.CANDIDATE_DTYPE)
    rec = np.zeros(len(cr), dtype=api.RECOVERED_DTYPE)
    wt = np.array([r[0] for r in wk], dtype=np.uint32)
    wr = np.zeros(len(wk), dtype=api.RECOVERED_DTYPE)
    for i, (t, attempts, r, _) in enumerate(cr):
        cands[i]["t"] = t
        p = cands[i]["p"]
        for k, (frame, crc) in enumerate(attempts):
            p["msg"][k] = list(frame)
            p["msgtype"][k] = frame[0] >> 3
            p["flags"][k] = _OK | (api.EVAL_P2_VALID if k else 0)
            p["errorbit"][k] = 255
            p["crc"][k] = crc
        cands[i]["p"] = p
        if r is not None:
            rec[i]["status"], frame, rec[i]["nflips"] = r
            rec[i]["msg"] = list(frame)
            rec[i]["signal"] = 1000 + i
    for i, (_, _, r, _) in enumerate(wk):
        wr[i]["status"], frame, wr[i]["nflips"] = r
        wr[i]["msg"] = list(frame)
        wr[i]["signal"] = 2000 + i
    return cands, rec, wt, wr


def _run(cands, rec, wt, wr, nbuf=1, **cfg):
    res = api.Resolver(**cfg)
    res.run(cands, R.tiled(cands, nbuf), recovered=rec, weak=(wt, wr))
    got = [(int(m.sample_pos) + 238, bytes(m.msg).hex(), int(m.crcok), int(m.recovered)) for m in res.take_messages()]
    off = api.Resolver(**cfg)
    off.run(cands, R.tiled(cands, nbuf))
    want, st, wst = W.model(off.take_messages(), cands, rec, wt, wr, cfg.get("check_crc", 1))
    assert (res.recovery_stats(), res.weak_stats()) == (st, wst)
    return got, res.recovery_stats(), res.weak_stats()


def test_weak_and_strict_recoveries_share_rules_3_and_6():
    bad = (_frame(9), 0x123)
    F = api.RECOVER_FOUND
    rows = [(1000, [(_frame(0), 0)], None, False),                       # a clean frame: the address is known
            (1100, [], (F, _frame(7), 1), True),                         # inside the clean frame's span: not visited
            (2000, [], (F, _frame(1), 2), True),                         # weak recovery ...
            (2100, [bad], (F, _frame(2), 1), False),                     # ... a strict one inside its span: rule 3
            (2300, [bad], (F, _frame(3), 1), False),                     # strict recovery after the span
            (2400, [], (F, _frame(4), 1), True),                         # weak inside the strict span: rule 3
            (2500, [(_frame(5), 0)], None, False),                       # good: rule 6 drops the strict one at 2300
            (4000, [], (F, _frame(6), 1), True),                         # weak recovery ...
            (4100, [(_frame(8), 0)], None, False),                       # ... dropped by rule 6
            (6000, [], (api.RECOVER_AMBIGUOUS, _frame(9), 3), True),
            (7000, [], (F, synth.make_frame(17, 5, bytes.fromhex("aaaaaa") + bytes(7)), 1), True),
            (131072 + 5, [], (F, _frame(10), 1), True)]                  # opens buffer 1
    cands, rec, wt, wr = _records(rows)
    for cfg in (dict(), dict(check_crc=0)):
        got, st, wst = _run(cands, rec, wt, wr, nbuf=2, **cfg)
        assert [(m[0], m[3]) for m in got if m[3]] == [(2000, 2), (131072 + 5, 2)], cfg
        assert wst == dict(considered=6, found=4, ambiguous=1, unknown_address=1, dropped=1, delivered=2)
        assert st == dict(considered=2, found=1, ambiguous=0, unknown_address=0, dropped=1, delivered=0)


def test_weak_list_is_checked():
    cands, rec, wt, wr = _records([(1000, [(_frame(0), 0)], None, False), (2000, [], (1, _frame(1), 1), True),
                                   (3000, [], (1, _frame(2), 1), True)])
    with pytest.raises(ValueError):
        api.Resolver().run(cands, R.tiled(cands, 1), recovered=rec, weak=(wt[::-1], wr))
    with pytest.raises(ValueError):
        api.Resolver().run(cands, R.tiled(cands, 1), recovered=rec, weak=(wt, wr[:1]))
    with pytest.raises(ValueError):
        api.Resolver().run(cands, R.tiled(cands, 1), weak=(wt, wr))


def test_c_host_option_parses(tmp_path):
    r = subprocess.run([str(ROOT / "dump1090-b200"), "--recover-weak", "--ifile", str(tmp_path / "missing")],
                       capture_output=True, text=True)
    assert r.returncode == 1 and "Unknown" not in r.stderr and "Opening data file" in r.stderr
    path = tmp_path / "x.bin"
    np.full(BUF, 127, np.uint8).tofile(path)
    r = subprocess.run([str(ROOT / "dump1090-b200"), "--ifile", str(path), "--recover-weak", "--gpu-resolve"],
                       capture_output=True, text=True)
    assert r.returncode == 1 and "cannot be combined with --gpu-resolve" in r.stderr and r.stdout == ""


# ---------------------------------------------------------------- GPU


def _padded(data):
    nbuf = data.size // BUF + 1
    p = np.full(nbuf * BUF, 127, dtype=np.uint8)
    p[: data.size] = data
    return p, nbuf


def _gpu_streams():
    yield "modes1", C.modes1()
    for snr in (6, 8, 10, 12):
        yield f"fleet{snr}", _fleet(snr)
    yield "traffic1", synth.random_traffic(300000, 400, 1)
    yield "ties", S.tie_rich(11)
    yield "saturated", synth.random_traffic(300000, 300, 9, amp_range=(120.0, 128.0))
    yield "retry_at_j0", S.retry_at_buffer_start()
    for k, (_, _, d) in enumerate(S.random_alphabet_cases(6)):
        yield f"alphabet{k}", d


GPU_STREAMS = dict(_gpu_streams())


def _assert_records(got, want, what):
    for f in ("msg", "status", "nflips", "signal", "pad"):
        bad = np.flatnonzero((got[f] != want[f]).reshape(got.size, -1).any(axis=1))
        assert bad.size == 0, f"{what}: field {f} differs at {bad[:5].tolist()}"


@pytest.mark.gpu
def test_weak_device_equals_restatement(gpu_decoder_factory, checker_libs):
    total = 0
    for name, data in GPU_STREAMS.items():
        padded, nbuf = _padded(data)
        dec = gpu_decoder_factory()
        launches = dec.launch_count()
        dec.detect_host(padded.ctypes.data, nbuf, None)
        dec.weak_device()
        cands, _ = dec.detect_fetch(nbuf)
        n, t, rec = dec.weak_fetch()
        assert dec.launch_count() - launches == 6, name                  # scan, evaluation; weak scan, order, gather, search
        want = W.weak_positions(data, nbuf)
        assert n == want.size and np.array_equal(t, want), name
        _assert_records(rec, W.weak_records(data, t), name)
        assert np.intersect1d(t, cands["t"].astype(np.uint32)).size == 0, name
        assert (rec["status"] != api.RECOVER_INELIGIBLE).all()
        total += n
    assert total > 1000


@pytest.mark.gpu
def test_weak_device_edges(gpu_decoder_factory, checker_libs):
    """The carry block, j = 131069 of the last buffer, one-buffer batches with a carry, the EOF buffer."""
    data = _fleet(7, 2500)
    padded, nbuf = _padded(data)
    # plant the start of a weak-looking window at the last scanned position of the last buffer and at
    # the first positions of the batch (read from the carry block)
    found_edges = set()
    dec = gpu_decoder_factory()
    for b0 in range(nbuf):
        carry = bytes(padded[b0 * BUF - api.CARRY_BYTES: b0 * BUF]) if b0 else None
        chunk = np.ascontiguousarray(padded[b0 * BUF: (b0 + 1) * BUF])
        dec.detect_host(chunk.ctypes.data, 1, carry)
        dec.weak_device()
        n, t, rec = dec.weak_fetch()
        # the restatement of this one-buffer batch: the carry's samples, then the buffer
        stream = np.concatenate([np.frombuffer(carry, np.uint8) if carry else np.full(api.CARRY_BYTES, 127, np.uint8), chunk])
        M = W.padded_mags(stream[api.CARRY_BYTES:], 1)
        M[: 238] = R.magnitudes(stream[: api.CARRY_BYTES])
        tt = np.arange(131070)
        want = tt[W.conditions(M[tt[:, None] + np.arange(W.WINDOW)[None, :]])[0]].astype(np.uint32)
        assert np.array_equal(t, want), b0
        if n and t[0] < 238:
            found_edges.add("carry")
    assert "carry" in found_edges
    # j = 131069 of every buffer of a batch: a weak window built there by hand
    win = np.full(2 * 30, 127, np.uint8)
    amps = np.zeros(30)
    amps[[0, 2, 7, 9]] = 40
    amps[[4, 11]] = 2
    amps[3] = 45                                                          # m3 > m2: the reference's test fails
    for i, bit in enumerate([1, 0, 0, 0, 1]):                             # DF 17
        amps[16 + 2 * i + (1 - bit)] = 30
    win[0::2] = (127 + amps).astype(np.uint8)
    stream = np.full(3 * BUF, 127, np.uint8)
    for b in range(3):
        s = b * 131072 + 131069 - 238
        stream[2 * s: 2 * s + win.size] = win
    dec.detect_host(stream.ctypes.data, 3, None)
    dec.weak_device()
    n, t, _ = dec.weak_fetch()
    want = W.weak_positions(stream, 3)
    assert np.array_equal(t, want) and {b * 131072 + 131069 for b in range(3)} <= set(t.tolist())
    # the EOF buffer (no drop): what the streaming decode finds equals the restatement of every buffer
    cpu = W.cpu_decode(data, {})
    gpu = gpu_decoder_factory(recover=True, weak_preambles=True)
    gpu.decode(data)
    assert gpu.weak_recovery_stats() == cpu[3]


@pytest.mark.gpu
def test_weak_device_capacity(gpu_decoder_factory, checker_libs):
    """A stream dense in weak positions: the count is exact, a caller's array gets the first positions
    and records and nothing past its capacity, also when the capacity is above the context's first
    scratch list (the batch is then repeated with a larger one); the context's own buffers grow."""
    nbuf = 4
    rng = np.random.default_rng(5)
    data = np.full(nbuf * BUF, 127, np.uint8)
    amps = np.zeros(30)
    amps[[0, 2, 7, 9]] = 40
    amps[3] = 45                                                          # the reference's test fails
    for i, bit in enumerate([1, 0, 0, 1, 0]):                             # DF 18
        amps[16 + 2 * i + (1 - bit)] = 30
    for s in range(0, nbuf * 131072 - 30, 30):
        data[2 * s: 2 * s + 60: 2] = (127 + amps + rng.integers(0, 2, 30)).astype(np.uint8)
    want = W.weak_positions(data, nbuf)
    first_scratch = nbuf * 131072 // 512 + 4096                          # the context's first scratch list
    assert want.size > 3 * first_scratch
    want_rec = W.weak_records(data, want)
    torch = pytest.importorskip("torch")
    d_iq = torch.from_numpy(data).cuda()
    sentinel = 1000                                                       # an in-range position
    for cap in (first_scratch - 120, first_scratch + 5000, want.size + 100):
        d_pos = torch.full((cap + 64,), sentinel, dtype=torch.int32, device="cuda")
        d_rec = torch.full(((cap + 64) * 20,), 0xCD, dtype=torch.uint8, device="cuda")
        dec = gpu_decoder_factory()                                       # a fresh context: its first scratch list overflows
        dec.detect_device(d_iq.data_ptr(), nbuf, None)
        dec.weak_device(d_pos.data_ptr(), d_rec.data_ptr(), cap)
        n, t, _ = dec.weak_fetch()
        assert n == want.size and t.size == 0, cap
        torch.cuda.synchronize()
        k = min(cap, want.size)
        pos = d_pos.cpu().numpy().view(np.uint32)
        assert np.array_equal(pos[:k], want[:k]) and (pos[k:] == sentinel).all(), cap
        recs = d_rec.cpu().numpy()
        assert (recs[k * 20:] == 0xCD).all(), cap
        _assert_records(recs[: k * 20].view(api.RECOVERED_DTYPE), want_rec[:k], f"capacity {cap}")
        # own buffers: every position
        dec.detect_device(d_iq.data_ptr(), nbuf, None)
        dec.weak_device()
        n, t, rec = dec.weak_fetch()
        assert n == want.size and np.array_equal(t, want)
        _assert_records(rec, want_rec, "own buffers")


def _compare(dec, cpu, what):
    msgs, stats, rstats, wstats = cpu[:4]
    got = dec.take_messages() if not isinstance(what, list) else what
    assert [bytes(m) for m in got] == [bytes(m) for m in msgs]
    assert (dec.stats(), dec.recovery_stats(), dec.weak_recovery_stats()) == (stats, rstats, wstats)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fleet6", "fleet8", "fleet10", "modes1", "ties", "retry_at_j0"])
@pytest.mark.parametrize("kw", FLAGS, ids=_kid)
def test_decode_equals_cpu_path(name, kw, gpu_decoder_factory, checker_libs):
    data = GPU_STREAMS[name]
    for drop in (0, 1):
        cpu = W.cpu_decode(data, kw, drop_eof=drop)
        for extra in (dict(), dict(max_batch_bytes=BUF)):
            dec = gpu_decoder_factory(recover=True, weak_preambles=True, drop_eof_buffer=drop, **R.flag_cfg(kw), **extra)
            _compare(dec, cpu, dec.decode(data))
            _compare(dec, cpu, dec.decode(data, chunk=100003))
    # the reference's messages and statistics are unchanged
    off = gpu_decoder_factory(**R.flag_cfg(kw))
    got_off = off.decode(data)
    on = gpu_decoder_factory(recover=True, weak_preambles=True, **R.flag_cfg(kw))
    got_on = on.decode(data)
    assert [bytes(m) for m in got_on if not m.recovered] == [bytes(m) for m in got_off] and on.stats() == off.stats()


@pytest.mark.gpu
def test_signal_on(gpu_decoder_factory, checker_libs):
    data = GPU_STREAMS["fleet8"]
    cpu = W.cpu_decode(data, {}, signal=True)
    dec = gpu_decoder_factory(recover=True, weak_preambles=True, signal=True)
    got = dec.decode(data)
    want = cpu[0]
    assert len(got) == len(want) and sum(m.recovered == 2 for m in got) > 5
    for g, w in zip(got, want):
        if w.recovered:
            assert bytes(g) == bytes(w) and g.signal > 0
        else:
            c = g.copy()
            c.signal = 0
            assert bytes(c) == bytes(w)
    assert dec.weak_recovery_stats() == cpu[3]


@pytest.mark.gpu
def test_launches_and_bytes_with_the_switch_off(gpu_decoder_factory, checker_libs):
    data = GPU_STREAMS["fleet8"]
    nb = data.size // BUF + 1
    plain = gpu_decoder_factory(recover=True, max_batch_bytes=BUF)
    got = plain.decode(data)
    off = gpu_decoder_factory(recover=True, weak_preambles=False, max_batch_bytes=BUF)
    off.set_weak_preambles(False)
    assert [bytes(m) for m in off.decode(data)] == [bytes(m) for m in got] and off.launch_count() == plain.launch_count()
    # weak preambles without recovery do nothing
    alone = gpu_decoder_factory(weak_preambles=True, max_batch_bytes=BUF)
    ref = gpu_decoder_factory(max_batch_bytes=BUF)
    assert [bytes(m) for m in alone.decode(data)] == [bytes(m) for m in ref.decode(data)]
    assert alone.launch_count() == ref.launch_count()
    on = gpu_decoder_factory(recover=True, weak_preambles=True, max_batch_bytes=BUF)
    on.decode(data)
    assert on.launch_count() == plain.launch_count() + 4 * nb                # four more launches per batch


@pytest.mark.gpu
def test_switch_between_batches_and_reset(gpu_decoder_factory, checker_libs):
    data = np.concatenate([GPU_STREAMS["fleet8"], GPU_STREAMS["fleet10"]])
    cut = 3 * BUF
    cpu = W.cpu_decode(data, {})
    dec = gpu_decoder_factory(recover=True, max_batch_bytes=BUF)
    dec.reset()
    dec.process(data[:cut])
    dec.set_weak_preambles(True)
    dec.process(data[cut:])
    dec.finish()
    got = dec.take_messages()
    keep = [m for m in cpu[0] if m.recovered != 2 or (m.sample_pos + 238) >> 17 >= 3]
    # a weak recovery in buffers 0..2 may have taken a span from a strict one: compare buffers 3.. only
    late = lambda ms: [bytes(m) for m in ms if (m.sample_pos + 238) >> 17 >= 3]
    assert late(got) == late(keep) and sum(m.recovered == 2 for m in got) > 0
    dec.reset()
    dec.process(data[: cut + 5000])
    dec.reset()
    _compare(dec, cpu, dec.decode(data))


@pytest.mark.gpu
def test_refused_with_gpu_resolve(gpu_decoder_factory):
    dec = gpu_decoder_factory(gpu_resolve=1)
    with pytest.raises(RuntimeError, match="gpu_resolve"):
        dec.set_weak_preambles(True)
    with pytest.raises(RuntimeError, match="gpu_resolve"):
        gpu_decoder_factory(gpu_resolve=1, weak_preambles=True)
    dec.set_weak_preambles(False)
    got = dec.decode(GPU_STREAMS["fleet8"])
    assert all(m.recovered == 0 for m in got) and dec.weak_recovery_stats()["considered"] == 0


@pytest.mark.gpu
def test_two_gpus(gpu_decoder_factory, checker_libs):
    data = np.concatenate([GPU_STREAMS["fleet8"], GPU_STREAMS["fleet10"], GPU_STREAMS["traffic1"]])
    for kw in (dict(), dict(check_crc=0, aggressive=1)):
        cpu = W.cpu_decode(data, kw)
        dec = gpu_decoder_factory(recover=True, weak_preambles=True, n_gpus=2, max_batch_bytes=2 * BUF, **R.flag_cfg(kw))
        _compare(dec, cpu, dec.decode(data))


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(), dict(check_crc=0)], ids=_kid)
def test_pool_equals_single_stream(kw, gpu_decoder_factory, checker_libs):
    n_rx = 4
    streams = []
    for r in range(n_rx):
        d, _ = synth.fleet_at(7 + r, 1000 + 300 * r, 500 + r)
        streams.append(d[: (d.size // BUF) * BUF])
    rng = np.random.default_rng(9)
    with api.ReceiverPool(n_rx, recover=True, weak_preambles=True, **R.flag_cfg(kw)) as pool:
        pos = [0] * n_rx
        inflight = 0
        while any(pos[r] < streams[r].size for r in range(n_rx)):
            ids = [r for r in range(n_rx) if pos[r] < streams[r].size and rng.random() < 0.7]
            if not ids:
                continue
            pool.submit(ids, [streams[r][pos[r]: pos[r] + BUF] for r in ids])
            for r in ids:
                pos[r] += BUF
            inflight += 1
            if inflight == 2:
                pool.collect()
                inflight -= 1
        while inflight:
            pool.collect()
            inflight -= 1
        total = 0
        for r in range(n_rx):
            dec = gpu_decoder_factory(recover=True, weak_preambles=True, drop_eof_buffer=1, **R.flag_cfg(kw))
            want = dec.decode(streams[r])
            got = pool.take(r)
            assert [bytes(m) for m in got] == [bytes(m) for m in want], r
            assert pool.weak_recovery_stats(r) == dec.weak_recovery_stats() and pool.recovery_stats(r) == dec.recovery_stats()
            assert pool.stats(r) == dec.stats()
            total += sum(m.recovered == 2 for m in got)
        assert total > 5
        pool.reset(0)
        assert pool.weak_recovery_stats(0)["considered"] == 0


@pytest.mark.gpu
def test_c_host_recover_weak(gpu_decoder_factory, checker_libs, tmp_path):
    data = np.concatenate([GPU_STREAMS["fleet8"], GPU_STREAMS["fleet10"]])
    path = tmp_path / "fleet.bin"
    data.tofile(path)
    exe = str(ROOT / "dump1090-b200")
    dec = gpu_decoder_factory(recover=True, weak_preambles=True)
    msgs = dec.decode(data)
    assert sum(m.recovered == 2 for m in msgs) > 5
    raw = subprocess.run([exe, "--ifile", str(path), "--recover-weak", "--raw"], capture_output=True, text=True, check=True)
    assert raw.stdout.splitlines() == [m.raw_line() for m in msgs]
    st = subprocess.run([exe, "--ifile", str(path), "--recover-weak", "--stats"], capture_output=True, text=True, check=True)
    lines = st.stderr.strip().splitlines()
    fmt = "{considered} considered, {found} found, {ambiguous} ambiguous, {unknown_address} unknown address, " \
          "{dropped} dropped, {delivered} delivered"
    assert lines == ["recovery: " + fmt.format(**dec.recovery_stats()), "weak preambles: " + fmt.format(**dec.weak_recovery_stats())]
