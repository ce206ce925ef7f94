"""Soft-decision recovery of weak DF17/DF18 frames of known aircraft (modes_set_recovery,
modes_recover_device, modes_resolver_run_recovered, modes_pool_set_recovery).

The reference computations are in tests/recover_model.py: a numpy restatement of the recovery
record from the raw stream bytes, and a Python model of the resolve rules 1-6 of include/modes_b200.h
that derives the skip states and the address cache from the recovery-off decode.  CPU tests cover the
arithmetic (host build of modes_recover_core.cuh), the host resolve's rules and the ground truth; GPU
tests the kernel and every decode path."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import checker as C
import edge_corpora as E
import recover_model as R
import streams as S
from dump1090_b200 import api, synth

ROOT = C.ROOT
SHIM = ROOT / "tests" / "_build" / "librecover_core_host.so"
BUF = api.BUFFER_BYTES
FLAGS = [dict(), dict(aggressive=1), dict(fix=0), dict(check_crc=0)]


def _kid(k):
    return "-".join(f"{a}{b}" for a, b in k.items()) or "default"


# ---------------------------------------------------------------- CPU: arithmetic


@pytest.fixture(scope="module")
def shim():
    subprocess.run(["make", "-s", "shim"], cwd=ROOT, check=True)
    lib = ctypes.CDLL(str(SHIM))
    lib.shim_recover.restype = ctypes.c_int
    lib.shim_recover.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    return lib


def _shim_records(shim, wins):
    wins = np.ascontiguousarray(wins, dtype=np.uint8).reshape(-1, 448)
    out = np.zeros(wins.shape[0], dtype=api.RECOVERED_DTYPE)
    assert shim.shim_recover(wins.ctypes.data, wins.shape[0], out.ctypes.data) == 0
    return out


_restated = E.restated


def _assert_same(got, want, what):
    for f in ("msg", "status", "nflips", "signal", "pad"):
        bad = np.flatnonzero((got[f] != want[f]).reshape(got.size, -1).any(axis=1))
        assert bad.size == 0, f"{what}: field {f} differs at {bad[:5].tolist()}"


def test_shim_equals_restatement_on_random_windows(shim):
    cases = E.recover_random_windows()
    for name, wins in cases.items():
        _assert_same(_shim_records(shim, wins), _restated(wins), name)
    assert (_restated(cases["all_equal_df17"])["status"] != api.RECOVER_INELIGIBLE).all()


def test_clean_and_repaired_frames(shim):
    wins, sent, expect = E.recover_frame_windows()
    got = _shim_records(shim, wins)
    want = _restated(wins)
    _assert_same(got, want, "frames")
    assert (want["status"] == api.RECOVER_FOUND).all()
    same = np.array([bytes(r["msg"]) == f for r, f in zip(want, sent)])
    # the sent frame, unless the restatement finds a lighter solution inside the ten positions
    lighter = want["nflips"] < np.array(expect)
    assert (same | lighter).all() and same.mean() > 0.95
    assert (want["nflips"][same] == np.array(expect)[same]).all()


def test_confident_error_and_other_formats(shim):
    wins = E.recover_confident_windows()                                 # a confident bit wrong; other formats
    got, want = _shim_records(shim, wins), _restated(wins)
    _assert_same(got, want, "confident/other")
    assert (want["status"][:40] != api.RECOVER_FOUND).sum() >= 35
    assert (want["status"][40:] == api.RECOVER_INELIGIBLE).all()


def test_constructed_ambiguity(shim):
    """Three bits of a weight-6 codeword flipped, its six positions among the ten least confident:
    two solutions of weight 3."""
    wins = E.recover_ambiguity_windows()
    assert len(wins) == 155
    got, want = _shim_records(shim, wins), _restated(wins)
    _assert_same(got, want, "ambiguity")
    assert (want["status"] == api.RECOVER_AMBIGUOUS).all() and (want["nflips"] == 3).all()


# ---------------------------------------------------------------- CPU: the resolve rules


def _fleet(snr, n=1500):
    return synth.fleet_at(snr, n, 2000 + snr)


def _cpu_streams():
    yield "modes1", C.modes1()
    for seed in (1, 2):
        yield f"traffic{seed}", synth.random_traffic(300000, 400, seed)
    for snr in (8, 10, 14):
        yield f"fleet{snr}", _fleet(snr)[0]


CPU_STREAMS = dict(_cpu_streams())


def _off_run(arr, tiles, kw):
    res = api.Resolver(**R.flag_cfg(kw))
    res.run(arr, tiles)
    return res.take_messages(), res.stats()


@pytest.mark.parametrize("name", list(CPU_STREAMS))
@pytest.mark.parametrize("kw", FLAGS, ids=_kid)
def test_resolve_rule_equals_model(name, kw, checker_libs, monkeypatch):
    data = CPU_STREAMS[name]
    msgs, stats, rstats, arr, rec = R.cpu_decode(data, kw, signal=True)
    tiles = R.tiled(arr, data.size // BUF + 1)
    off, off_stats = _off_run(arr, tiles, kw)
    # the reference's messages and counters are untouched
    assert [bytes(m) for m in msgs if not m.recovered] == [bytes(m) for m in off]
    assert stats == off_stats
    want, want_stats = R.model(off, arr, rec, kw.get("check_crc", 1))
    got = [(int(m.sample_pos), bytes(m.msg), int(m.nfixed), int(m.signal)) if m.recovered else bytes(m) for m in msgs]
    assert got == [w if isinstance(w, tuple) else bytes(w) for w in want]
    assert rstats == want_stats
    recd = [m for m in msgs if m.recovered]
    if name.startswith("fleet") and name != "fleet14":
        assert len(recd) > 5
    # a recovered message is a clean frame through the reference's own field decode
    if recd:
        frames = np.array([list(m.msg) for m in recd], dtype=np.uint8)
        ref, _ = C.oracle_decode_frames(frames)
        for m, r in zip(recd, ref):
            assert C.msg_fields(m) == C.msg_fields(r)
            assert (m.crcok, m.crc, m.errorbit, m.phase_corrected, m.iid, m.recovered) == (1, 0, -1, 0, 0, 1)
            assert m.msgtype in (17, 18) and m.nfixed <= api.RECOVER_BITS
    # with no FOUND record nothing changes
    none = rec.copy()
    none["status"] = np.where(none["status"] == api.RECOVER_FOUND, api.RECOVER_NOT_FOUND, none["status"])
    res = api.Resolver(**R.flag_cfg(kw))
    res.run(arr, tiles, recovered=none)
    assert [bytes(m) for m in res.take_messages()] == [bytes(m) for m in off] and res.stats() == off_stats
    assert res.recovery_stats()["delivered"] == 0
    # the parts of a long record array are judged concurrently: the same messages and statistics
    for parts, part_tiles in (("1", None), ("4", "8")):
        monkeypatch.setenv("MODES_RESOLVE_PARTS", parts)
        if part_tiles:
            monkeypatch.setenv("MODES_RESOLVE_PART_TILES", part_tiles)
        res = api.Resolver(**R.flag_cfg(kw))
        res.run(arr, tiles, recovered=rec)
        assert [bytes(m) for m in res.take_messages()] == [bytes(m) for m in msgs], parts
        assert res.recovery_stats() == rstats and res.stats() == stats


def test_ground_truth_fleet_sweep(checker_libs):
    """Every recovered frame was transmitted; the low-SNR points keep recovering (minimum counts pinned
    so that a generator change cannot hollow the test out)."""
    floor = {8: 10, 10: 25}
    for snr in (6, 8, 10, 12, 15):
        data, truth = synth.fleet_at(snr, 2000, 1000 + snr)
        msgs, _, rstats, _, _ = R.cpu_decode(data, dict(aggressive=1))
        recd = [m.hex() for m in msgs if m.recovered]
        assert all(h in truth for h in recd), snr
        assert len(recd) >= floor.get(snr, 0), (snr, len(recd), rstats)


def test_ground_truth_random_traffic(checker_libs):
    n = 0
    for seed in (31, 32, 33):
        data, truth = synth.random_traffic(131072 * 6, 1500, seed, amp_range=(8.0, 40.0), sigma=4.0, max_flips=0,
                                           return_truth=True)
        sent = {f.hex() for _, f, _ in truth}
        for kw in (dict(), dict(aggressive=1)):
            msgs, *_ = R.cpu_decode(data, kw)
            recd = [m.hex() for m in msgs if m.recovered]
            assert all(h in sent for h in recd), (seed, kw)
            n += len(recd)
    assert n >= 10


def test_c_host_option_parses(tmp_path):
    """--recover is an option of the C host (decoding needs the GPU; an unreadable file fails first)."""
    r = subprocess.run([str(ROOT / "dump1090-b200"), "--recover", "--ifile", str(tmp_path / "missing")],
                       capture_output=True, text=True)
    assert r.returncode == 1 and "Unknown" not in r.stderr and "Opening data file" in r.stderr


def test_c_host_refuses_recover_with_gpu_resolve(tmp_path):
    """The refusal comes before any file or device is touched."""
    path = tmp_path / "x.bin"
    np.full(BUF, 127, np.uint8).tofile(path)
    for args in (["--recover", "--gpu-resolve"], ["--gpu-resolve", "--raw", "--recover"]):
        r = subprocess.run([str(ROOT / "dump1090-b200"), "--ifile", str(path), *args], capture_output=True, text=True)
        assert r.returncode == 1 and "--recover cannot be combined with --gpu-resolve" in r.stderr
        assert r.stdout == ""


# ---- the rules on hand-made records

_OK = api.EVAL_GATE_OK | api.EVAL_DECODED
_ADDR = bytes.fromhex("4ca1b2")


def _frame(k):
    return synth.make_frame(17, 5, _ADDR + bytes([(11 << 3), k, 2 * k, 3, 4, 5, k ^ 0x55]))


def _records(rows):
    """rows: (j, attempts, recovery) in stream order, buffer 0; attempts: [(frame, crc)] for pass 0 and 1;
    recovery: None or (status, frame, nflips)."""
    cands = np.zeros(len(rows), dtype=api.CANDIDATE_DTYPE)
    rec = np.zeros(len(rows), dtype=api.RECOVERED_DTYPE)
    for i, (j, attempts, r) in enumerate(rows):
        cands[i]["t"] = j
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
    return cands, rec


def _run(cands, rec, **cfg):
    res = api.Resolver(**cfg)
    res.run(cands, R.tiled(cands, 1), recovered=rec)
    return [(int(m.sample_pos) + 238, bytes(m.msg).hex(), int(m.crcok), int(m.recovered)) for m in res.take_messages()], \
        res.recovery_stats(), res.stats()


def _expect_model(cands, rec, cfg):
    off = api.Resolver(**cfg)
    off.run(cands, R.tiled(cands, 1))
    _, want = R.model(off.take_messages(), cands, rec, cfg.get("check_crc", 1))
    return want


def test_rule6_drops_inside_the_span_and_keeps_the_order():
    bad = (_frame(9), 0x123)
    rows = [(1000, [(_frame(0), 0)], None),                                  # a clean frame: the address is known
            (2000, [bad, bad], (api.RECOVER_FOUND, _frame(1), 3)),            # recovered ...
            (2050, [bad, bad], None),
            (2100, [(_frame(2), 0)], None)]                                   # ... and the reference decodes within 241
    cands, rec = _records(rows)
    for cfg in (dict(), dict(check_crc=0)):
        msgs, st, _ = _run(cands, rec, **cfg)
        assert not any(m[3] for m in msgs), cfg
        assert st == dict(considered=1, found=1, ambiguous=0, unknown_address=0, dropped=1, delivered=0)
        assert st == _expect_model(cands, rec, cfg)
        off = api.Resolver(**cfg)
        off.run(cands, R.tiled(cands, 1))
        assert [m[:3] for m in msgs] == [(int(m.sample_pos) + 238, bytes(m.msg).hex(), int(m.crcok)) for m in off.take_messages()]
    # with check_crc = 0 the failed attempts at 2000 and 2050 are delivered, in order, before the good one
    msgs, _, _ = _run(cands, rec, check_crc=0)
    assert [m[0] for m in msgs] == [1000, 2000, 2000, 2050, 2050, 2100]


def test_rule6_keeps_at_the_end_of_the_span():
    bad = (_frame(9), 0x123)
    rows = [(1000, [(_frame(0), 0)], None),
            (2000, [bad], (api.RECOVER_FOUND, _frame(1), 2)),
            (2000 + 240, [bad], None),
            (2000 + 241, [(_frame(2), 0)], None)]
    cands, rec = _records(rows)
    for cfg in (dict(), dict(check_crc=0)):
        msgs, st, _ = _run(cands, rec, **cfg)
        assert [m for m in msgs if m[3]] == [(2000, _frame(1).hex(), 1, 1)]
        assert st["dropped"] == 0 and st["delivered"] == 1 and st == _expect_model(cands, rec, cfg)
        # the recovered message comes before the later deliveries
        assert [m[0] for m in msgs] == sorted(m[0] for m in msgs)
    msgs, _, _ = _run(cands, rec, check_crc=0)
    assert [m[0] for m in msgs] == [1000, 2000, 2000, 2240, 2241]          # three at 2000: two attempts + recovered
    assert [m[3] for m in msgs] == [0, 0, 1, 0, 0]


def test_ambiguous_and_rule3():
    bad = (_frame(9), 0x123)
    rows = [(1000, [(_frame(0), 0)], None),
            (1500, [bad], (api.RECOVER_AMBIGUOUS, _frame(9), 3)),            # counted, nothing delivered
            (2000, [bad], (api.RECOVER_FOUND, _frame(1), 1)),                # delivered
            (2100, [bad], (api.RECOVER_FOUND, _frame(2), 1)),                # inside its span: rule 3
            (2100 + 140, [bad], (api.RECOVER_AMBIGUOUS, _frame(9), 3)),      # inside too: not counted as ambiguous
            (2241, [bad], (api.RECOVER_FOUND, _frame(3), 2)),                # first position after the span
            (2241 + 241, [], (api.RECOVER_FOUND, _frame(4), 1)),             # gate failed: still visited
            (5000, [bad], (api.RECOVER_FOUND, synth.make_frame(17, 5, bytes.fromhex("aaaaaa") + bytes(7)), 1)),
            (6000, [bad], (api.RECOVER_NOT_FOUND, _frame(9), 0)),
            (7000, [(bytes([11 << 3]) + bytes(13), 5)], (api.RECOVER_INELIGIBLE, bytes([11 << 3]) + bytes(13), 0))]
    cands, rec = _records(rows)
    cands[6]["p"]["flags"] = 0                                                # no attempt passes the gate
    for cfg in (dict(), dict(check_crc=0), dict(aggressive=1)):
        msgs, st, _ = _run(cands, rec, **cfg)
        assert [m[0] for m in msgs if m[3]] == [2000, 2241, 2482], cfg
        assert st == dict(considered=8, found=4, ambiguous=1, unknown_address=1, dropped=0, delivered=3)
        assert st == _expect_model(cands, rec, cfg)
    # a new buffer resets the span
    rows2 = rows[:3] + [(131072 + 10, [bad], (api.RECOVER_FOUND, _frame(5), 1))]
    cands, rec = _records(rows2)
    res = api.Resolver()
    res.run(cands, R.tiled(cands, 2), recovered=rec)
    assert [int(m.sample_pos) + 238 for m in res.take_messages() if m.recovered] == [2000, 131072 + 10]


def test_recovery_record_count_is_checked():
    cands, rec = _records([(1000, [(_frame(0), 0)], None), (2000, [], None)])
    with pytest.raises(ValueError):
        api.Resolver().run(cands, R.tiled(cands, 1), recovered=rec[:1])


@pytest.mark.parametrize("kw", [dict(), dict(check_crc=0)], ids=_kid)
def test_shards_equal_the_run_shard_by_shard(kw, checker_libs):
    data = np.concatenate([_fleet(8)[0], _fleet(10)[0], synth.random_traffic(131072 * 3, 600, 5)])
    msgs, stats, rstats, arr, rec = R.cpu_decode(data, kw, signal=True)
    nbuf = data.size // BUF + 1
    cut = [0, 2, 5, 6, nbuf]
    shards, recs = [], []
    for a, b in zip(cut[:-1], cut[1:]):
        sel = ((arr["t"] >> 17) >= a) & ((arr["t"] >> 17) < b)
        c = arr[sel].copy()
        c["t"] -= a << 17
        shards.append((c, R.tiled(c, b - a), a))
        recs.append(rec[sel].copy())
    one = api.Resolver(**R.flag_cfg(kw))
    for (c, t, b), r in zip(shards, recs):
        one.run(c, t, b, recovered=r)
    together = api.Resolver(**R.flag_cfg(kw))
    together.run_shards(shards, recovered=recs)
    want = [bytes(m) for m in msgs]
    assert [bytes(m) for m in one.take_messages()] == want
    assert [bytes(m) for m in together.take_messages()] == want
    assert one.recovery_stats() == together.recovery_stats() == rstats and together.stats() == stats
    assert rstats["delivered"] > 10


# ---------------------------------------------------------------- GPU


def _padded(data):
    nbuf = data.size // BUF + 1
    p = np.full(nbuf * BUF, 127, dtype=np.uint8)
    p[: data.size] = data
    return p, nbuf


def _gpu_streams():
    yield "modes1", C.modes1()
    for seed in (1, 2, 3):
        yield f"traffic{seed}", synth.random_traffic(300000, 400, seed)
    yield "ties", S.tie_rich(11)
    yield "saturated", synth.random_traffic(300000, 300, 9, amp_range=(120.0, 128.0))
    yield "retry_at_j0", S.retry_at_buffer_start()
    for snr in (8, 10, 14):
        yield f"fleet{snr}", _fleet(snr)[0]


GPU_STREAMS = dict(_gpu_streams())


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["default", "warp"])
def test_records_equal_restatement(variant, gpu_decoder_factory, checker_libs, monkeypatch):
    if variant != "default":
        monkeypatch.setenv("MODES_EVAL_VARIANT", variant)
    cases = list(GPU_STREAMS.items()) + [(f"alphabet{k}", d) for k, (_, _, d) in enumerate(S.random_alphabet_cases())]
    eligible = 0
    for name, data in cases:
        padded, nbuf = _padded(data)
        dec = gpu_decoder_factory(aggressive=1)
        launches = dec.launch_count()
        dec.detect_host(padded.ctypes.data, nbuf, None)
        dec.recover_device()
        cands, _ = dec.detect_fetch(nbuf)
        got = dec.recover_fetch()
        assert dec.launch_count() - launches == 3
        assert got.size == cands.size
        _assert_same(got, R.restate_records(data, cands["t"]), name)
        eligible += int((got["status"] != api.RECOVER_INELIGIBLE).sum())
    assert eligible > 1000


def _compare(got_msgs, got_stats, got_rstats, cpu, what):
    msgs, stats, rstats = cpu[:3]
    assert [bytes(m) for m in got_msgs] == [bytes(m) for m in msgs], what
    assert got_stats == stats and got_rstats == rstats, what


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(GPU_STREAMS))
@pytest.mark.parametrize("kw", FLAGS, ids=_kid)
def test_decode_equals_cpu_path(name, kw, gpu_decoder_factory, checker_libs):
    data = GPU_STREAMS[name]
    off = gpu_decoder_factory(**R.flag_cfg(kw))
    got_off = off.decode(data)
    for drop in (0, 1):
        cpu = R.cpu_decode(data, kw, drop_eof=drop)
        for extra in (dict(), dict(max_batch_bytes=BUF)):
            dec = gpu_decoder_factory(recover=True, drop_eof_buffer=drop, **R.flag_cfg(kw), **extra)
            _compare(dec.decode(data), dec.stats(), dec.recovery_stats(), cpu, (drop, extra))
            _compare(dec.decode(data, chunk=100003), dec.stats(), dec.recovery_stats(), cpu, (drop, extra, "chunked"))
    on = gpu_decoder_factory(recover=True, **R.flag_cfg(kw))
    got_on = on.decode(data)
    assert [bytes(m) for m in got_on if not m.recovered] == [bytes(m) for m in got_off]
    assert on.stats() == off.stats()


@pytest.mark.gpu
def test_launches_and_bytes_with_the_switch_off(gpu_decoder_factory, checker_libs):
    data = GPU_STREAMS["fleet10"]
    plain = gpu_decoder_factory(max_batch_bytes=BUF)
    got = plain.decode(data)
    n_plain = plain.launch_count()
    off = gpu_decoder_factory(recover=False, max_batch_bytes=BUF)
    off.set_recovery(False)
    assert [bytes(m) for m in off.decode(data)] == [bytes(m) for m in got]
    assert off.launch_count() == n_plain and all(m.recovered == 0 for m in got)
    on = gpu_decoder_factory(recover=True, max_batch_bytes=BUF)
    on.decode(data)
    assert on.launch_count() == n_plain + data.size // BUF + 1                # one more launch per batch


@pytest.mark.gpu
def test_switch_between_batches_and_reset(gpu_decoder_factory, checker_libs):
    data = np.concatenate([GPU_STREAMS["fleet8"], GPU_STREAMS["fleet10"]])
    cut = 3 * BUF
    cpu = R.cpu_decode(data, {})
    msgs_cpu = cpu[0]
    dec = gpu_decoder_factory(max_batch_bytes=BUF)
    dec.reset()
    dec.process(data[:cut])
    dec.set_recovery(True)
    dec.process(data[cut:])
    dec.finish()
    got = dec.take_messages()
    # buffers 0..2 were decoded without recovery: the CPU path's recovered messages from buffer 3 on
    keep = [m for m in msgs_cpu if not m.recovered or (m.sample_pos + 238) >> 17 >= 3]
    assert [bytes(m) for m in got] == [bytes(m) for m in keep]
    # a reset in the middle of a stream: the next decode starts clean
    dec.reset()
    dec.process(data[: cut + 5000])
    dec.reset()
    _compare(dec.decode(data), dec.stats(), dec.recovery_stats(), cpu, "after reset")


@pytest.mark.gpu
def test_signal_and_levels_on(gpu_decoder_factory, checker_libs):
    data = GPU_STREAMS["fleet10"]
    cpu = R.cpu_decode(data, {}, signal=True)
    dec = gpu_decoder_factory(recover=True, signal=True, levels=True)
    got = dec.decode(data)
    assert len(dec.take_levels()) == data.size // BUF + 1
    want = cpu[0]
    assert len(got) == len(want)
    for g, w in zip(got, want):
        if w.recovered:
            assert bytes(g) == bytes(w) and g.signal > 0                   # the record's signal, as restated
        else:
            c = g.copy()
            c.signal = 0
            assert bytes(c) == bytes(w)
    assert dec.recovery_stats() == cpu[2] and cpu[2]["delivered"] > 5


@pytest.mark.gpu
def test_two_gpus(gpu_decoder_factory, checker_libs):
    data = np.concatenate([GPU_STREAMS["fleet8"], GPU_STREAMS["fleet10"], GPU_STREAMS["traffic1"]])
    for kw in (dict(), dict(check_crc=0, aggressive=1)):
        cpu = R.cpu_decode(data, kw)
        dec = gpu_decoder_factory(recover=True, n_gpus=2, max_batch_bytes=2 * BUF, **R.flag_cfg(kw))
        _compare(dec.decode(data), dec.stats(), dec.recovery_stats(), cpu, kw)


@pytest.mark.gpu
def test_refused_with_gpu_resolve(gpu_decoder_factory):
    dec = gpu_decoder_factory(gpu_resolve=1)
    with pytest.raises(RuntimeError, match="gpu_resolve"):
        dec.set_recovery(True)
    with pytest.raises(RuntimeError, match="gpu_resolve"):
        gpu_decoder_factory(gpu_resolve=1, recover=True)
    dec.set_recovery(False)
    assert dec.recovery_stats()["considered"] == 0
    got = dec.decode(GPU_STREAMS["fleet10"])
    assert all(m.recovered == 0 for m in got)


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(), dict(check_crc=0)], ids=_kid)
def test_pool_equals_single_stream(kw, gpu_decoder_factory, checker_libs):
    """Receivers out of lock step, two batches in flight: each receiver's messages and recovery
    statistics equal a single-stream decode of its own stream.  Without the CRC check a candidate can
    deliver three messages (both failed attempts and a recovered one)."""
    n_rx = 4
    streams = []
    for r in range(n_rx):
        d, _ = synth.fleet_at(8 + 2 * r, 1000 + 300 * r, 500 + r)
        streams.append(d[: (d.size // BUF) * BUF])
    rng = np.random.default_rng(9)
    with api.ReceiverPool(n_rx, recover=True, **R.flag_cfg(kw)) as pool:
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
        total = triples = 0
        for r in range(n_rx):
            dec = gpu_decoder_factory(recover=True, drop_eof_buffer=1, **R.flag_cfg(kw))
            want = dec.decode(streams[r])
            got = pool.take(r)
            assert [bytes(m) for m in got] == [bytes(m) for m in want], r
            assert pool.recovery_stats(r) == dec.recovery_stats() and pool.stats(r) == dec.stats()
            total += sum(m.recovered for m in got)
            pos = [m.sample_pos for m in got]
            triples += sum(1 for m in got if m.recovered and pos.count(m.sample_pos) == 3)
        assert total > 10
        if kw.get("check_crc", 1) == 0:
            assert triples > 5
        pool.reset(0)
        assert pool.recovery_stats(0)["considered"] == 0


@pytest.mark.gpu
def test_c_host_recover(gpu_decoder_factory, checker_libs, tmp_path):
    data = np.concatenate([GPU_STREAMS["fleet8"], GPU_STREAMS["fleet10"]])
    path = tmp_path / "fleet.bin"
    data.tofile(path)
    exe = str(ROOT / "dump1090-b200")
    msgs = gpu_decoder_factory(recover=True).decode(data)
    assert sum(m.recovered for m in msgs) > 10
    raw = subprocess.run([exe, "--ifile", str(path), "--recover", "--raw"], capture_output=True, text=True, check=True)
    assert raw.stdout.splitlines() == [m.raw_line() for m in msgs]
    with_signal = gpu_decoder_factory(recover=True, signal=True).decode(data)
    beast = subprocess.run([exe, "--ifile", str(path), "--recover", "--beast"], capture_output=True, check=True)
    assert beast.stdout == b"".join(m.beast() for m in with_signal)
    sbs = subprocess.run([exe, "--ifile", str(path), "--recover", "--sbs"], capture_output=True, text=True, check=True)
    tr = api.Tracker()
    lines = []
    for m in msgs:
        u = tr.update(m, api.STREAM_EPOCH_MS + m.sample_pos // 2000)
        if u:
            lines.append(u[1])
    assert sbs.stdout == "".join(lines)
    st = subprocess.run([exe, "--ifile", str(path), "--recover", "--stats"], capture_output=True, text=True, check=True)
    plain = subprocess.run([exe, "--ifile", str(path), "--stats"], capture_output=True, text=True, check=True)
    assert st.stdout == plain.stdout
    rs = gpu_decoder_factory(recover=True)
    rs.decode(data)
    want = rs.recovery_stats()
    assert st.stderr.strip() == ("recovery: {considered} considered, {found} found, {ambiguous} ambiguous, "
                                 "{unknown_address} unknown address, {dropped} dropped, {delivered} delivered").format(**want)
