"""CPU (-m "not gpu"): the product's host-side code and the C-ABI surface (no device compute)."""
import ctypes
import hashlib
import re
from pathlib import Path

import numpy as np
import pytest

import checker as C
import golden_util as G
import streams as S
from dump1090_b200 import api, synth

ROOT = Path(__file__).resolve().parent.parent


def test_library_exports_every_declared_symbol():
    header = (ROOT / "include" / "modes_b200.h").read_text()
    declared = set(re.findall(r"\b(modes_[a-z_0-9]+)\s*\(", header)) - {"modes_sink_fn"}
    assert declared == set(api.EXPORTS)
    L = ctypes.CDLL(str(api.LIB_PATH))
    for name in sorted(declared):
        assert hasattr(L, name), name
    assert L.modes_abi_version() == 3


def test_struct_layouts():
    assert ctypes.sizeof(api.Message) == ctypes.sizeof(C.Msg) == 200
    assert ctypes.sizeof(api.FrameEval) == ctypes.sizeof(C.Pass) == 24
    assert ctypes.sizeof(api.Candidate) == ctypes.sizeof(C.Cand) == 56
    assert api.CANDIDATE_DTYPE.itemsize == 56 and api.TILE_DTYPE.itemsize == 8
    cfg = api.make_config()
    assert (cfg.fix_errors, cfg.aggressive, cfg.check_crc, cfg.drop_eof_buffer) == (1, 0, 1, 0)   # dump1090.c:305-315


def test_create_fails_loudly_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises(RuntimeError, match="no CPU path"):
        api.Decoder()


def _resolve_with_product(data, kw):
    cands = C.oracle_scan_candidates(data, fix=kw.get("fix", 1), aggressive=kw.get("aggressive", 0),
                                     drop_eof=kw.get("drop_eof", 0))
    arr = np.frombuffer(b"".join(bytes(c) for c in cands), dtype=api.CANDIDATE_DTYPE) if cands \
        else np.zeros(0, dtype=api.CANDIDATE_DTYPE)
    # split the candidate list into a few "tiles" to exercise the tile walk
    cuts = sorted({0, len(cands) // 3, len(cands) // 2, len(cands)})
    tiles = np.array([(a, b - a) for a, b in zip(cuts, cuts[1:])] or [(0, 0)], dtype=api.TILE_DTYPE)
    r = api.Resolver(fix_errors=kw.get("fix", 1), aggressive=kw.get("aggressive", 0), check_crc=kw.get("check_crc", 1))
    r.run(arr, tiles)
    return r.take_messages(), list(r.stats().values())


@pytest.mark.parametrize("name,cid", G.CASES)
def test_resolver_reproduces_golden(name, cid, checker_libs):
    """Product resolve + field decode (modes_resolve.cpp), fed with the oracle's candidate records,
    must reproduce the reference's messages, fields and statistics."""
    doc = G.load(name)
    case = doc["cases"][cid]
    msgs, st = _resolve_with_product(G.make_input(doc), case["flags"])
    assert [C.msg_fields(m) for m in msgs] == case["messages"]
    assert st == case["stats"]


def test_resolver_sample_positions(checker_libs):
    data = synth.random_traffic(300000, 300, 21)
    msgs, _ = _resolve_with_product(data, {})
    exp, _ = C.oracle_decode(data)
    assert [m.sample_pos for m in msgs] == [m.sample_pos for m in exp]


def test_resolver_shard_boundaries_are_invisible(checker_libs):
    """Feeding the resolver buffer by buffer (as shards arrive from different GPUs) changes nothing."""
    data = synth.random_traffic(600000, 700, 22)
    cands = C.oracle_scan_candidates(data)
    arr = np.frombuffer(b"".join(bytes(c) for c in cands), dtype=api.CANDIDATE_DTYPE)
    whole = api.Resolver()
    whole.run(arr, np.array([(0, arr.size)], dtype=api.TILE_DTYPE))
    ref = [m.raw_line() for m in whole.take_messages()]
    parts = api.Resolver()
    for k in range(int(arr["t"].max() >> 17) + 1):
        sel = arr[(arr["t"] >> 17) == k].copy()
        sel["t"] -= k << 17                       # shard-local positions + buffer_base
        parts.run(sel, np.array([(0, sel.size)], dtype=api.TILE_DTYPE), buffer_base=k)
    assert [m.raw_line() for m in parts.take_messages()] == ref
    assert parts.stats() == whole.stats()


def test_synth_is_deterministic():
    s = synth.random_traffic(50000, 60, 3)
    assert hashlib.sha256(s.tobytes()).hexdigest() == hashlib.sha256(synth.random_traffic(50000, 60, 3).tobytes()).hexdigest()
    assert s.dtype == np.uint8 and s.size == 100000
    t = synth.tile_to(s, 250001)
    assert t.size == 250001 and np.array_equal(t[:100000], s) and np.array_equal(t[100000:200000], s)


def test_synth_parity_against_known_frames():
    for hx in ("8D451E8B99019699C00B0A81F36E", "8D4B969699155600E87406F5B69F"):
        b = bytes.fromhex(hx)
        assert synth.make_frame(17, b[0] & 7, b[1:11]) == b


@pytest.mark.parametrize("nshards,name", [pytest.param(n, "traffic", id=str(n)) for n in (2, 3, 8)]
                         + [pytest.param(n, name, id=f"{n}-{name}") for name in S.CHAINS for n in (2, 3, 8)])
def test_parallel_shard_resolve_is_exact(nshards, name, checker_libs):
    """modes_resolver_run_shards (speculative ICAO cache at shard boundaries, verified) == sequential,
    also on chains through the address cache where every shard's guess depends on the previous one."""
    data = synth.random_traffic(131072 * 9 + 4000, 1400, 23, n_aircraft=40) if name == "traffic" else S.chain(name)
    cands = C.oracle_scan_candidates(data, aggressive=1)
    arr = np.frombuffer(b"".join(bytes(c) for c in cands), dtype=api.CANDIDATE_DTYPE)
    seq = api.Resolver(aggressive=1)
    seq.run(arr, np.array([(0, arr.size)], dtype=api.TILE_DTYPE))
    want = [C.msg_fields(m, with_pos=True) for m in seq.take_messages()]
    nbuf = int(arr["t"].max() >> 17) + 1
    from dump1090_b200 import sharded
    shards = []
    for first, count in sharded.shard_plan(nbuf, nshards):
        sel = arr[((arr["t"] >> 17) >= first) & ((arr["t"] >> 17) < first + count)].copy()
        sel["t"] -= first << 17
        shards.append((sel, np.array([(0, sel.size)], dtype=api.TILE_DTYPE), first))
    par = api.Resolver(aggressive=1)
    par.run_shards(shards)
    got = [C.msg_fields(m, with_pos=True) for m in par.take_messages()]
    assert got == want
    assert par.stats() == seq.stats()
    # state carries over to a following call exactly as in the sequential resolver
    more = synth.random_traffic(300000, 300, 24, n_aircraft=40)
    c2 = C.oracle_scan_candidates(more, aggressive=1)
    a2 = np.frombuffer(b"".join(bytes(c) for c in c2), dtype=api.CANDIDATE_DTYPE)
    t2 = np.array([(0, a2.size)], dtype=api.TILE_DTYPE)
    seq.run(a2, t2, buffer_base=nbuf); par.run(a2, t2, buffer_base=nbuf)
    assert [m.raw_line() for m in par.take_messages()] == [m.raw_line() for m in seq.take_messages()]


def test_parallel_shard_resolve_recovers_from_a_wrong_guess(checker_libs, capfd, monkeypatch):
    """The first guess of a shard's starting ICAO cache comes from the tail of the previous shard.
    An address announced only early in shard 0 is missing from that guess; a DF4 reply from it in
    shard 1 is then judged wrongly, the verification catches it, and the shard is resolved again."""
    from dump1090_b200 import sharded
    nbuf = 24
    n = 131072 * nbuf
    me = bytes([0x58, 0xC3, 0x82, 0xD6, 0x90, 0xC8, 0xAC])               # an airborne-position ME field
    a, b = 0x4840D6, 0x3C6444
    frames = [(131072 + 5000, synth.make_frame(17, 5, a.to_bytes(3, "big") + me), 80.0, 0.3, 0.0)]   # A: once, early
    for k in range(nbuf):                                                 # B: all along
        frames.append((131072 * k + 40000, synth.make_frame(17, 5, b.to_bytes(3, "big") + me), 70.0, 1.1, 0.0))
    frames.append((131072 * 14 + 9000, synth.make_frame(4, 0, bytes([0x01, 0x85, 0x10]), icao_for_ap=a), 75.0, 0.7, 0.0))
    frames.append((131072 * 20 + 9000, synth.make_frame(5, 0, bytes([0x02, 0x20, 0x31]), icao_for_ap=b), 75.0, 0.2, 0.0))
    data = synth.synth_stream(n, frames, seed=9)
    cands = C.oracle_scan_candidates(data)
    arr = np.frombuffer(b"".join(bytes(c) for c in cands), dtype=api.CANDIDATE_DTYPE)

    def tiled(sel, n_buffers):                                            # one tile per TILE_SAMPLES positions, like the scan kernel
        g = (sel["t"] + 2) // api.TILE_SAMPLES
        nt = api.tiles_for(n_buffers)
        cnt = np.bincount(g, minlength=nt).astype(np.uint32)
        t = np.zeros(nt, dtype=api.TILE_DTYPE)
        t["count"] = cnt
        t["offset"] = np.concatenate([[0], np.cumsum(cnt)[:-1]])
        return t

    seq = api.Resolver()
    seq.run(arr, tiled(arr, nbuf + 1))
    want = [C.msg_fields(m, with_pos=True) for m in seq.take_messages()]
    assert any(m["msgtype"] == 4 for m in want) and any(m["msgtype"] == 5 for m in want)
    shards = []
    for first, count in sharded.shard_plan(nbuf, 2):
        sel = arr[((arr["t"] >> 17) >= first) & ((arr["t"] >> 17) < first + count)].copy()
        sel["t"] -= first << 17
        shards.append((sel, tiled(sel, count), first))
    monkeypatch.setenv("MODES_RESOLVE_TIMING", "1")
    par = api.Resolver()
    capfd.readouterr()
    par.run_shards(shards)
    assert "2 rounds" in capfd.readouterr().err                           # the guess was wrong, and noticed
    assert [C.msg_fields(m, with_pos=True) for m in par.take_messages()] == want
    assert par.stats() == seq.stats()


@pytest.mark.timeout(180)
def test_two_resolvers_on_two_threads(checker_libs):
    """Distinct contexts are independent (include/modes_b200.h): two resolvers delivering >= 2048
    messages each into arrays from two threads at once (the struct-building pool is shared by the
    process) produce exactly what they produce alone.  (With the pool's job state unprotected this
    test hangs or delivers unbuilt structs.)"""
    import threading
    data = synth.random_traffic(131072 * 40, 9000, 77, n_aircraft=30)
    cands = C.oracle_scan_candidates(data, cap=400000)
    one = np.frombuffer(b"".join(bytes(c) for c in cands), dtype=api.CANDIDATE_DTYPE)
    reps = 24                                            # the same 40 buffers again and again: ~250 000 messages per call
    arr = np.tile(one, reps)
    arr["t"] += np.repeat(np.arange(reps, dtype=np.int64) * 40 * api.BUFFER_SAMPLES, one.size)
    tiles = np.array([(0, arr.size)], dtype=api.TILE_DTYPE)

    def run_once(r):
        ctypes.memset(r._out, 0xEE, ctypes.sizeof(r._out))   # a struct that is never built must show
        r.reset_state(); r.rearm_output(); r.run(arr, tiles)
        n = r.output_count()
        return n, hashlib.sha256(bytes(memoryview(r._out)[:n])).hexdigest()

    solo = api.Resolver(check_crc=0)
    solo.set_output_array(arr.size * 2)
    want = run_once(solo)
    assert want[0] >= 2048
    rs = [api.Resolver(check_crc=0) for _ in range(2)]
    for r in rs:
        r.set_output_array(arr.size * 2)
    results, errors = [[], []], []

    gate = threading.Barrier(2)

    def worker(k):
        try:
            for _ in range(12):
                gate.wait()                              # both calls start together
                results[k].append(run_once(rs[k]))
        except BaseException as e:                       # noqa: BLE001
            errors.append(e)

    th = [threading.Thread(target=worker, args=(k,)) for k in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errors
    assert all(x == want for k in range(2) for x in results[k])


def test_host_wait_mode_is_validated():
    L = api.lib()
    assert L.modes_set_host_wait(2) == -1 and L.modes_set_host_wait(-1) == -1
    assert L.modes_set_host_wait(1) == 0 and L.modes_set_host_wait(0) == 0
