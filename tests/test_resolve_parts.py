"""The verdict pass cut into parts for the host's threads (modes_resolve.cpp: cut_parts / judge_parts).

A long record array is judged in a few parts of whole buffers at once, each from a guessed address
cache that is verified afterwards; the result must be exactly the sequential pass's — messages,
fields, stream positions, statistics, and the state a following call starts from.  Records come
from the oracle's candidate scan (no GPU needed); MODES_RESOLVE_PARTS / MODES_RESOLVE_PART_TILES
force the cut on streams of a few buffers (the defaults cut only arrays of >= 8192 tiles)."""
import numpy as np
import pytest

import checker as C
import streams as S
from dump1090_b200 import api, synth


def records_of(data, **kw):
    cands = C.oracle_scan_candidates(data, **kw)
    return np.frombuffer(b"".join(bytes(c) for c in cands), dtype=api.CANDIDATE_DTYPE) if cands \
        else np.zeros(0, dtype=api.CANDIDATE_DTYPE)


def tiled(sel, n_buffers, scatter_seed=None):
    """The scan kernel's tile table for a record array: one tile per TILE_SAMPLES positions; with a
    seed the tiles' runs lie scattered through the array (tiles are appended as they finish)."""
    g = (sel["t"] + 2) // api.TILE_SAMPLES
    nt = api.tiles_for(n_buffers)
    cnt = np.bincount(g, minlength=nt).astype(np.uint32)
    off = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.uint32)
    t = np.zeros(nt, dtype=api.TILE_DTYPE)
    t["count"] = cnt
    t["offset"] = off
    if scatter_seed is None:
        return sel, t
    rng = np.random.default_rng(scatter_seed)
    order = np.argsort(np.arange(nt) + rng.integers(0, 40, nt), kind="stable")
    new_off = np.zeros(nt, dtype=np.uint32)
    new_off[order] = np.concatenate([[0], np.cumsum(cnt[order])[:-1]])
    out = np.zeros_like(sel)
    within = np.arange(sel.size) - np.repeat(off, cnt)
    out[np.repeat(new_off, cnt) + within] = sel
    t["offset"] = new_off
    return out, t


def decode(resolver):
    return [C.msg_fields(m, with_pos=True) for m in resolver.take_messages()]


@pytest.fixture
def sequential(monkeypatch):
    def run(fn):
        monkeypatch.setenv("MODES_RESOLVE_PARTS", "1")
        try:
            return fn()
        finally:
            monkeypatch.delenv("MODES_RESOLVE_PARTS")
    return run


@pytest.mark.parametrize("name,parts,part_tiles",
                         [pytest.param("traffic", p, t, id=f"{p}-{t}") for p, t in [(2, 1), (3, 7), (5, 1), (16, 1), (64, 1)]]
                         + [pytest.param(name, p, 1, id=f"{name}-{p}-1") for name in S.CHAINS for p in (2, 3, 16)])
@pytest.mark.parametrize("flags", [dict(), dict(aggressive=1), dict(fix_errors=0), dict(check_crc=0)])
def test_parts_equal_the_sequential_pass(name, parts, part_tiles, flags, checker_libs, monkeypatch, sequential):
    """Random traffic, and chains through the address cache (tests/streams.address_chain) whose
    every buffer decides what the next one reads: a guess is wrong part after part."""
    if name == "traffic":
        nbuf = 9
        data = synth.random_traffic(131072 * nbuf + 4000, 1500, 31, n_aircraft=40)
    else:
        nbuf = S.CHAINS[name][1]
        data = S.chain(name)
    arr = records_of(data, fix=flags.get("fix_errors", 1), aggressive=flags.get("aggressive", 0))
    arr, tiles = tiled(arr, nbuf + 1, scatter_seed=parts)
    more = records_of(synth.random_traffic(300000, 300, 32, n_aircraft=40), fix=flags.get("fix_errors", 1),
                      aggressive=flags.get("aggressive", 0))
    more_tiles = np.array([(0, more.size)], dtype=api.TILE_DTYPE)

    def both_calls():
        r = api.Resolver(**flags)
        r.run(arr, tiles)
        first = decode(r)
        st = dict(r.stats())
        cache = r.get_cache().copy()
        r.run(more, more_tiles, buffer_base=nbuf + 1)                     # the state carries over
        return first, st, cache, decode(r), dict(r.stats())

    want = sequential(both_calls)
    monkeypatch.setenv("MODES_RESOLVE_PARTS", str(parts))
    monkeypatch.setenv("MODES_RESOLVE_PART_TILES", str(part_tiles))
    got = both_calls()
    assert got[0] == want[0] and len(got[0]) >= (500 if name == "traffic" else nbuf)
    assert got[1] == want[1]
    assert np.array_equal(got[2], want[2])
    assert got[3] == want[3] and got[4] == want[4]


def test_parts_in_the_tentative_and_shard_calls(checker_libs, monkeypatch, sequential):
    """run_tentative + commit (one rank of a sharded decode) and run_shards cut their arrays too."""
    nbuf = 12
    data = synth.random_traffic(131072 * nbuf, 1800, 33, n_aircraft=60)
    arr = records_of(data, aggressive=1)
    arr, tiles = tiled(arr, nbuf, scatter_seed=3)

    def whole():
        r = api.Resolver(aggressive=1)
        r.run(arr, tiles)
        return decode(r), dict(r.stats()), r.get_cache().copy()

    want = sequential(whole)
    monkeypatch.setenv("MODES_RESOLVE_PARTS", "4")
    monkeypatch.setenv("MODES_RESOLVE_PART_TILES", "2")
    r = api.Resolver(aggressive=1)
    r.set_cache(None)
    r.run_tentative(arr, tiles)
    assert np.array_equal(r.get_cache(), want[2])                         # the end cache is known before the commit
    r.commit()
    assert decode(r) == want[0] and dict(r.stats()) == want[1]
    # two shards of six buffers, each cut again
    from dump1090_b200 import sharded
    shards = []
    for first, count in sharded.shard_plan(nbuf, 2):
        sel = arr[((arr["t"] >> 17) >= first) & ((arr["t"] >> 17) < first + count)].copy()
        sel["t"] -= first << 17
        sel.sort(order="t")
        s, t = tiled(sel, count, scatter_seed=first + 1)
        shards.append((s, t, first))
    monkeypatch.setenv("MODES_RESOLVE_PARTS", "6")
    monkeypatch.setenv("MODES_RESOLVE_TIMING", "1")
    p = api.Resolver(aggressive=1)
    p.run_shards(shards)
    assert decode(p) == want[0] and dict(p.stats()) == want[1]
    assert np.array_equal(p.get_cache(), want[2])


def test_a_wrong_guess_inside_one_array_is_noticed(checker_libs, capfd, monkeypatch, sequential):
    """An address announced once, early in the first part, is missing from the guess the second part
    starts from (the guess is what the tail of the first part writes); its DF4 reply in the second
    part is then judged wrongly, the verification notices, and the part is judged again."""
    nbuf = 24
    me = bytes([0x58, 0xC3, 0x82, 0xD6, 0x90, 0xC8, 0xAC])
    a, b = 0x4840D6, 0x3C6444
    frames = [(131072 + 5000, synth.make_frame(17, 5, a.to_bytes(3, "big") + me), 80.0, 0.3, 0.0)]
    for k in range(nbuf):
        frames.append((131072 * k + 40000, synth.make_frame(17, 5, b.to_bytes(3, "big") + me), 70.0, 1.1, 0.0))
    frames.append((131072 * 14 + 9000, synth.make_frame(4, 0, bytes([0x01, 0x85, 0x10]), icao_for_ap=a), 75.0, 0.7, 0.0))
    frames.append((131072 * 20 + 9000, synth.make_frame(5, 0, bytes([0x02, 0x20, 0x31]), icao_for_ap=b), 75.0, 0.2, 0.0))
    arr = records_of(synth.synth_stream(131072 * nbuf, frames, seed=9))
    arr, tiles = tiled(arr, nbuf + 1)

    def whole():
        r = api.Resolver()
        r.run(arr, tiles)
        return decode(r), dict(r.stats())

    want = sequential(whole)
    assert any(m["msgtype"] == 4 for m in want[0]) and any(m["msgtype"] == 5 for m in want[0])
    monkeypatch.setenv("MODES_RESOLVE_PARTS", "2")
    monkeypatch.setenv("MODES_RESOLVE_PART_TILES", "1")
    monkeypatch.setenv("MODES_RESOLVE_TIMING", "1")
    capfd.readouterr()
    got = whole()
    err = capfd.readouterr().err
    assert "in 2 parts, 2 rounds" in err
    assert got == want


def test_parts_with_silence_and_few_records(checker_libs, monkeypatch, sequential):
    """Long stretches without a candidate (parts that come out empty or merge), a single record, none."""
    nbuf = 20
    frames = []
    for k in (0, 1, 17, 18, 19):                                          # traffic only at both ends
        for i in range(30):
            icao = 0x400000 + 7 * i
            frames.append((131072 * k + 2000 + 4000 * i, synth.make_frame(17, 5, icao.to_bytes(3, "big") + bytes(7)), 70.0, 0.5, 0.0))
    arr = records_of(synth.synth_stream(131072 * nbuf, frames, seed=4))
    # keep only the records near the injected frames: the rest of the stream is "silent"
    keep = np.isin(arr["t"] >> 17, [0, 1, 17, 18, 19])
    arr = arr[keep].copy()
    assert arr.size > 100
    for sel in (arr, arr[:1].copy(), arr[:0].copy()):
        s, tiles = tiled(sel, nbuf + 1)

        def whole():
            r = api.Resolver()
            r.run(s, tiles)
            return decode(r), dict(r.stats()), r.get_cache().copy()

        want = sequential(whole)
        for parts in (2, 7, 40):
            monkeypatch.setenv("MODES_RESOLVE_PARTS", str(parts))
            monkeypatch.setenv("MODES_RESOLVE_PART_TILES", "1")
            got = whole()
            assert got[0] == want[0] and got[1] == want[1] and np.array_equal(got[2], want[2])
