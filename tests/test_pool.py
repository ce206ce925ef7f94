"""Many receivers on one GPU (modes_pool_*, SURVEY.md 8(f) item 4): every receiver's messages, fields,
stream positions and statistics must equal a decode of that receiver's stream alone.

The CPU test drives the host half (modes_pool_resolve) with candidate records that the oracle's scan
produces over the batch exactly as the pool lays it out (pad, data, pad, data, ...): it checks the
layout argument — a data buffer's candidates depend on nothing but that buffer and the 238 carried
samples — and the per-receiver re-basing / address caches.  The GPU test runs modes_pool_ingest."""
import numpy as np
import pytest

import checker as C
import streams as S
from dump1090_b200 import api, synth

BUF = api.BUFFER_BYTES


def _streams(n_rx, n_buf):
    """n_rx different streams of n_buf whole buffers: dense traffic, frames straddling buffer seams."""
    out = []
    for r in range(n_rx):
        s = synth.random_traffic(n_buf * 131072, 120 * n_buf + 37 * r, seed=100 + r)
        assert s.size == n_buf * BUF
        out.append(s)
    return out


def _chain_streams(n_rx, n_buf):
    """n_rx streams of n_buf whole buffers, each a chain through the address cache
    (streams.address_chain) of its own kind, length and phase: receiver r is silent for r % 3
    buffers, then runs a chain of the remaining buffers.  A cache shared or lost between batches
    breaks the chain."""
    out = []
    for r in range(n_rx):
        phase = r % 3
        kind = S.CHAIN_KINDS[r % len(S.CHAIN_KINDS)]
        quiet = synth.synth_stream(phase * 131072, [], sigma=1.0, seed=50 + r)
        s = np.concatenate([quiet, S.address_chain(n_buf - phase, kind, seed=r + 1)])
        assert s.size == n_buf * BUF
        out.append(s)
    return out


def _schedule(n_rx, n_buf, seed):
    """Which receivers deliver a buffer in which call: every receiver n_buf times, not in lock step."""
    rng = np.random.default_rng(seed)
    left = [n_buf] * n_rx
    calls = []
    while any(left):
        ids = [r for r in range(n_rx) if left[r] and rng.random() < 0.7]
        rng.shuffle(ids)
        if not ids:
            continue
        for r in ids:
            left[r] -= 1
        calls.append(ids)
    return calls


def _expect(stream, kw):
    # a live receiver has no end of file: without the all-padding buffer the reference processes after the last read (dump1090.c:497 vs :2989)
    msgs, stats = C.oracle_decode(stream, drop_eof=1, **kw)
    return [m.hexline() for m in msgs], [C.msg_fields(m, with_pos=True) for m in msgs], stats


def _check(pool, streams, kw):
    for r, s in enumerate(streams):
        got = pool.take(r)
        lines, fields, stats = _expect(s, kw)
        assert [m.raw_line() for m in got] == lines, f"receiver {r}"
        assert [C.msg_fields(m, with_pos=True) for m in got] == fields, f"receiver {r}"
        assert list(pool.stats(r).values()) == stats, f"receiver {r}"


def _pool_cases():
    """(flags, stream mix), named by the flags for ordinary traffic and flags-chains for chains."""
    for mix in ("traffic", "chains"):
        for kw in (dict(), dict(aggressive=1), dict(fix=0), dict(check_crc=0)):
            kid = "-".join(f"{a}{b}" for a, b in kw.items()) or "default"
            yield pytest.param(kw, mix, id=kid if mix == "traffic" else f"{kid}-{mix}")


@pytest.mark.parametrize("kw,mix", list(_pool_cases()))
def test_pool_resolve_matches_single_stream_decodes(kw, mix, checker_libs):
    n_rx, n_buf = (5, 3) if mix == "traffic" else (5, 8)
    streams = _streams(n_rx, n_buf) if mix == "traffic" else _chain_streams(n_rx, n_buf)
    cfg = dict(fix_errors=kw.get("fix", 1), aggressive=kw.get("aggressive", 0), check_crc=kw.get("check_crc", 1))
    nxt = [0] * n_rx
    with api.ReceiverPool(n_rx, **cfg) as pool:
        for ids in _schedule(n_rx, n_buf, seed=3):
            batch = np.full(2 * len(ids) * BUF, 127, dtype=np.uint8)
            for i, r in enumerate(ids):
                k = nxt[r]
                if k:                                                   # the pad buffer's tail = this receiver's carry
                    batch[(2 * i + 1) * BUF - api.CARRY_BYTES: (2 * i + 1) * BUF] = streams[r][k * BUF - api.CARRY_BYTES: k * BUF]
                batch[(2 * i + 1) * BUF: (2 * i + 2) * BUF] = streams[r][k * BUF: (k + 1) * BUF]
                nxt[r] += 1
            recs = C.oracle_scan_candidates(batch, fix=cfg["fix_errors"], aggressive=cfg["aggressive"], cap=400000)
            cands = np.frombuffer(b"".join(bytes(c) for c in recs), dtype=api.CANDIDATE_DTYPE) if recs else np.zeros(0, api.CANDIDATE_DTYPE)
            g = (cands["t"] + 2) // api.TILE_SAMPLES
            n_tiles = api.tiles_for(2 * len(ids))
            cnt = np.bincount(g, minlength=n_tiles).astype(np.uint32)
            tiles = np.zeros(n_tiles, dtype=api.TILE_DTYPE)
            tiles["count"] = cnt
            tiles["offset"] = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.uint32)
            pool.resolve(ids, cands, tiles)
        assert [pool.buffers(r) for r in range(n_rx)] == [n_buf] * n_rx
        _check(pool, streams, kw)


def test_pool_output_array(checker_libs):
    """modes_pool_set_output: the same messages in one caller-owned array with the receiver of each."""
    n_rx, n_buf = 3, 2
    streams = _streams(n_rx, n_buf)
    with api.ReceiverPool(n_rx) as pool:
        out, out_rx = pool.set_output_array(20000)
        per_rx = [[] for _ in range(n_rx)]
        for k in range(n_buf):
            batch = np.full(2 * n_rx * BUF, 127, dtype=np.uint8)
            for i in range(n_rx):
                if k:
                    batch[(2 * i + 1) * BUF - api.CARRY_BYTES: (2 * i + 1) * BUF] = streams[i][k * BUF - api.CARRY_BYTES: k * BUF]
                batch[(2 * i + 1) * BUF: (2 * i + 2) * BUF] = streams[i][k * BUF: (k + 1) * BUF]
            recs = C.oracle_scan_candidates(batch, fix=1, aggressive=0, cap=400000)
            cands = np.frombuffer(b"".join(bytes(c) for c in recs), dtype=api.CANDIDATE_DTYPE)
            g = (cands["t"] + 2) // api.TILE_SAMPLES
            cnt = np.bincount(g, minlength=api.tiles_for(2 * n_rx)).astype(np.uint32)
            tiles = np.zeros(cnt.size, dtype=api.TILE_DTYPE)
            tiles["count"] = cnt
            tiles["offset"] = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.uint32)
            pool.rearm_output()
            pool.resolve(list(range(n_rx)), cands, tiles)
            n = pool.output_count()
            assert 0 < n <= len(out) and list(out_rx[:n]) == sorted(out_rx[:n])       # receiver by receiver, as listed
            for j in range(n):
                per_rx[out_rx[j]].append(out[j].raw_line())
        for r in range(n_rx):
            assert per_rx[r] == _expect(streams[r], {})[0]
            assert per_rx[r] == [m.raw_line() for m in pool.take(r)]                   # the sink saw the same


def test_pool_rejects_bad_calls(checker_libs):
    with api.ReceiverPool(3, max_batch=2) as pool:
        empty = np.zeros(0, api.CANDIDATE_DTYPE)
        with pytest.raises(RuntimeError, match="listed twice"):
            pool.resolve([1, 1], empty, np.zeros(api.tiles_for(4), api.TILE_DTYPE))
        with pytest.raises(RuntimeError, match="out of range"):
            pool.resolve([3], empty, np.zeros(api.tiles_for(2), api.TILE_DTYPE))
        with pytest.raises(RuntimeError, match="created for 2"):
            pool.resolve([0, 1, 2], empty, np.zeros(api.tiles_for(6), api.TILE_DTYPE))


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(), dict(aggressive=1), dict(fix=0), dict(check_crc=0)],
                         ids=lambda k: "-".join(f"{a}{b}" for a, b in k.items()) or "default")
def test_pool_ingest_matches_single_stream_decodes(kw, checker_libs):
    n_rx, n_buf = 7, 3
    streams = _streams(n_rx, n_buf)
    streams[-1] = _chain_streams(1, n_buf)[0]                           # a receiver whose cache carries a chain
    cfg = dict(fix_errors=kw.get("fix", 1), aggressive=kw.get("aggressive", 0), check_crc=kw.get("check_crc", 1))
    nxt = [0] * n_rx
    with api.ReceiverPool(n_rx, max_batch=5, **cfg) as pool:
        for ids in _schedule(n_rx, n_buf, seed=4):
            for lo in range(0, len(ids), 5):                            # at most max_batch receivers per call
                part = ids[lo: lo + 5]
                pool.ingest(part, [streams[r][nxt[r] * BUF: (nxt[r] + 1) * BUF] for r in part])
                for r in part:
                    nxt[r] += 1
        _check(pool, streams, kw)
        # two batches in flight, a receiver in both of them
        for r in range(n_rx):
            pool.reset(r)
        k = 0
        pool.submit([0, 1, 2], [streams[r][0:BUF] for r in (0, 1, 2)])
        for k in range(1, n_buf):
            pool.submit([2, 0, 1], [streams[r][k * BUF: (k + 1) * BUF] for r in (2, 0, 1)])
            pool.collect()
        pool.collect()
        with pytest.raises(RuntimeError, match="no batch in flight"):
            pool.collect()
        for r in (0, 1, 2):
            assert [m.raw_line() for m in pool.take(r)] == _expect(streams[r], kw)[0]
            assert list(pool.stats(r).values()) == _expect(streams[r], kw)[2]
        # all buffers of a call in one host block (constant distance): the strided upload
        for r in range(n_rx):
            pool.reset(r)
        for k in range(n_buf):
            block = np.stack([streams[r][k * BUF: (k + 1) * BUF] for r in range(5)])
            pool.ingest(list(range(5)), [block[r] for r in range(5)])
        for r in range(5):
            assert [m.raw_line() for m in pool.take(r)] == _expect(streams[r], kw)[0]
        # a receiver that starts a new stream
        pool.reset(2)
        for k in range(n_buf):
            pool.ingest([2], [streams[4][k * BUF: (k + 1) * BUF]])
        got = pool.take(2)
        assert [m.raw_line() for m in got] == _expect(streams[4], kw)[0]
