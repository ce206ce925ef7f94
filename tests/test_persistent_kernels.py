"""The persistent scan (K1, modes_scan2.cu), frame-evaluation (K2, modes_eval_fused.cu and
modes_kernels.cu) and weak-preamble (modes_weak.cu) kernels past each warp's first tile and chunk,
and on windows that start in the carry block.

Both K1 and K2 hand work out from a global counter and prepare the next item while they finish the
current one, so part of their code only runs from a warp's second tile or chunk on: K1's tile
hand-out, the copy-out of the previous tile's list and the loads of the next tile's first rows; K2's
staging of the next chunk behind the current chunk's verdicts and its three-deep hand-out.  Streams
under a megabyte on a full H100 grid give every warp one tile and at most one chunk.  The device
harness tests/device_shim/scan_eval_device.cu (linked against the product's own objects) launches the
kernels with a chosen SM count; the launchers size their grids from it, so with one to three SMs a few
buffers put every warp through many tiles and chunks.  Windows that start in the carry block
(v <= 240) take the kernels' slow staging paths, which only the first 240 positions of a batch reach.

The model throughout is the oracle's candidate records, byte for byte: a batch with a carry is modelled
as a pad buffer whose last 476 bytes are the carry, followed by the body (oracle_model)."""
import ctypes
import subprocess

import numpy as np
import pytest

import checker as C
import recover_model as R
import streams as S
import test_gpu_edges as GE
import weak_model as W
from dump1090_b200 import api, synth

pytestmark = pytest.mark.gpu

ROOT = C.ROOT
DSHIM = ROOT / "tests" / "_build" / "libscan_eval_device.so"
BUF = api.BUFFER_BYTES
NS = api.BUFFER_SAMPLES
CARRY = api.CARRY_BYTES
HALO = 240                                # virtual samples before the body: 2 unused + 238 carried
TILE = api.TILE_SAMPLES
LAST_J = 131069                           # the last position the scan visits in a buffer
REC = 56                                  # bytes of a candidate record
SENTINEL = 0x5A                           # dev_eval fills its records with it before the launch
VARIANTS = ["fused", "fused2", "lean", "serial", "warp"]
FLAGS = [(1, 0), (1, 1), (0, 0)]          # (fix_errors, aggressive)
# K2's persistent grid per SM (modes_eval_fused.cu, modes_kernels.cu: one CTA of 12 or 16 warps per SM;
# the warp-per-candidate kernel four CTAs of 8 warps) and the candidates a warp takes at a time
K2_WARPS_PER_SM = {"fused": 12, "fused2": 16, "lean": 12, "serial": 12, "warp": 32}
K2_CHUNK = {"fused": 32, "fused2": 32, "lean": 32, "serial": 32, "warp": 8}
MIN_ITERATIONS = 4                        # tiles and chunks every warp must reach
SM_COUNTS = [1, 2, 3]


@pytest.fixture(scope="module")
def shim():
    subprocess.run(["make", "-s", "dshim"], cwd=ROOT, check=True)
    lib = ctypes.CDLL(str(DSHIM))
    u32, i32, p = ctypes.c_uint32, ctypes.c_int, ctypes.c_void_p
    lib.dev_error.restype = ctypes.c_char_p
    lib.dev_limits.argtypes = [p]
    lib.dev_scan.argtypes = [p, u32, p, i32, u32, p, p, p]
    lib.dev_eval.argtypes = [p, u32, p, p, u32, u32, u32, i32, i32, i32, p]
    lib.dev_weak.argtypes = [p, u32, p, u32, u32, i32, u32, u32, p, p]
    lim = np.zeros(2, np.int32)
    assert lib.dev_limits(lim.ctypes.data) == 0, lib.dev_error()
    lib.sm_count, lib.max_ctas_per_sm = int(lim[0]), int(lim[1])
    assert lib.sm_count >= max(SM_COUNTS) and lib.max_ctas_per_sm > 0
    return lib


# ---------------------------------------------------------------- batches and the model


def whole_buffers(data):
    """data padded with no-signal samples to whole buffers plus the EOF buffer, as the streaming decode
    submits it (test_gpu_parity._check_candidates)."""
    nbuf = data.size // BUF + 1
    body = np.full(nbuf * BUF, 127, dtype=np.uint8)
    body[: data.size] = data
    return body, nbuf


def oracle_records(data, fix=1, aggressive=0, drop_eof=1, cap=None):
    """The oracle's candidate records of a stream as an (n, 56) byte array."""
    a = np.ascontiguousarray(data, dtype=np.uint8)
    lib = C.oracle_lib()
    lib.oracle_scan_candidates.restype = ctypes.c_long
    cap = cap or max(4096, a.size // 16)
    out = (C.Cand * cap)()
    n = lib.oracle_scan_candidates(a.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(a.size), int(fix), int(aggressive),
                                   int(drop_eof), out, ctypes.c_size_t(cap))
    assert 0 <= n <= cap
    return np.frombuffer(out, dtype=np.uint8, count=n * REC).reshape(n, REC).copy()


def rec_t(recs):
    return recs[:, :8].copy().view("<i8").ravel()


def oracle_model(body, carry, fix=1, aggressive=0, cap=None):
    """The records of a batch of whole buffers `body` with carry block `carry` (None: no signal): the
    oracle over a pad buffer whose last 476 bytes are the carry, then the body; the pad buffer's own
    candidates dropped and t made batch-relative."""
    pad = np.full(BUF, 127, dtype=np.uint8)
    if carry is not None:
        pad[-CARRY:] = np.frombuffer(bytes(carry), dtype=np.uint8)
    recs = oracle_records(np.concatenate([pad, body]), fix, aggressive, drop_eof=1, cap=cap)
    t = rec_t(recs)
    keep = t >= NS
    recs = recs[keep]
    recs[:, :8] = (t[keep] - NS).astype("<i8").view(np.uint8).reshape(-1, 8)
    return recs


def carry_arg(carry):
    return None if carry is None else np.ascontiguousarray(np.frombuffer(bytes(carry), dtype=np.uint8))


def dev_scan(lib, body, nbuf, carry, sm, capacity=None):
    capacity = capacity or nbuf * NS // 4
    cand = np.zeros(capacity, dtype=np.uint32)
    tiles = np.zeros(api.tiles_for(nbuf), dtype=api.TILE_DTYPE)
    counters = np.zeros(4, dtype=np.uint32)
    c = carry_arg(carry)
    rc = lib.dev_scan(body.ctypes.data, nbuf, None if c is None else c.ctypes.data, sm, capacity, cand.ctypes.data,
                      tiles.ctypes.data, counters.ctypes.data)
    assert rc == 0, lib.dev_error()
    return cand, tiles, counters


def dev_eval(lib, body, nbuf, carry, v, fix, aggressive, sm, capacity=None, counter=None):
    v = np.ascontiguousarray(v, dtype=np.uint32)
    out = np.zeros((v.size, REC), dtype=np.uint8)
    c = carry_arg(carry)
    rc = lib.dev_eval(body.ctypes.data, nbuf, None if c is None else c.ctypes.data, v.ctypes.data, v.size,
                      v.size if capacity is None else capacity, v.size if counter is None else counter,
                      fix, aggressive, sm, out.ctypes.data)
    assert rc == 0, lib.dev_error()
    return out


def eval_all(lib, monkeypatch, variant, *args, **kw):
    monkeypatch.setenv("MODES_EVAL_VARIANT", variant)
    return dev_eval(lib, *args, **kw)


def assert_records(got, want, what):
    assert got.shape == want.shape, f"{what}: {got.shape[0]} records, expected {want.shape[0]}"
    assert np.array_equal(got[:, :8], want[:, :8]), f"{what}: candidate positions differ"
    bad = np.flatnonzero((got != want).any(axis=1))
    assert bad.size == 0, (f"{what}: {bad.size} of {want.shape[0]} records differ, first at {bad[0]}: "
                           f"{got[bad[0]].tolist()} != {want[bad[0]].tolist()}")


def tile_order(tiles, counters):
    """K1's tile records: every tile written, the non-empty (offset, count) ranges disjoint and covering
    [0, counters[0]); the candidate array's indices in tile order."""
    assert not np.any((tiles["offset"] == 0xFFFFFFFF) & (tiles["count"] == 0xFFFFFFFF)), "a tile record was not written"
    ne = tiles[tiles["count"] > 0]
    by_off = np.sort(ne, order="offset")
    ends = by_off["offset"].astype(np.int64) + by_off["count"]
    assert by_off.size == 0 or by_off["offset"][0] == 0
    assert np.array_equal(by_off["offset"][1:].astype(np.int64), ends[:-1]), "tile ranges overlap or leave gaps"
    assert int(tiles["count"].sum(dtype=np.int64)) == int(counters[0])
    return np.concatenate([np.arange(o, o + c) for o, c in ne] or [np.zeros(0, int)]).astype(np.int64)


def check_scan(cand, tiles, counters, want_t):
    """K1 against the oracle's positions; returns (the positions as K1 left them, their order by tile)."""
    assert counters[1] == 0, "unexpected overflow"
    order = tile_order(tiles, counters)
    v = cand[order].astype(np.int64)
    tile_of = np.repeat(np.arange(tiles.size), tiles["count"])
    assert np.array_equal(v // TILE, tile_of), "a candidate listed under another tile"
    assert np.array_equal(v - 2, want_t), "K1's positions differ from the oracle's"
    return cand[: counters[0]].copy(), order


def k1_tiles_per_warp(lib, nbuf, sm):
    """A lower bound on the tiles every K1 warp takes: its grid is at most sm x (CTAs an SM holds), of
    one warp each (modes_scan2.cu: launch_scan), and at most one warp per tile."""
    n_tiles = api.tiles_for(nbuf)
    return n_tiles / min(n_tiles, sm * lib.max_ctas_per_sm)


def k2_chunks_per_warp(n, variant, sm):
    return -(-n // K2_CHUNK[variant]) / (sm * K2_WARPS_PER_SM[variant])


# ---------------------------------------------------------------- streams


def _dense_sparse():
    """The _periodic patterns of test_gpu_edges (more than 256 candidates per tile, more than 512
    survivors, exactly 256) laid into every other K1 tile, light traffic in between: dense tiles
    followed by fast-path tiles, over and over."""
    patterns = [[1, 0, 1, 0, 0, 0, 0, 1, 0, 1, 0, 0, 0, 0, 0], [1, 0, 1, 0, 0, 0, 0],
                [1, 0, 1, 0, 0, 0, 0, 1, 0, 1, 0, 0, 0, 0, 0, 0]]
    nsamp = 26 * NS - 5000
    data = synth.random_traffic(nsamp, 1500, 77)
    n_tiles = (nsamp + HALO) // TILE
    for k, g in enumerate(range(2, n_tiles, 2)):
        s0, s1 = g * TILE - HALO, (g + 1) * TILE - HALO               # body samples of virtual tile g
        data[2 * s0: 2 * s1] = GE._periodic(patterns[k % 3], s1 - s0)
    return data


def _streams():
    yield "traffic", lambda: synth.random_traffic(25 * NS - 3000, 8000, 5)
    yield "tie_rich", lambda: S.tie_rich(11, n_frames=11000)
    yield "alphabets", lambda: synth.tile_to(np.concatenate([d for _, _, d in S.random_alphabet_cases()]), 26 * BUF - 777)
    yield "dense_sparse", _dense_sparse


STREAMS = dict(_streams())


# ---------------------------------------------------------------- harness checks


def test_harness_refuses_invalid_requests(shim):
    """Nothing runs for an SM count outside [1, SMs], a window outside [0, 240 + N) or a capacity
    beyond the arrays."""
    body = np.full(BUF, 127, np.uint8)
    cand = np.zeros(64, np.uint32)
    tiles = np.zeros(api.tiles_for(1), api.TILE_DTYPE)
    counters = np.zeros(4, np.uint32)
    for sm in (0, -1, shim.sm_count + 1):
        assert shim.dev_scan(body.ctypes.data, 1, None, sm, 64, cand.ctypes.data, tiles.ctypes.data, counters.ctypes.data) != 0
    out = np.zeros((4, REC), np.uint8)
    for v in ([1, 300, 301, 302], [300, NS, 301, 302], [300, 301, 302, 0xFFFFFFFF]):
        vv = np.array(v, np.uint32)
        assert shim.dev_eval(body.ctypes.data, 1, None, vv.ctypes.data, 4, 4, 4, 1, 0, 1, out.ctypes.data) != 0
    vv = np.array([2, 300, NS - 1, 241], np.uint32)
    assert shim.dev_eval(body.ctypes.data, 1, None, vv.ctypes.data, 4, 5, 4, 1, 0, 1, out.ctypes.data) != 0
    assert shim.dev_eval(body.ctypes.data, 1, None, vv.ctypes.data, 4, 4, 4, 1, 0, 0, out.ctypes.data) != 0
    assert shim.dev_eval(body.ctypes.data, 1, None, vv.ctypes.data, 4, 4, 4, 1, 0, 1, out.ctypes.data) == 0, shim.dev_error()
    pos, cnt = np.zeros(8, np.uint32), np.zeros(1, np.uint32)
    assert shim.dev_weak(body.ctypes.data, 1, None, 1, 1, 1, 8, 8, pos.ctypes.data, cnt.ctypes.data) != 0
    assert shim.dev_weak(body.ctypes.data, 1, None, 0, 0, 1, 8, 8, pos.ctypes.data, cnt.ctypes.data) != 0
    assert shim.dev_weak(body.ctypes.data, 1, None, 0, 1, 1, 8, 8, pos.ctypes.data, cnt.ctypes.data) == 0, shim.dev_error()
    assert cnt[0] == 0


# ---------------------------------------------------------------- many tiles and chunks per warp


@pytest.mark.parametrize("name", list(STREAMS))
def test_many_tiles_and_chunks_per_warp(name, shim, checker_libs, monkeypatch):
    """K1 and every K2 variant at 1, 2 and 3 SMs (each warp through many tiles and chunks) and on the
    full grid: K1's positions, tile records and every evaluated record equal the oracle's."""
    body, nbuf = whole_buffers(STREAMS[name]())
    models = {f: oracle_model(body, None, *f) for f in FLAGS}
    want_t = rec_t(models[FLAGS[0]])
    n = want_t.size
    for sm in SM_COUNTS + [shim.sm_count]:
        cand, tiles, counters = dev_scan(shim, body, nbuf, None, sm)
        v, order = check_scan(cand, tiles, counters, want_t)
        if sm in SM_COUNTS:
            assert k1_tiles_per_warp(shim, nbuf, sm) >= MIN_ITERATIONS
        for variant in VARIANTS:
            if sm in SM_COUNTS:
                assert k2_chunks_per_warp(n, variant, sm) >= MIN_ITERATIONS, (variant, sm, n)
            for f in FLAGS:
                got = eval_all(shim, monkeypatch, variant, body, nbuf, None, v, *f, sm)
                assert_records(got[order], models[f], f"{name} {variant} sm={sm} fix,aggressive={f}")
    print(f"\n{name}: {nbuf} buffers, {n} candidates; at 1 SM >= {k1_tiles_per_warp(shim, nbuf, 1):.1f} tiles per K1 warp, "
          + ", ".join(f"{vv} {k2_chunks_per_warp(n, vv, 1):.1f}" for vv in VARIANTS) + " chunks per K2 warp")


def test_k1_capacity_across_many_tiles(shim, checker_libs):
    """K1 at one SM with room for a third of the candidates: the overflow flag, stored counts within
    the capacity, and every stored entry the oracle's candidate of that rank within its tile (which
    tiles get slots depends on the order the warps reach them)."""
    body, nbuf = whole_buffers(STREAMS["tie_rich"]())
    want_v = rec_t(oracle_model(body, None)) + 2
    capacity = want_v.size // 3
    cand, tiles, counters = dev_scan(shim, body, nbuf, None, 1, capacity)
    assert counters[0] == want_v.size and counters[1] == 1
    assert int(tiles["count"].sum(dtype=np.int64)) <= capacity
    ne = tiles[tiles["count"] > 0]
    by_off = np.sort(ne, order="offset")
    assert np.all(by_off["offset"][1:].astype(np.int64) >= by_off["offset"][:-1].astype(np.int64) + by_off["count"][:-1])
    assert np.all(by_off["offset"].astype(np.int64) + by_off["count"] <= capacity)
    per_tile = np.split(want_v, np.searchsorted(want_v // TILE, np.arange(1, tiles.size)))
    full = partial = 0
    for g in np.flatnonzero(tiles["count"]):
        o, c = int(tiles["offset"][g]), int(tiles["count"][g])
        assert c <= per_tile[g].size
        assert np.array_equal(cand[o: o + c], per_tile[g][:c]), f"tile {g}"
        full += c == per_tile[g].size
        partial += c < per_tile[g].size
    assert full > 10 and partial <= 1


# ---------------------------------------------------------------- the carry block


def _tie_window(frame, rng):
    """I/Q of a preamble + frame drawn from a few amplitudes: ties, weak pairs and copied bits."""
    bits = np.unpackbits(np.frombuffer(frame, np.uint8))
    amp = np.zeros(16 + 2 * bits.size, dtype=np.int64)
    amp[[0, 2, 7, 9]] = 110
    hi, lo = rng.choice([40, 100, 100, 1], bits.size), rng.choice([0, 0, 1, 40], bits.size)
    tie = rng.random(bits.size) < 0.25
    lo = np.where(tie, hi, lo)
    amp[16::2] = np.where(bits == 1, hi, lo)
    amp[17::2] = np.where(bits == 1, lo, hi)
    iq = np.full((amp.size, 2), 127, dtype=np.uint8)
    iq[:, 0] = np.clip(127 + amp, 0, 255)
    iq[:, 1] = 127 - rng.choice([0, 0, 1, 40, 100], amp.size) // 2
    return iq.ravel()


def _frame(k):
    rng = synth.Counter(1000 + k)
    icao = (0x400000 + rng.below(0x3FFFFF)).to_bytes(3, "big")
    if (k // 2) % 2 == 0:
        return synth.make_frame(17, 5, icao + bytes(rng.below(256) for _ in range(7)))
    return synth.make_frame(11, 5, icao)


def carry_batch(t0, style):
    """One buffer whose batch position t0 holds a DF17 or DF11 preamble (stream sample t0 - 238: for
    t0 < 238 it starts in the carry), with strong or tie-rich amplitudes.  (body, carry)."""
    frame = _frame(t0)
    s = NS - 238 + t0                                      # its first sample in [pad buffer, body]
    if style == "strong":
        stream = synth.synth_stream(2 * NS, [(s, frame, 80.0, 0.3 * t0, 0.3 * ((t0 >> 1) & 1))], sigma=1.2, seed=t0)
    else:
        stream = synth.synth_stream(2 * NS, [], sigma=1.0, seed=t0)
        win = _tie_window(frame, np.random.default_rng(t0))
        stream[2 * s: 2 * s + win.size] = win
    return np.ascontiguousarray(stream[BUF:]), bytes(stream[BUF - CARRY: BUF])


def test_carry_block_preambles(shim, gpu_decoder_factory, checker_libs, monkeypatch):
    """A preamble at every t in [0, 254) of a batch's first buffer (the window starting in the carry
    block up to t = 238, v = t + 2 around kHaloSamples = 240), strong and tie-rich: the public path
    with the default kernels, and all five K2 variants, record for record."""
    import torch
    dec = gpu_decoder_factory()
    halo_seen = 0
    for style in ("strong", "ties"):
        for t0 in range(254):
            body, carry = carry_batch(t0, style)
            want = oracle_model(body, carry)
            t = rec_t(want)
            assert t0 in t, (style, t0)
            halo_seen += int(np.count_nonzero(t <= HALO - 2))
            monkeypatch.delenv("MODES_EVAL_VARIANT", raising=False)
            d = torch.from_numpy(body).cuda()
            dec.detect_device(d.data_ptr(), 1, carry)
            cands, tiles = dec.detect_fetch(1)
            order = np.concatenate([np.arange(o, o + c) for o, c in tiles] or [np.zeros(0, int)]).astype(int)
            assert_records(cands.view(np.uint8).reshape(-1, REC)[order], want, f"public {style} t={t0}")
            f = FLAGS[t0 % 3]
            want_f = want if f == (1, 0) else oracle_model(body, carry, *f)
            for variant in VARIANTS:
                got = eval_all(shim, monkeypatch, variant, body, 1, carry, t + 2, *f, shim.sm_count)
                assert_records(got, want_f, f"{variant} {style} t={t0} fix,aggressive={f}")
    assert halo_seen >= 2 * 239


# ---------------------------------------------------------------- fabricated candidate lists


def _corrupt_df17(rng, flips):
    icao = (0x400000 + rng.below(0x3FFFFF)).to_bytes(3, "big")
    return synth.flip_bits(synth.make_frame(17, 5, icao + bytes(rng.below(256) for _ in range(7))),
                           [rng.below(112) for _ in range(flips)])


def fabricated_batch():
    """Four buffers and a carry with candidates in the carry block (a periodic preamble pattern across
    it), at j = 0 of every buffer (first attempts that fail: the retry without phase correction), at
    j = 131069 of the last buffer, and traffic in both walk directions.  (body, nbuf, carry)."""
    nb = 4
    rng = synth.Counter(4242)
    frames = []
    for k in range(nb):                                                   # j = 0 of buffer k
        frames.append((NS * (k + 1) - 238, _corrupt_df17(rng, 3), 70.0 + 5 * k, 0.4 * k, 0.0))
    for i in range(1200):                                                 # both walk directions
        s = NS + 1000 + 420 * i + rng.below(50)
        if abs((s + 238) % NS - NS / 2) > NS / 2 - 600:                   # clear of the frames at j = 0
            continue
        frames.append((s, _corrupt_df17(rng, i % 3), 15.0 + rng.below(90), 0.1 * i, [0.0, 0.3, 0.6, 0.8][i % 4]))
    frames.append((NS + nb * NS - 3 - 238, _corrupt_df17(rng, 1), 80.0, 0.5, 0.2))   # j = 131069 of the last buffer
    stream = synth.synth_stream((nb + 1) * NS, frames, sigma=1.5, seed=4242)
    s0, s1 = NS - 238, NS + 200
    stream[2 * s0: 2 * s1] = GE._periodic([1, 0, 1, 0, 0, 0, 0, 1, 0, 1, 0, 0, 0, 0, 0], s1 - s0)
    return np.ascontiguousarray(stream[BUF:]), nb, bytes(stream[BUF - CARRY: BUF])


def backwards(body, carry, v):
    """Which positions the phase-corrected retry walks backwards: early > late of dump1090.c:1498-1517,
    early = 2 (m[-1] + m[6]), late = 2 (m[3] + m[10]), m[x] = virtual sample v + x.  Used only to
    compose the lists."""
    virt = np.concatenate([np.full(4, 127, np.uint8), np.frombuffer(carry, np.uint8), body])
    mag = R.magnitudes(virt).astype(np.int64)
    m = lambda x: mag[v + x]
    return (m(-1) + m(6)) * 2 > (m(3) + m(10)) * 2


def fabricated_lists(t, body, nbuf, carry):
    """Named position lists (v = t + 2) drawn from the oracle's candidates t."""
    v = t + 2
    halo, inner = v[v <= HALO], v[v > HALO]
    back = backwards(body, carry, inner)
    fwd, bwd = inner[~back], inner[back]
    j0 = v[(t % NS) == 0]
    last = v[t == nbuf * NS - NS + LAST_J]
    assert halo.size >= 8 and fwd.size >= 64 and bwd.size >= 64 and j0.size == nbuf and last.size == 1
    cyc = lambda a, n, s=0: a[(s + np.arange(n)) % a.size]
    alt = np.empty(32, np.int64)
    alt[0::2], alt[1::2] = fwd[:16], bwd[:16]
    mixed = np.concatenate([v[::7], v[1::5]])
    blocks = {
        "all_halo": cyc(halo, 32),
        "halo_lane0": np.concatenate([halo[:1], cyc(inner, 31, 5)]),
        "halo_lane31": np.concatenate([cyc(inner, 31, 9), halo[-1:]]),
        "halo_31_body_1": np.concatenate([cyc(halo, 31, 1), inner[:1]]),
        "body_1_halo_31": np.concatenate([inner[-1:], cyc(halo, 31, 2)]),
        "repeats": np.full(32, inner[inner.size // 2]),
        "forward": fwd[:32], "backward": bwd[:32], "alternating": alt,
        "seams": cyc(np.concatenate([j0, last]), 32),
    }
    # each chunk of 32 is one composition (and so one warp's walk directions, or its staging path)
    assert not backwards(body, carry, blocks["forward"]).any() and backwards(body, carry, blocks["backward"]).all()
    assert np.array_equal(backwards(body, carry, alt), np.arange(32) % 2 == 1)
    assert (blocks["all_halo"] <= HALO).all() and np.count_nonzero(blocks["halo_lane0"] <= HALO) == 1
    assert np.count_nonzero(blocks["halo_31_body_1"] <= HALO) == 31
    composed = np.concatenate(list(blocks.values()))
    lists = {"composed": composed, "reverse": v[::-1].copy()}
    for n in (1, 31, 32, 33):
        lists[f"n{n}"] = mixed[:n]
    lists["n2049"] = cyc(np.concatenate([composed, mixed]), 32 * 64 + 1)
    return lists


def test_fabricated_candidate_lists(shim, checker_libs, monkeypatch):
    """K2 on lists no scan produces but the kernels must take: windows in the carry block in every
    lane mix, repeats, reverse stream order, 1 to 32k+1 candidates, the j = 0 retry of every buffer
    and j = 131069 of the last, chunks that walk all forwards, all backwards or alternately; and the
    hand-out bounded by min(counter, capacity), the records beyond it untouched."""
    body, nbuf, carry = fabricated_batch()
    models = {f: oracle_model(body, carry, *f) for f in FLAGS}
    t = rec_t(models[FLAGS[0]])
    by_v = {f: dict(zip((rec_t(m) + 2).tolist(), m)) for f, m in models.items()}
    lists = fabricated_lists(t, body, nbuf, carry)
    for name, v in lists.items():
        for f in FLAGS:
            want = np.stack([by_v[f][int(x)] for x in v])
            for variant in VARIANTS:
                for sm in (1, shim.sm_count):
                    got = eval_all(shim, monkeypatch, variant, body, nbuf, carry, v, *f, sm)
                    assert_records(got, want, f"{name} {variant} sm={sm} fix,aggressive={f}")
    v = lists["n2049"]
    want = np.stack([by_v[(1, 0)][int(x)] for x in v])
    for variant in VARIANTS:
        assert k2_chunks_per_warp(v.size, variant, 1) >= MIN_ITERATIONS
        for capacity in (v.size, v.size - 37):
            for counter in (capacity + 5, capacity, capacity - 50, 0):
                got = eval_all(shim, monkeypatch, variant, body, nbuf, carry, v, 1, 0, 1, capacity, counter)
                k = min(capacity, counter)
                assert_records(got[:k], want[:k], f"{variant} capacity={capacity} counter={counter}")
                assert (got[k:] == SENTINEL).all(), f"{variant}: records written past min(counter, capacity) = {k}"


# ---------------------------------------------------------------- full grid, one large batch


def test_full_grid_one_large_batch(gpu_decoder_factory, checker_libs, monkeypatch):
    """The capture tiled to 1 GiB through the public path on the full grid: about 43 tiles per K1 warp
    and 17 chunks per K2 warp; every record equals the oracle's, for fused and fused2."""
    import torch
    body, nbuf = whole_buffers(synth.tile_to(C.modes1(), 1 << 30))
    want = oracle_records(body, cap=1 << 20)
    d = torch.from_numpy(body).cuda()
    dec = gpu_decoder_factory()
    for variant in ("fused", "fused2"):
        monkeypatch.setenv("MODES_EVAL_VARIANT", variant)
        dec.detect_device(d.data_ptr(), nbuf)
        cands, tiles = dec.detect_fetch(nbuf)
        order = np.concatenate([np.arange(o, o + c) for o, c in tiles if c]).astype(np.int64)
        assert_records(cands.view(np.uint8).reshape(-1, REC)[order], want, variant)
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    print(f"\n1 GiB: {want.shape[0]} candidates, {tiles.size} tiles: {tiles.size / (12 * n_sm):.1f} tiles per K1 warp "
          f"(12 warps per SM), {want.shape[0] / 32 / (12 * n_sm):.1f} chunks per fused warp")
    assert want.shape[0] > 800000


# ---------------------------------------------------------------- weak preambles across order rounds


def _weak_window():
    """The DF17 window of test_weak_device_edges: weak, and the reference's test fails (m3 > m2)."""
    win = np.full(2 * 30, 127, np.uint8)
    amps = np.zeros(30)
    amps[[0, 2, 7, 9]] = 40
    amps[[4, 11]] = 2
    amps[3] = 45
    for i, bit in enumerate([1, 0, 0, 0, 1]):
        amps[16 + 2 * i + (1 - bit)] = 30
    win[0::2] = (127 + amps).astype(np.uint8)
    return win


def test_weak_order_rounds(shim, gpu_decoder_factory, checker_libs):
    """A batch of 520 buffers (16 640 weak-scan tiles: weak_order_kernel works in rounds of 16 384),
    silent but for weak windows in buffers 0, 511, 512, 513 and the last, some within 32 tiles of the
    round boundary: the public list and the harness at one SM equal the restatement."""
    import torch
    nbuf = 520
    planted = [0, 511, 512, 513, nbuf - 1]
    stream = np.full(nbuf * BUF, 127, np.uint8)
    win = _weak_window()
    for b in planted:
        for j in (300, 4096 * 31 + 77, 65536 + 11, LAST_J - 40, LAST_J):
            s = b * NS + j - 238
            stream[2 * s: 2 * s + win.size] = win
    want = []
    for b in planted:                          # the restatement, buffer by buffer (the rest is silent)
        prev = stream[(b - 1) * BUF: b * BUF] if b else np.full(BUF, 127, np.uint8)
        t = W.weak_positions(np.concatenate([prev, stream[b * BUF: (b + 1) * BUF]]), 2).astype(np.int64)
        want.append(t[t >= NS] - NS + b * NS)
    want = np.concatenate(want)
    assert want.size >= 5 * len(planted)
    d = torch.from_numpy(stream).cuda()
    dec = gpu_decoder_factory()
    dec.detect_device(d.data_ptr(), nbuf)
    dec.weak_device()
    n, t, _ = dec.weak_fetch()
    assert n == want.size and np.array_equal(t.astype(np.int64), want)
    pos, cnt = np.zeros(want.size + 16, np.uint32), np.zeros(1, np.uint32)
    rc = shim.dev_weak(stream.ctypes.data, nbuf, None, 0, 1, 1, pos.size, 4096, pos.ctypes.data, cnt.ctypes.data)
    assert rc == 0, shim.dev_error()
    assert cnt[0] == want.size
    assert np.array_equal(pos[: want.size].astype(np.int64), want) and (pos[want.size:] == 0xFFFFFFFF).all()
