"""-m gpu: the device resolve (K3, modes_resolve_gpu.cu) record for record, at the grids and batch sizes
where its kernels take more than one item of work, and the hex door's address-cache writes carried into
device-resolved batches.

The replay kernel runs at most 4 CTAs of 8 warps per SM and strides over the buffers, so a warp takes a
second buffer (reloading its shared cache, restarting its written / read-first sets, skipping buffers
that need no replay) only in batches of more than 32 * SM count buffers; the offsets kernel gives each
of its 1024 threads more than one buffer only past 1024 buffers.  The product's default batch is 256
buffers.  The device harness tests/device_shim/resolve_device.cu (linked against the product's own
object) runs launch_gpu_resolve with a chosen SM count and delivery capacity on batches of any size.

The resolve reads only candidate records and tiles, so the batches are built without I/Q: whole buffers
of the oracle's candidate records from a set of source streams are relocated into target buffers
(t' = t - 131072 k + 131072 b) and tiled; tiles straddle buffers as they do in real batches.  The address
chains of tests/streams.py keep their buffers consecutive, so their dependency through the cache (which
the fixed rounds cannot settle, so the in-order fallback runs) survives.  Expected values come from the
product's sequential host resolver on the same arrays: the deliveries, statistics and end cache from one
run over the batch, each buffer's start cache and delivery count from a run fed one buffer at a time."""
import functools
import hashlib
import subprocess

import ctypes
import numpy as np
import pytest

import checker as C
import repair_corpus as R
import streams as S
from dump1090_b200 import api, synth

pytestmark = pytest.mark.gpu

ROOT = C.ROOT
DSHIM = ROOT / "tests" / "_build" / "libresolve_device.so"
HSHIM = ROOT / "tests" / "_build" / "libresolve_core_host.so"
NS = api.BUFFER_SAMPLES
BUF = api.BUFFER_BYTES
WARPS_PER_SM = 32                         # the replay grid: at most 4 CTAs of 8 warps per SM
ROUNDS = 4                                # replay + hand-over rounds before the in-order fallback
EVAL_DTYPE = api.CANDIDATE_DTYPE["p"].base
DELIVERY_DTYPE = np.dtype([("t", "<i8"), ("eval", EVAL_DTYPE), ("extra", "<u4"), ("bits", "<u4")])
assert DELIVERY_DTYPE.itemsize == 40
MSG_DTYPE = np.dtype(api.Message)
AP_FORMATS = (0, 4, 5, 16, 20, 21, 24)
GATE_DECODED = 1 | 4                      # MODES_EVAL_GATE_OK | MODES_EVAL_DECODED


# ---------------------------------------------------------------- the harnesses


@pytest.fixture(scope="module")
def dev():
    subprocess.run(["make", "-s", "dshim"], cwd=ROOT, check=True)
    lib = ctypes.CDLL(str(DSHIM))
    u32, u64, i32, p = ctypes.c_uint32, ctypes.c_uint64, ctypes.c_int, ctypes.c_void_p
    lib.dev_error.restype = ctypes.c_char_p
    lib.dev_limits.argtypes = [p]
    lib.dev_resolve.argtypes = [p, u64, p, u32, u32, p, i32, i32, u32, u32, p, p, p, p, p, p, p]
    lim = np.zeros(3, np.int32)
    assert lib.dev_limits(lim.ctypes.data) == 0, lib.dev_error()
    lib.sm_count, lib.guard, lib.guard_byte = int(lim[0]), int(lim[1]), int(lim[2])
    assert lib.sm_count >= 3 and lib.guard > 0
    return lib


@pytest.fixture(scope="module")
def host_shim(checker_libs):
    subprocess.run(["make", "-s", "shim"], cwd=ROOT, check=True)
    lib = ctypes.CDLL(str(HSHIM))
    lib.shim_resolve_buffers.restype = ctypes.c_long
    return lib


def run_device(dev, arr, tiles, n_buffers, cache0, check_crc, sm_count, capacity, alloc=None):
    """The harness's outputs as a dict; the delivery array covers the whole allocation and its guard."""
    alloc = capacity if alloc is None else alloc
    out = np.zeros(alloc + dev.guard, DELIVERY_DTYPE)
    r = dict(out=out, stats=np.zeros(8, np.uint64), flags=np.zeros(3, np.uint32), cache=np.zeros(1024, np.uint32),
             n_deliv=np.zeros(n_buffers, np.uint32), offsets=np.zeros(n_buffers + 1, np.uint32),
             start=np.zeros((n_buffers, 1024), np.uint32))
    cache0 = np.ascontiguousarray(cache0, np.uint32)
    rc = dev.dev_resolve(arr.ctypes.data if arr.size else None, arr.size, tiles.ctypes.data, tiles.size, n_buffers,
                         cache0.ctypes.data, int(check_crc), int(sm_count), int(capacity), int(alloc), out.ctypes.data,
                         r["stats"].ctypes.data, r["flags"].ctypes.data, r["cache"].ctypes.data, r["n_deliv"].ctypes.data,
                         r["offsets"].ctypes.data, r["start"].ctypes.data)
    assert rc == 0, dev.dev_error()
    return r


def needs_fallback(host_shim, arr, tiles, n_buffers, cache0, check_crc):
    """Whether the device's schedule (ROUNDS rounds of guessing) leaves the caches unsettled, by the CPU
    restatement of the same algorithm (tests/host_shim/resolve_core_host.cpp); also its delivery count."""
    out = (ctypes.c_int64 * 8)()                                         # room for no delivery: cap = 0
    stats = (ctypes.c_int64 * 8)()
    start = np.ascontiguousarray(cache0, np.uint32)
    end = np.zeros(1024, np.uint32)
    rounds, fallback = ctypes.c_int(0), ctypes.c_int(0)
    n = host_shim.shim_resolve_buffers(arr.ctypes.data_as(ctypes.c_void_p), tiles.ctypes.data_as(ctypes.c_void_p),
                                       ctypes.c_size_t(tiles.size), ctypes.c_size_t(n_buffers), int(check_crc),
                                       start.ctypes.data_as(ctypes.c_void_p), out, ctypes.c_size_t(0), stats,
                                       end.ctypes.data_as(ctypes.c_void_p), ctypes.byref(rounds), api.TILE_SAMPLES,
                                       ROUNDS, ctypes.byref(fallback))
    assert n >= 0
    return bool(fallback.value), int(n)


# ---------------------------------------------------------------- source records and composed batches


def _tiled(arr, n_buffers):
    g = (arr["t"] + 2) // api.TILE_SAMPLES
    nt = api.tiles_for(n_buffers)
    cnt = np.bincount(g, minlength=nt).astype(np.uint32)
    t = np.zeros(nt, dtype=api.TILE_DTYPE)
    t["count"] = cnt
    t["offset"] = np.concatenate([[0], np.cumsum(cnt)[:-1]])
    return t


@functools.lru_cache(maxsize=None)
def _streams():
    s = {"modes1": C.modes1(),
         "traffic": synth.random_traffic(131072 * 9 + 5000, 1500, 77, n_aircraft=20),
         "dense_fleet": synth.random_traffic(131072 * 30, 9000, 5, n_aircraft=60),
         # a preamble every 60 samples: with check_crc = 0 nearly every candidate delivers both attempts
         "dense_ties": S.tie_rich(21, n_frames=17800, levels=(0, 40, 100), period=60),
         "retry_at_j0": S.retry_at_buffer_start(),
         "repair0": R.repair_stream(0.0),
         "repair_frac": R.repair_stream(R.RETRY_FRAC)}
    s.update(S.chain_streams())
    return s


FILLERS = ["modes1", "traffic", "dense_fleet", "dense_ties", "retry_at_j0", "repair0", "repair_frac"]


@functools.lru_cache(maxsize=None)
def _pool(fix, aggressive):
    """stream name -> the oracle's candidate records of each of its buffers, t relative to the buffer.
    A chain keeps only the buffers of its chain (not the empty end-of-stream buffer)."""
    pool = {}
    for name, data in _streams().items():
        cands = C.oracle_scan_candidates(data, fix=fix, aggressive=aggressive, cap=400000)
        arr = np.frombuffer(b"".join(bytes(c) for c in cands), dtype=api.CANDIDATE_DTYPE).copy()
        nbuf = S.CHAINS[name][1] if name in S.CHAINS else data.size // BUF + 1
        bounds = np.searchsorted(arr["t"], np.arange(nbuf + 1, dtype=np.int64) * NS)
        pool[name] = []
        for k in range(nbuf):
            r = arr[bounds[k]: bounds[k + 1]].copy()
            r["t"] -= k * NS
            pool[name].append(r)
    return pool


def compose(n_buffers, chains=(), seed=0, fix=1, aggressive=0, pieces=()):
    """A batch of n_buffers buffers: each chain (name, first buffer) at consecutive buffers from its first
    buffer on, each piece (name, source buffer, target buffer) at its target buffer, every other buffer a
    source buffer drawn from FILLERS in a fixed pseudo-random order.  Returns (records, tiles, layout)."""
    pool = _pool(fix, aggressive)
    fill = [(n, k) for n in FILLERS for k in range(len(pool[n]))]
    rng = np.random.default_rng(1000 + seed)
    layout = [fill[i] for i in rng.integers(0, len(fill), n_buffers)]
    for name, first in chains:
        n = len(pool[name])
        assert 0 <= first and first + n <= n_buffers, (name, first, n_buffers)
        layout[first: first + n] = [(name, k) for k in range(n)]
    for name, k, b in pieces:
        layout[b] = (name, k)
    parts = []
    for b, (name, k) in enumerate(layout):
        r = pool[name][k].copy()
        r["t"] += b * NS
        parts.append(r)
    arr = np.concatenate(parts)
    return arr, _tiled(arr, n_buffers), layout


def random_cache(arr, seed):
    """A start cache with a random address in about half the slots and, over them, the addresses of
    about half the batch's address/parity replies (their syndromes) in their own slots."""
    rng = np.random.default_rng(seed)
    cache = np.where(rng.random(1024) < 0.5, rng.integers(1, 1 << 24, 1024), 0).astype(np.uint32)
    p = arr["p"][:, 0]
    replies = np.unique(p["crc"][np.isin(p["msgtype"], AP_FORMATS) & (p["crc"] != 0)])
    for a in replies[rng.random(replies.size) < 0.5]:
        cache[S.icao_slot(int(a))] = a
    return cache


def expected(arr, tiles, n_buffers, cache0, check_crc, fix, aggressive):
    """The product's sequential host resolver on the same arrays: (messages, statistics, end cache) from
    one run over the batch; (start caches, delivery counts) from a run fed one buffer at a time."""
    kw = dict(fix_errors=fix, aggressive=aggressive, check_crc=check_crc)
    cap = 2 * arr.size + 16
    seq = api.Resolver(**kw)
    seq.set_cache(cache0)
    out = seq.set_output_array(cap)
    seq.run(arr, tiles)
    msgs = np.frombuffer(out, dtype=MSG_DTYPE, count=seq.output_count()).copy()
    stats, end = list(seq.stats().values()), seq.get_cache()
    seq.close()

    per = api.Resolver(**kw)
    per.set_cache(cache0)
    per.set_output_array(cap)
    starts = np.zeros((n_buffers, 1024), np.uint32)
    counts = np.zeros(n_buffers, np.int64)
    bounds = np.searchsorted(arr["t"], np.arange(n_buffers + 1, dtype=np.int64) * NS)
    for b in range(n_buffers):
        starts[b] = per.get_cache()
        r = arr[bounds[b]: bounds[b + 1]].copy()
        r["t"] -= b * NS
        c0 = per.output_count()
        per.run(r, _tiled(r, 1), buffer_base=b)
        counts[b] = per.output_count() - c0
    assert np.array_equal(per.get_cache(), end) and counts.sum() == msgs.size
    per.close()
    return msgs, stats, end, starts, counts


def check_deliveries(got, want, arr):
    """Device deliveries (DELIVERY_DTYPE) against the host resolver's messages, in order: position, the
    attempt delivered (the record's pass, all 24 bytes), frame bytes, crcok, phase_corrected, the
    address of an address/parity reply or the DF11 interrogator id."""
    n = want.size
    assert got.size == n
    t = got["t"]
    bad = np.flatnonzero(t - 238 != want["sample_pos"])
    assert bad.size == 0, f"delivery {bad[0]}: t = {t[bad[0]]}, expected sample_pos {want['sample_pos'][bad[0]]}"
    idx = np.searchsorted(arr["t"], t)
    assert np.array_equal(arr["t"][idx], t)
    rec = arr[idx]
    # the pass: two deliveries at one position are its first attempt and its retry; one alone is the retry
    # when it is phase-corrected or the first attempt did not pass the gate and decode
    same_prev = np.r_[False, t[1:] == t[:-1]]
    same_next = np.r_[t[1:] == t[:-1], False]
    first_ok = (rec["p"][:, 0]["flags"] & GATE_DECODED) == GATE_DECODED
    alone = np.where((want["phase_corrected"] != 0) | ~first_ok, 1, 0)
    want_pass = np.where(same_prev, 1, np.where(same_next, 0, alone))
    ev = np.ascontiguousarray(rec["p"][np.arange(n), want_pass]).view(np.uint8).reshape(n, EVAL_DTYPE.itemsize)
    gev = np.ascontiguousarray(got["eval"]).view(np.uint8).reshape(n, EVAL_DTYPE.itemsize)
    diff = np.flatnonzero((gev != ev).any(axis=1))
    assert diff.size == 0,f"delivery {diff[0]} at t = {t[diff[0]]}: not pass {want_pass[diff[0]]} of its record"
    nbytes = want["msgbits"] // 8
    mask = np.arange(14)[None, :] < nbytes[:, None]
    assert np.array_equal(np.where(mask, got["eval"]["msg"], 0), np.where(mask, want["msg"], 0))
    bits = got["bits"]
    assert np.array_equal(bits & 1, want["crcok"]) and np.array_equal((bits >> 8) & 1, want["phase_corrected"])
    assert not (bits & ~np.uint32(0x10101)).any()
    is_ap = (bits >> 16) & 1 == 1
    aa = (want["aa1"].astype(np.uint32) << 16) | (want["aa2"].astype(np.uint32) << 8) | want["aa3"].astype(np.uint32)
    assert np.array_equal(got["extra"][is_ap], aa[is_ap])
    assert np.array_equal(got["extra"][~is_ap].astype(np.int64), want["iid"][~is_ap].astype(np.int64))
    assert np.isin(got["eval"]["msgtype"][is_ap], AP_FORMATS).all()


def check_batch(dev, host_shim, n_buffers, sm_count, chains=(), seed=0, cache="zero", check_crc=1, fix=1, aggressive=0,
                capacity=None, pieces=()):
    """One batch through the device resolve against the host resolver; capacity: None for room for every
    delivery (two per candidate, as the product sizes it), else a number or a function of the total."""
    arr, tiles, _ = compose(n_buffers, chains, seed, fix, aggressive, pieces)
    cache0 = np.zeros(1024, np.uint32) if cache == "zero" else random_cache(arr, seed)
    msgs, stats, end, starts, counts = expected(arr, tiles, n_buffers, cache0, check_crc, fix, aggressive)
    total = int(counts.sum())
    fallback, n_shim = needs_fallback(host_shim, arr, tiles, n_buffers, cache0, check_crc)
    assert n_shim == total
    if chains:
        assert fallback, "the batch's chains settle within the fixed rounds: the in-order fallback is not reached"
    alloc = 2 * arr.size + 16                        # every delivery the batch can make: writes past cap stay in range
    cap = alloc if capacity is None else capacity(total)
    r = run_device(dev, arr, tiles, n_buffers, cache0, check_crc, sm_count, cap, alloc)
    assert r["flags"][0] == 0
    assert r["flags"][2] == total
    assert r["flags"][1] == (1 if total > cap else 0)
    assert np.array_equal(r["n_deliv"], counts), f"first wrong count: buffer {np.flatnonzero(r['n_deliv'] != counts)[:1]}"
    assert np.array_equal(r["offsets"], np.concatenate([[0], np.cumsum(counts)]))
    bad = np.flatnonzero((r["start"] != starts).any(axis=1))
    assert bad.size == 0, f"start cache of buffer {bad[0]} differs"
    assert np.array_equal(r["cache"], end)
    assert [int(v) for v in r["stats"]] == stats
    written = min(total, cap)
    check_deliveries(r["out"][:written], msgs[:written], arr)
    untouched = r["out"][written:].view(np.uint8)
    assert (untouched == dev.guard_byte).all(), \
        f"deliveries written at or past {written} (capacity {cap}, allocation {alloc} + guard {dev.guard})"
    return total, fallback


# ---------------------------------------------------------------- cases


def _warp_chains(n_buffers):
    """Chains across warp boundaries (warps take consecutive buffers: buffers 30-41 span three warps at
    one SM's 32 warps, and the next warp in a CTA of 8), and one that ends at the batch's last buffer."""
    want = [("chain_df4", 30), ("chain_df20", 90), ("chain_df11_iid", 125), ("chain_evict", 190)]
    out = [(n, f) for n, f in want if f + S.CHAINS[n][1] <= n_buffers]
    if n_buffers >= 250:
        out.append(("chain_seam", n_buffers - S.CHAINS["chain_seam"][1]))
    return out


@pytest.mark.parametrize("n_buffers", [1, 31, 32, 33, 64, 65, 97, 257])
@pytest.mark.parametrize("sm_count", [1, 2, 3])
def test_multi_buffer_warps(dev, host_shim, sm_count, n_buffers):
    """32 * sm_count warps over more buffers: the rerun skip between two buffers of one warp, the shared
    cache reloaded and the written / read-first sets restarted for each buffer."""
    check_batch(dev, host_shim, n_buffers, sm_count, _warp_chains(n_buffers), seed=n_buffers)


@pytest.mark.parametrize("sm_count", [1, 3, 0], ids=["sm1", "sm3", "full_grid"])
def test_warp_restarts_its_sets_per_buffer(dev, host_shim, sm_count):
    """A writer buffer and its reader one grid stride later, so that one warp replays both: the reader's
    first read of the writer's slot must mark it read-first (and so replayed with the inherited cache), whatever
    the warp's previous buffer wrote.  Two-buffer dependencies settle in the fixed rounds: no fallback hides
    a wrong verdict of the rounds."""
    sm = sm_count or dev.sm_count
    w = WARPS_PER_SM * sm
    n = w + 40 if not sm_count else 2 * w + 40
    pairs = []
    for i, name in enumerate(S.CHAINS):
        pairs += [(name, 0, 5 + 7 * i), (name, 1, 5 + 7 * i + w)]
    _, fallback = check_batch(dev, host_shim, n, sm, seed=13, pieces=pairs)
    assert not fallback


@pytest.mark.parametrize("cache", ["zero", "random"])
@pytest.mark.parametrize("sm_count", [1, 3])
def test_start_cache(dev, host_shim, sm_count, cache):
    check_batch(dev, host_shim, 257, sm_count, _warp_chains(257), seed=7, cache=cache)


@pytest.mark.parametrize("n_buffers", [1023, 1024, 1025, 2048, 2049, 4096])
@pytest.mark.parametrize("full", [True, False], ids=["full_grid", "one_sm"])
def test_offsets_past_1024_buffers(dev, host_shim, n_buffers, full):
    """The offsets kernel's 1024 threads take ceil(n / 1024) buffers each."""
    mid = n_buffers // 2
    check_batch(dev, host_shim, n_buffers, dev.sm_count if full else 1, [("chain_df4", mid), ("chain_df20", mid + 20)],
                seed=n_buffers, cache="random" if n_buffers % 2 else "zero")


def _grid_sizes(sm_count):
    w = WARPS_PER_SM * sm_count
    return [w + 1, 2 * w + 5]


@pytest.mark.parametrize("which", [0, 1])
@pytest.mark.parametrize("cache", ["zero", "random"])
def test_past_the_full_grid(dev, host_shim, which, cache):
    """More buffers than the full grid has warps, with chains at the start, the middle and the end of the
    batch (the last one ending at its last buffer): the in-order fallback over thousands of buffers."""
    n = _grid_sizes(dev.sm_count)[which]
    seam = S.CHAINS["chain_seam"][1]
    chains = [("chain_df4", 0), ("chain_df11_iid", n // 2 - 4), ("chain_evict", n // 2 + 40), ("chain_seam", n - seam)]
    total, _ = check_batch(dev, host_shim, n, dev.sm_count, chains, seed=11 + which, cache=cache)
    assert total > n


def test_past_the_full_grid_settled(dev, host_shim):
    """The same geometry without chains: the rounds settle the caches and the fallback returns at once."""
    n = _grid_sizes(dev.sm_count)[0]
    check_batch(dev, host_shim, n, dev.sm_count, (), seed=21, cache="random")


FLAG_SETS = [dict(check_crc=0), dict(aggressive=1), dict(fix=0), dict(check_crc=0, aggressive=1)]


@pytest.mark.parametrize("kw", FLAG_SETS, ids=lambda k: "-".join(f"{a}{b}" for a, b in k.items()))
@pytest.mark.parametrize("geometry", ["sm2_97", "full_grid"])
def test_flags(dev, host_shim, kw, geometry):
    """check_crc = 0 (both attempts of a candidate delivered) and the repair flags the records were made with."""
    sm, n = (2, 97) if geometry == "sm2_97" else (dev.sm_count, _grid_sizes(dev.sm_count)[0])
    chains = _warp_chains(n) if n < 1000 else [("chain_df4", 0), ("chain_df20", n - S.CHAINS["chain_df20"][1])]
    check_batch(dev, host_shim, n, sm, chains, seed=3, check_crc=kw.get("check_crc", 1), fix=kw.get("fix", 1),
                aggressive=kw.get("aggressive", 0))


CAPACITIES = {"exact": lambda n: n, "one_short": lambda n: n - 1, "half": lambda n: n // 2}


@pytest.mark.parametrize("capacity", list(CAPACITIES))
@pytest.mark.parametrize("geometry", ["sm2_257", "full_grid"])
def test_delivery_capacity(dev, host_shim, capacity, geometry):
    """A delivery buffer of exactly the total, one short of it and about half of it: flags[1] is raised
    exactly when the total exceeds the capacity, nothing is written at or past it, and what is below it
    is the expected deliveries.  check_crc = 0 spreads the deliveries over every buffer."""
    sm, n = (2, 257) if geometry == "sm2_257" else (dev.sm_count, _grid_sizes(dev.sm_count)[0])
    total, _ = check_batch(dev, host_shim, n, sm, _warp_chains(n) if n < 1000 else [("chain_df4", 5)], seed=5,
                           check_crc=0, capacity=CAPACITIES[capacity])
    assert total > 10 * n


def test_invalid_requests_run_nothing(dev):
    arr, tiles, _ = compose(3, (), seed=1)
    cache0 = np.zeros(1024, np.uint32)
    alloc = 2 * arr.size + 16
    out = np.zeros(alloc + dev.guard, DELIVERY_DTYPE)
    small = [np.zeros(k, t) for k, t in ((8, np.uint64), (3, np.uint32), (1024, np.uint32), (3, np.uint32), (4, np.uint32),
                                          (3 * 1024, np.uint32))]

    def call(records=arr, n_records=None, tl=tiles, n_tiles=None, n_buffers=3, sm=1, capacity=alloc, alloc=alloc):
        return dev.dev_resolve(records.ctypes.data, records.size if n_records is None else n_records, tl.ctypes.data,
                               tl.size if n_tiles is None else n_tiles, n_buffers, cache0.ctypes.data, 1, sm, capacity,
                               alloc, out.ctypes.data, *[a.ctypes.data for a in small])
    assert call(sm=0) != 0 and call(sm=dev.sm_count + 1) != 0
    assert call(n_buffers=0) != 0
    assert call(n_tiles=tiles.size - 1) != 0
    assert call(n_records=arr.size - 1) != 0
    assert call(capacity=alloc + 1) != 0
    assert call(alloc=2 * arr.size - 1, capacity=16) != 0
    assert (out.view(np.uint8) == 0).all()
    assert call() == 0, dev.dev_error()


# ---------------------------------------------------------------- the product path


def test_decoder_batches_past_the_full_grid(dev, gpu_decoder_factory, checker_libs):
    """Decoder(gpu_resolve=1) with one batch of more than 32 * SM count buffers followed by its two halves
    (run_buffers halves the last batch of a call), a chain at the first seam: the host resolve's output."""
    max_b = WARPS_PER_SM * dev.sm_count + 64
    n_bytes = 2 * max_b * BUF + 12345
    data = synth.tile_to(C.modes1(), n_bytes)
    chain = S.chain("chain_df4")
    at = (max_b - 5) * BUF
    data[at: at + chain.size] = chain
    digests = []
    for gpu in (0, 1):
        dec = gpu_decoder_factory(gpu_resolve=gpu, max_batch_bytes=max_b * BUF)
        out = dec.set_output_array(1_300_000)
        dec.reset(); dec.rearm_output(); dec.process(data); dec.finish()
        n = dec.output_count()
        assert n < len(out)
        a = np.frombuffer(out, dtype=np.uint8, count=n * 200)
        digests.append((n, hashlib.sha256(a.tobytes()).hexdigest(), dec.stats()))
        dec.set_output_array(0)
        dec.close()
    assert digests[0][0] > 900_000
    assert digests[0] == digests[1]


# ---------------------------------------------------------------- the hex door and the device resolve

HEX_ADDRS = [0x3C6DD1, 0x4B1A22, 0xA0B0C1, 0x71C0DE, 0x50F00D]
ME = bytes([0x58, 0xC3, 0x82, 0xD6, 0x90, 0xC8, 0xAC])
IIDS = [7, 11, 13, 14, 19, 21, 22, 25, 26, 28]     # below 80, three or more bits set (streams._IIDS)


def hex_frames():
    """Clean DF17s announcing HEX_ADDRS: what the hex door writes into the address cache."""
    return [synth.make_frame(17, 5, a.to_bytes(3, "big") + ME) for a in HEX_ADDRS]


def _reply(k, x):
    """The k-th reply from address x: DF4 / DF5 / DF20 / DF21 with x in the address/parity field, or a
    DF11 whose parity carries an interrogator id (validated through its address, dump1090.c:1204-1209)."""
    kind = k % 5
    if kind == 0:
        return synth.make_frame(4, 0, bytes([0x01, 0x85, 0x10 + (k & 7)]), icao_for_ap=x)
    if kind == 1:
        return synth.make_frame(5, 0, bytes([0x02, 0x0C, 0x30 + (k & 7)]), icao_for_ap=x)
    if kind == 2:
        return synth.make_frame(20, 0, bytes([0x10, 0x00, 0x1C, 0x38]) + ME[:6], icao_for_ap=x)
    if kind == 3:
        return synth.make_frame(21, 0, bytes([0x20, 0x0B, 0x55, 0x9C]) + ME[1:7], icao_for_ap=x)
    f = synth.make_frame(11, 5, x.to_bytes(3, "big"))
    return f[:4] + (int.from_bytes(f[4:], "big") ^ IIDS[k % len(IIDS)]).to_bytes(3, "big")


HEX_SAMPLES = 4 * NS + 50000


def hex_stream(rate):
    """Replies from HEX_ADDRS only (nothing in the stream announces them) every 1500 samples, at 2 MHz or
    2.4 MS/s."""
    frames = [(3000 + 1500 * k, _reply(k, HEX_ADDRS[k % len(HEX_ADDRS)]), 80.0, 0.3 + 0.1 * k, 0.0)
              for k in range((HEX_SAMPLES - 4000) // 1500)]
    return synth.synth_stream_at(HEX_SAMPLES * rate // 2_000_000, frames, sigma=1.0, seed=9, sample_rate=rate)


def _from_hex_addrs(m):
    if m.msgtype == 11:
        return m.iid != 0 and (m.aa1 << 16 | m.aa2 << 8 | m.aa3) in HEX_ADDRS
    return m.msgtype in AP_FORMATS and m.crcok and (m.aa1 << 16 | m.aa2 << 8 | m.aa3) in HEX_ADDRS


def run_sequence(factory, gpu, rate, seq):
    """seq: "first" (reset, hex door, process, finish), "whole" / "partial" (process up to a buffer seam /
    into a buffer, hex door, process the rest, finish), "none" (no hex-door call).  Returns (hex-door
    messages, stream messages, statistics)."""
    data = hex_stream(rate)
    dec = factory(gpu_resolve=gpu, input_rate=rate)
    dec.reset()
    split = {"first": 0, "whole": 2 * BUF, "partial": 2 * BUF + 30000, "none": 0}[seq] * rate // 2_000_000
    split -= split % 2
    dec.process(data[:split])
    hexed = dec.decode_frames(hex_frames()) if seq != "none" else []
    dec.process(data[split:])
    dec.finish()
    out = ([C.msg_fields(m) for m in hexed], dec.take_messages(), dec.stats())
    dec.close()
    return out


@pytest.mark.parametrize("seq", ["first", "whole", "partial"])
@pytest.mark.parametrize("rate", [2_000_000, 2_400_000])
def test_hex_door_writes_reach_device_resolve(seq, rate, gpu_decoder_factory, checker_libs):
    """The hex door writes the context's address cache; the next batches see its writes whichever side
    resolves them.  The replies are delivered only because of the hex-door call."""
    runs = [run_sequence(gpu_decoder_factory, gpu, rate, seq) for gpu in (0, 1)]
    hexed, msgs, stats = zip(*runs)
    assert hexed[0] == hexed[1] and all(h["crcok"] for h in hexed[1])
    for got in msgs:
        assert sum(_from_hex_addrs(m) for m in got) > 20
    assert [m.raw_line() for m in msgs[1]] == [m.raw_line() for m in msgs[0]]
    assert [C.msg_fields(m, with_pos=True) for m in msgs[1]] == [C.msg_fields(m, with_pos=True) for m in msgs[0]]
    assert stats[1] == stats[0]
    for gpu in (0, 1):
        _, control, _ = run_sequence(gpu_decoder_factory, gpu, rate, "none")
        assert not any(_from_hex_addrs(m) for m in control)


def test_hex_door_then_device_resolve_equals_oracle(gpu_decoder_factory, checker_libs):
    """Reset, hex door, stream: the oracle on the stream behind one buffer that holds the announcing frames
    as clean I/Q (its messages dropped, positions shifted by one buffer)."""
    _, got, _ = run_sequence(gpu_decoder_factory, 1, 2_000_000, "first")
    pre = synth.synth_stream(NS, [(1000 + 2000 * i, f, 80.0, 0.5, 0.0) for i, f in enumerate(hex_frames())], sigma=1.0,
                             seed=4)
    pre[-api.CARRY_BYTES:] = 127                   # the carry into the stream's first buffer: no signal, as after a reset
    exp, _ = C.oracle_decode(np.concatenate([pre, hex_stream(2_000_000)]), cap=100000)
    pre_msgs = [m for m in exp if m.sample_pos < NS - 238]
    assert sorted((m.aa1 << 16 | m.aa2 << 8 | m.aa3) for m in pre_msgs if m.msgtype == 17) == sorted(HEX_ADDRS)
    exp = [m for m in exp if m.sample_pos >= NS - 238]
    want = [dict(C.msg_fields(m, with_pos=True), sample_pos=int(m.sample_pos) - NS) for m in exp]
    assert [C.msg_fields(m, with_pos=True) for m in got] == want
    assert sum(_from_hex_addrs(m) for m in got) > 20
