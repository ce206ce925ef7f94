"""The receiver pool (modes_pool_*) at the size it runs at: every receiver of a 256-receiver pool, the
host resolve cut into several blocks, both input rates and every pass.

Each receiver's stream is its own: every input buffer (receiver r, its k-th call) carries a clean DF17
frame of address 0x800000 | r << 8 | k in front of background that no other receiver holds at the same
time, so a receiver handed another's buffer, messages or receiver id fails the direct check (`_planted`)
without trusting any reference.

The CPU tests drive the host half (modes_pool_resolve) with the oracle's candidate records over the
pool's pad/data layout, with call sizes that move the block count and the cut points from call to call
(blocks: min(MODES_POOL_THREADS, ceil(n / 16)) over a call's n pairs).  They check each receiver against
the oracle, the sink's global order, the caller's output array (also cut by its capacity inside the third
block), and that the thread count changes no byte.  The GPU tests run ReceiverPool(256, max_batch=256)
with a third of the receivers at 2.4 MS/s, and a 520-receiver pool whose strided weak-preamble scan has
more tiles than weak_order_kernel takes in one round."""
import ctypes
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest

import checker as C
import pool_rate_model as PM
import resample_model as RM
import streams as S
from dump1090_b200 import api, synth

ROOT = C.ROOT
BUF = api.BUFFER_BYTES
B = api.BUFFER_SAMPLES
CARRY = api.CARRY_BYTES
R2, R24 = 2_000_000, 2_400_000
PLANT_ME = bytes([0x58, 0xC3, 0x82, 0xD6, 0x90, 0xC8, 0xAC])     # an airborne-position ME field
FLAG_SETS = [dict(), dict(aggressive=1), dict(fix=0), dict(check_crc=0)]   # test_pool's four


def _kid(k):
    return "-".join(f"{a}{b}" for a, b in k.items()) or "default"


def _cfg(kw):
    return dict(fix_errors=kw.get("fix", 1), aggressive=kw.get("aggressive", 0), check_crc=kw.get("check_crc", 1))


def _blocks(n, threads):
    """pool_resolve's blocks of a call of n pairs: [(i0, i1)]."""
    nb = max(1, min(threads, (n + 15) // 16))
    return [(n * b // nb, n * (b + 1) // nb) for b in range(nb)]


def _threads():
    """MODES_POOL_THREADS as the library reads it."""
    try:
        v = int(os.environ.get("MODES_POOL_THREADS", "4"))
    except ValueError:
        v = 0
    return max(1, min(64, v))


# ---------------------------------------------------------------- streams


def _banks(n_rt=24, n_fleet=8, with_24=False):
    """Background buffers: dense random traffic and a weak-rich 8 dB fleet at 2 MHz, and (with_24) a
    fleet sampled at 2.4 MS/s; one buffer per row."""
    rt = synth.random_traffic(n_rt * B, 120 * n_rt, seed=4401)
    fl = synth.fleet_at(8, n_fleet * B // 400 + 8, 4402)[0][: n_fleet * BUF]
    banks = {R2: np.concatenate([rt, fl]).reshape(-1, BUF)}
    if with_24:
        f24 = synth.fleet_at_rate(12, 16 * B * 5 // 6 // 400 + 8, 4403)[0]
        banks[R24] = np.concatenate([f24[: 16 * BUF], rt[: 8 * BUF]]).reshape(-1, BUF)
    return banks


def planted_frame(r, k):
    return synth.make_frame(17, 5, (0x800000 | r << 8 | k).to_bytes(3, "big") + PLANT_ME)


def _stream(r, n_buf, rate, banks, chain=False):
    """Receiver r's input stream of n_buf buffers and its planted frames [(2 MHz position, frame)].
    Background (r, k) is bank buffer (r + 5k) mod len(bank) rotated by 62 (16 r + k) bytes, an amount
    no other (receiver, buffer) uses; chain receivers run an address chain (streams.address_chain)
    through their own cache instead.  Each buffer then gets a stretch of fresh noise with one clean
    DF17 frame naming (r, k), away from the chains' frames and from 2 MHz buffer seams."""
    if chain:
        s = S.address_chain(n_buf, S.CHAIN_KINDS[r % len(S.CHAIN_KINDS)], seed=r + 1)
    else:
        bank = banks[rate]
        s = np.concatenate([np.roll(bank[(r + 5 * k) % len(bank)], 62 * (16 * r + k)) for k in range(n_buf)])
    plants = []
    seg_in = 720 if rate == R24 else 600                       # input samples: 600 at 2 MHz
    for k in range(n_buf):
        st = (k * B + 40000 + (r * 7919 + k * 104729) % 80000) // 6 * 6
        if ((st * R2 // rate + 300) + 238) % B > B - 400:      # keep the preamble off a 2 MHz seam
            st -= 1200
        f = planted_frame(r, k)
        seg = synth.synth_stream_at(seg_in, [(300, f, 90.0, 0.37 * k + 0.11 * r, 0.0)], sigma=1.5,
                                    seed=100000 + 16 * r + k, sample_rate=rate)
        s[2 * st: 2 * st + seg.size] = seg
        plants.append((st * R2 // rate + 300, f))
    return s, plants


def _planted(got, plants, n_decoded, every):
    """The planted frames a receiver delivered are exactly its own, in stream order, one for each
    planted frame of the buffers it decoded.  every: the frames planted in any receiver."""
    want = [f for p, f in plants if (p + 238) // B < n_decoded]
    mine = [bytes(m.msg) for m in got if bytes(m.msg) in every]
    assert mine == want, (len(mine), len(want))
    return len(want)


def _buffer_of(m):
    return (int(m.sample_pos) + 238) // B


class _Recorder:
    """A sink for the pool that keeps the global (receiver, message) sequence and the pool's own
    per-receiver lists (what ReceiverPool.take returns)."""

    def __init__(self, pool):
        self.pool, self.seq = pool, []
        self.fn = api.POOL_SINK_FN(self._on)
        pool._fn = self.fn                                       # what ingest / collect / resolve hand the library

    def _on(self, _user, receiver, mm):
        m = mm.contents.copy()
        self.seq.append((int(receiver), m))
        self.pool.messages[receiver].append(m)

    def since(self, at):
        return self.seq[at:]


# ---------------------------------------------------------------- CPU: the multi-block host resolve


CPU_RX = 66
CPU_SIZES = (1, 15, 16, 17, 31, 32, 33, 47, 48, 49, 63, 64, 65, CPU_RX)


def _cpu_plan(seed=5):
    """Calls of the sizes above; each names the receivers with the fewest buffers so far, in shuffled order."""
    rng = np.random.default_rng(seed)
    done = [0] * CPU_RX
    calls = []
    for n in CPU_SIZES:
        ids = sorted(range(CPU_RX), key=lambda r: (done[r], rng.random()))[:n]
        rng.shuffle(ids)
        calls.append([(r, done[r]) for r in ids])
        for r in ids:
            done[r] += 1
    return calls, done


@pytest.fixture(scope="module")
def cpu_world():
    calls, n_buf = _cpu_plan()
    banks = _banks()
    streams, plants = [], []
    for r in range(CPU_RX):
        s, p = _stream(r, n_buf[r], R2, banks, chain=r % 11 == 4)
        streams.append(s)
        plants.append(p)
    every = {f for p in plants for _, f in p}
    return dict(calls=calls, n_buf=n_buf, streams=streams, plants=plants, every=every, records={})


def _records(world, fix, aggressive):
    """Per call: the oracle's candidate records and tile table over the pool's layout of the call."""
    key = (fix, aggressive)
    if key not in world["records"]:
        out = []
        for call in world["calls"]:
            batch = np.full(2 * len(call) * BUF, 127, dtype=np.uint8)
            for i, (r, k) in enumerate(call):
                s = world["streams"][r]
                if k:                                          # the pad buffer's tail = this receiver's carry
                    batch[(2 * i + 1) * BUF - CARRY: (2 * i + 1) * BUF] = s[k * BUF - CARRY: k * BUF]
                batch[(2 * i + 1) * BUF: (2 * i + 2) * BUF] = s[k * BUF: (k + 1) * BUF]
            recs = C.oracle_scan_candidates(batch, fix=fix, aggressive=aggressive, cap=400_000)
            cands = np.frombuffer(b"".join(bytes(c) for c in recs), dtype=api.CANDIDATE_DTYPE) if recs \
                else np.zeros(0, api.CANDIDATE_DTYPE)
            n_tiles = api.tiles_for(2 * len(call))
            cnt = np.bincount((cands["t"] + 2) // api.TILE_SAMPLES, minlength=n_tiles).astype(np.uint32)
            tiles = np.zeros(n_tiles, dtype=api.TILE_DTYPE)
            tiles["count"] = cnt
            tiles["offset"] = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.uint32)
            out.append((np.ascontiguousarray(cands), tiles))
        world["records"][key] = out
    return world["records"][key]


def _set_output(pool, n, cap):
    """A caller-owned output array of n entries filled with 0xA5, of which the pool may use cap."""
    out = (api.Message * n)()
    ctypes.memset(ctypes.addressof(out), 0xA5, ctypes.sizeof(out))
    out_rx = np.full(n, 0xA5A5A5A5, dtype=np.uint32)
    assert api.lib().modes_pool_set_output(pool._h, ctypes.addressof(out), out_rx.ctypes.data, cap) == 0
    return out, out_rx


def _raw(out, n):
    return ctypes.string_at(ctypes.addressof(out), n * ctypes.sizeof(api.Message))


def _run_cpu(calls, records, cfg, cap_of=None):
    """The schedule through modes_pool_resolve, each call with a fresh output array of room for the call
    (or cap_of(call index) entries): per call (sink sequence, output bytes, out_rx, output_count)."""
    pool = api.ReceiverPool(CPU_RX, **cfg)
    rec = _Recorder(pool)
    per_call = []
    for ci, (call, (cands, tiles)) in enumerate(zip(calls, records)):
        room = 3 * cands.size + 64
        cap = room if cap_of is None else cap_of(ci)
        out, out_rx = _set_output(pool, room, cap)
        at = len(rec.seq)
        pool.resolve([r for r, _ in call], cands, tiles)
        per_call.append((rec.since(at), out, out_rx, pool.output_count()))
    return pool, per_call


def _expect_cpu(world, kw):
    """Per receiver: the oracle's messages (and statistics) of its stream, split by buffer."""
    want = []
    for r, s in enumerate(world["streams"]):
        msgs, stats = C.oracle_decode(s, drop_eof=1, **kw)
        by_buf = [[] for _ in range(world["n_buf"][r])]
        for m in msgs:
            by_buf[_buffer_of(m)].append(m)
        want.append((msgs, stats, by_buf))
    return want


@pytest.mark.parametrize("kw", FLAG_SETS, ids=_kid)
def test_multi_block_resolve_equals_oracle(kw, cpu_world, checker_libs):
    world = cpu_world
    calls = world["calls"]
    cfg = _cfg(kw)
    records = _records(world, cfg["fix_errors"], cfg["aggressive"])
    want = _expect_cpu(world, kw)
    threads = _threads()
    pool, per_call = _run_cpu(calls, records, cfg)
    shapes = set()
    for ci, (call, (seq, out, out_rx, count)) in enumerate(zip(calls, per_call)):
        n = len(call)
        shapes.add((n, len(_blocks(n, threads))))
        # the sink: the call's receivers in the listed order, each with the oracle's messages of its buffer
        expect = [(r, m.hexline()) for r, k in call for m in want[r][2][k]]
        assert [(r, m.raw_line()) for r, m in seq] == expect, f"call {ci}: {n} receivers"
        # the output array: the same sequence, receiver by receiver, and nothing past it
        assert count == len(seq)
        assert _raw(out, count) == b"".join(bytes(m) for _, m in seq), f"call {ci}"
        assert list(out_rx[:count]) == [r for r, _ in seq], f"call {ci}"
        assert (out_rx[count:] == 0xA5A5A5A5).all() and set(_raw(out, len(out))[count * ctypes.sizeof(api.Message):]) <= {0xA5}
    if threads == 4:
        assert {nb for _, nb in shapes} == {1, 2, 3, 4}
    covered = 0
    for r in range(CPU_RX):
        msgs, stats, _ = want[r]
        got = pool.take(r)
        assert pool.buffers(r) == world["n_buf"][r], r
        assert [m.raw_line() for m in got] == [m.hexline() for m in msgs], f"receiver {r}"
        assert [C.msg_fields(m, with_pos=True) for m in got] == [C.msg_fields(m, with_pos=True) for m in msgs], r
        assert list(pool.stats(r).values()) == stats, f"receiver {r}"
        covered += _planted(got, world["plants"][r], world["n_buf"][r], world["every"])
    assert covered == sum(world["n_buf"])
    pool.close()
    # the output array cut by its capacity inside the third block: the full run's prefix, its receivers,
    # and the count running on past the capacity
    cuts = {}
    for ci, (call, (seq, _, _, _)) in enumerate(zip(calls, per_call)):
        bl = _blocks(len(call), threads)
        if len(bl) < 3:
            continue
        pos = {r: i for i, (r, _) in enumerate(call)}
        before = sum(1 for r, _ in seq if pos[r] < bl[2][0])
        third = sum(1 for r, _ in seq if bl[2][0] <= pos[r] < bl[2][1])
        assert third > 1, ci
        cuts[ci] = before + third // 2
    assert len(cuts) >= 8 or threads < 3
    cut_pool, cut_calls = _run_cpu(calls, records, cfg, cap_of=lambda ci: cuts.get(ci, 0))
    cut_pool.close()
    for ci, cap in cuts.items():
        seq, out, out_rx, count = per_call[ci]
        _, cout, cout_rx, ccount = cut_calls[ci]
        assert ccount == count > cap, ci
        assert _raw(cout, cap) == _raw(out, cap), ci
        assert np.array_equal(cout_rx[:cap], out_rx[:cap]), ci
        assert (cout_rx[cap:] == 0xA5A5A5A5).all() and set(_raw(cout, len(cout))[cap * ctypes.sizeof(api.Message):]) <= {0xA5}, ci


def _digest(calls, records, cfg):
    """One hash over everything the schedule delivers: the sink sequence, the output arrays and their
    receivers, and every receiver's buffers and statistics."""
    pool, per_call = _run_cpu(calls, records, cfg)
    h = hashlib.sha256()
    for seq, out, out_rx, count in per_call:
        h.update(count.to_bytes(8, "little"))
        for r, m in seq:
            h.update(r.to_bytes(4, "little") + bytes(m))
        h.update(_raw(out, count) + out_rx[:count].tobytes())
    for r in range(CPU_RX):
        h.update(repr((pool.buffers(r), pool.stats(r))).encode())
    pool.close()
    return h.hexdigest()


def _digest_main(path):
    """Entry of the thread-count runs: the schedule in `path` through a process of its own."""
    z = np.load(path)
    n = int(z["n_calls"])
    calls = [[(int(r), 0) for r in z[f"ids{i}"]] for i in range(n)]
    records = [(z[f"c{i}"], z[f"t{i}"]) for i in range(n)]
    print("DIGEST", _digest(calls, records, {}))


def test_thread_count_changes_nothing(cpu_world, checker_libs, tmp_path):
    """MODES_POOL_THREADS is read once per process: the same schedule in processes with 1 to 64 host
    threads (one to five blocks per call) delivers the same bytes."""
    world = cpu_world
    records = _records(world, 1, 0)
    path = tmp_path / "schedule.npz"
    arrays = {"n_calls": np.array(len(world["calls"]))}
    for i, (call, (cands, tiles)) in enumerate(zip(world["calls"], records)):
        arrays[f"ids{i}"] = np.array([r for r, _ in call], np.uint32)
        arrays[f"c{i}"], arrays[f"t{i}"] = cands, tiles
    np.savez(path, **arrays)
    here = _digest(world["calls"], records, {})
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([str(ROOT), str(ROOT / "tests")]))
    code = f"import test_pool_scale as T; T._digest_main({str(path)!r})"
    for threads in (1, 2, 3, 4, 5, 64):
        env["MODES_POOL_THREADS"] = str(threads)
        run = subprocess.run([sys.executable, "-c", code], env=env, cwd=str(ROOT), capture_output=True, text=True, timeout=300)
        assert run.returncode == 0, run.stderr[-3000:]
        assert f"DIGEST {here}" in run.stdout.splitlines(), (threads, run.stdout[-500:])


# ---------------------------------------------------------------- GPU: the pool at the benchmark's size


GPU_RX = 256
PAIR_TARGETS = ((16, 1), (17, 2), (32, 1), (33, 3), (64, 1), (65, 2))   # (pairs, named receivers that complete nothing)


def _completes(c):
    """Whether a 2.4 MS/s receiver's own call c completes a 2 MHz buffer (pool_rate_model)."""
    return PM.ready_buffers((c + 1) * B) > PM.ready_buffers(c * B)


def _gpu_plan(n_rx=GPU_RX, seed=21):
    """rates, calls per receiver, and the calls: [(receiver, its own call index, 2 MHz buffer it decodes
    or None)].  First calls whose pair counts sit at the block thresholds while the named count does
    not; then two calls naming about half the pool (2.4 MS/s receivers start at different calls, so
    their resampling phases differ); then every receiver at once; then the rest of each receiver's calls."""
    rng = np.random.default_rng(seed)
    rates = [R24 if r % 3 == 1 else R2 for r in range(n_rx)]
    quota = [6 + (r // 3) % 3 for r in range(n_rx)]
    done = [0] * n_rx
    calls = []

    def decodes(r):
        if rates[r] == R2:
            return done[r]
        return PM.ready_buffers(done[r] * B) if _completes(done[r]) else None

    def add(ids):
        ids = list(ids)
        rng.shuffle(ids)
        calls.append([(int(r), done[r], decodes(r)) for r in ids])
        for r in ids:
            done[r] += 1

    def spare(r, keep):
        return done[r] < quota[r] - keep

    for pairs, extra in PAIR_TARGETS:
        cand = [r for r in rng.permutation(n_rx) if spare(r, 1)]
        idle = [r for r in cand if decodes(r) is None][:extra]
        busy = [r for r in cand if decodes(r) is not None][:pairs]
        assert len(idle) == extra and len(busy) == pairs
        add(idle + busy)
    for _ in range(2):
        add([r for r in range(n_rx) if spare(r, 1) and rng.random() < 0.5])
    add(range(n_rx))
    while any(spare(r, 0) for r in range(n_rx)):
        ids = [r for r in range(n_rx) if spare(r, 0) and rng.random() < 0.8]
        if ids:
            add(ids)
    return rates, quota, calls


def _decoded_buffers(rate, n_calls):
    return PM.ready_buffers(n_calls * B) if rate == R24 else n_calls


@pytest.fixture(scope="module")
def gpu_world():
    rates, quota, calls = _gpu_plan()
    banks = _banks(with_24=True)
    streams, plants, decoded = [], [], []
    for r in range(GPU_RX):
        s, p = _stream(r, quota[r], rates[r], banks, chain=r % 16 == 5 and rates[r] == R2)
        streams.append(s)
        plants.append(p)
        k = _decoded_buffers(rates[r], quota[r])
        decoded.append(RM.resample_range(s, 0, k * B) if rates[r] == R24 else s)     # the 2 MHz bytes decoded
    every = {f for p in plants for _, f in p}
    return dict(rates=rates, quota=quota, calls=calls, streams=streams, plants=plants, decoded=decoded, every=every)


def _call_buffers(world, call, strided):
    """The call's buffers: one host block at a constant distance (the strided upload), or the same
    block in reverse, so that the addresses fall and every buffer is copied on its own."""
    return _upload_views([world["streams"][r][c * BUF: (c + 1) * BUF] for r, c, _ in call], strided)


def _upload_views(bufs, strided):
    block = np.stack(bufs if strided else bufs[::-1])
    return [block[i] for i in range(len(bufs))] if strided else [block[len(bufs) - 1 - i] for i in range(len(bufs))]


def _check_call(call, seq, what):
    """One call's sink sequence: receivers in the listed order, each with messages of the buffer it
    decodes in this call only, and none from a receiver that completed no buffer."""
    pos = {r: i for i, (r, _, _) in enumerate(call)}
    want_buf = {r: m for r, _, m in call}
    last = -1
    for r, m in seq:
        assert r in pos and want_buf[r] is not None, (what, r)
        assert pos[r] >= last, (what, "sink order")
        last = pos[r]
        assert _buffer_of(m) == want_buf[r], (what, r, _buffer_of(m), want_buf[r])


def _drive(pool, world, mode):
    """The whole schedule: "ingest" (one call at a time) or "pipelined" (submit / collect with two
    batches in flight, many receivers in both).  Upload shapes alternate from call to call.  Returns the
    pair count of every call, as the receivers' decoded buffers moved."""
    rec = _Recorder(pool)
    calls = world["calls"]
    pairs = []
    if mode == "ingest":
        for ci, call in enumerate(calls):
            before = [pool.buffers(r) for r, _, _ in call]
            at = len(rec.seq)
            pool.ingest([r for r, _, _ in call], _call_buffers(world, call, ci % 2 == 0))
            _check_call(call, rec.since(at), (mode, ci))
            pairs.append(sum(pool.buffers(r) - b for (r, _, _), b in zip(call, before)))
        return pairs
    pending = []
    for ci, call in enumerate(calls):
        pool.submit([r for r, _, _ in call], _call_buffers(world, call, ci % 2 == 1))
        pending.append(ci)
        if len(pending) == 2:
            at = len(rec.seq)
            pool.collect()
            done = pending.pop(0)
            _check_call(calls[done], rec.since(at), (mode, done))
    while pending:
        at = len(rec.seq)
        pool.collect()
        done = pending.pop(0)
        _check_call(calls[done], rec.since(at), (mode, done))
    return None


def _references(world, factory, **cfg):
    """Per receiver, the single-stream decoder at its rate fed its whole input without finish(): messages,
    statistics, level records, recovery and weak-recovery statistics.  One decoder per rate, reset
    between receivers."""
    dec = {R2: factory(input_rate=R2, **cfg), R24: factory(input_rate=R24, **cfg)}
    out = []
    for r, s in enumerate(world["streams"]):
        d = dec[world["rates"][r]]
        d.reset()
        d.take_levels()
        d.process(s)
        out.append((d.take_messages(), d.stats(), d.take_levels(), d.recovery_stats(), d.weak_recovery_stats()))
    return out


def _same(got, want, what):
    assert len(got) == len(want), (what, len(got), len(want))
    for k, (g, w) in enumerate(zip(got, want)):
        assert bytes(g) == bytes(w), (what, k, g.raw_line(), w.raw_line())


def _gpu_pool(world, **kw):
    pool = api.ReceiverPool(GPU_RX, max_batch=GPU_RX, **kw)
    for r, hz in enumerate(world["rates"]):
        pool.set_input_rate(r, hz)
    return pool


def test_gpu_plan_reaches_the_thresholds():
    """The schedule (pure arithmetic, checked without a device): pair counts at 16/17/32/33/64/65 with more
    receivers named, a call of every receiver, 6-8 calls each, and 2.4 MS/s receivers that start at
    different calls."""
    rates, quota, calls = _gpu_plan()
    pairs = [sum(m is not None for _, _, m in call) for call in calls]
    named = [len(call) for call in calls]
    assert pairs[: len(PAIR_TARGETS)] == [p for p, _ in PAIR_TARGETS]
    assert [n - p for n, p in zip(named, pairs)][: len(PAIR_TARGETS)] == [e for _, e in PAIR_TARGETS]
    assert len(_blocks(17, 4)) != len(_blocks(16, 4)) and len(_blocks(33, 4)) != len(_blocks(32, 4))
    assert GPU_RX in named and sum(r == R24 for r in rates) * 3 >= GPU_RX - 2
    per_rx = [0] * GPU_RX
    first = {}
    for ci, call in enumerate(calls):
        for r, c, _ in call:
            assert c == per_rx[r]
            per_rx[r] += 1
            first.setdefault(r, ci)
    assert per_rx == quota and set(quota) == {6, 7, 8}
    assert len({first[r] for r in range(GPU_RX) if rates[r] == R24}) >= 4


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(), dict(check_crc=0, aggressive=1)], ids=_kid)
def test_full_pool_equals_oracle_and_single_stream(kw, gpu_world, gpu_decoder_factory, checker_libs):
    world = gpu_world
    cfg = _cfg(kw)
    refs = _references(world, gpu_decoder_factory, **cfg)
    oracle = [C.oracle_decode(d, drop_eof=1, **kw) for d in world["decoded"]]
    want_pairs = [sum(m is not None for _, _, m in call) for call in world["calls"]]
    n_msgs = 0
    for mode in ("ingest", "pipelined"):
        with _gpu_pool(world, **cfg) as pool:
            pairs = _drive(pool, world, mode)
            if pairs is not None:
                assert pairs == want_pairs
                print(f"\npool scale: calls {len(pairs)}, named {[len(c) for c in world['calls']]}, pairs {pairs}, "
                      f"blocks {[len(_blocks(p, 4)) for p in pairs]}")
            for r in range(GPU_RX):
                rate = world["rates"][r]
                k = pool.buffers(r)
                assert k == _decoded_buffers(rate, world["quota"][r]), (mode, r)
                got = pool.take(r)
                msgs, stats = oracle[r]
                assert [m.raw_line() for m in got] == [m.hexline() for m in msgs], (mode, r)
                assert [C.msg_fields(m, with_pos=True) for m in got] == [C.msg_fields(m, with_pos=True) for m in msgs], (mode, r)
                assert list(pool.stats(r).values()) == stats, (mode, r)
                _same(got, refs[r][0], (mode, r))
                assert pool.stats(r) == refs[r][1], (mode, r)
                _planted(got, world["plants"][r], k, world["every"])
                n_msgs += len(got)
    print(f"pool scale {_kid(kw)}: {n_msgs} messages compared over both drives")


@pytest.mark.gpu
@pytest.mark.parametrize("sw", [dict(signal=True), dict(arrival=True, signal=True), dict(levels=True), dict(recover=True),
                                dict(recover=True, weak_preambles=True)], ids=["signal", "arrival", "levels", "recover", "weak"])
def test_full_pool_every_switch_equals_single_stream(sw, gpu_world, gpu_decoder_factory):
    world = gpu_world
    refs = _references(world, gpu_decoder_factory, **sw)
    mode = "pipelined" if sw.get("arrival") or sw.get("recover") and not sw.get("weak_preambles") else "ingest"
    seen = dict(messages=0, signal=0, arrival=0, levels=0, recovered=0, weak=0)
    with _gpu_pool(world, **sw) as pool:
        _drive(pool, world, mode)
        for r in range(GPU_RX):
            msgs, stats, levels, rstats, wstats = refs[r]
            got = pool.take(r)
            _same(got, msgs, (sw, r))
            assert pool.stats(r) == stats, (sw, r)
            _planted(got, world["plants"][r], pool.buffers(r), world["every"])
            lv = pool.take_levels(r)
            assert np.array_equal(lv, levels), (sw, r)
            if sw.get("levels"):
                assert list(lv["buffer"]) == list(range(pool.buffers(r))), r
            assert pool.recovery_stats(r) == rstats and pool.weak_recovery_stats(r) == wstats, (sw, r)
            seen["messages"] += len(got)
            seen["signal"] += sum(m.signal > 0 for m in got)
            seen["arrival"] += sum(m.arrival != 0 for m in got)
            seen["levels"] += lv.size
            seen["recovered"] += sum(m.recovered == 1 for m in got)
            seen["weak"] += sum(m.recovered == 2 for m in got)
    print(f"\npool scale {'+'.join(sw)} ({mode}): {seen}")
    if sw.get("signal"):
        assert seen["signal"] > 1000
    if sw.get("arrival"):
        assert seen["arrival"] > 1000
    if sw.get("levels"):
        assert seen["levels"] == sum(_decoded_buffers(world["rates"][r], world["quota"][r]) for r in range(GPU_RX))
    if sw.get("recover"):
        assert seen["recovered"] > 10
    if sw.get("weak_preambles"):
        assert seen["weak"] > 10


WIDE_RX = 520
WEAK_TILE_SAMPLES = 4096                # kWeakTileSamples
ORDER_ROUND_TILES = 16 * 1024           # weak_order_kernel: 16 tiles per thread, 1024 threads


@pytest.mark.gpu
def test_weak_order_rounds_in_the_pool(gpu_decoder_factory):
    """520 receivers in one call: the strided weak-preamble scan covers 520 data buffers, 32 tiles each,
    past the 16 384 tiles of one weak_order_kernel round.  Every receiver equals the single-stream
    decoder, and weak recoveries land on both sides of the 512th data buffer."""
    n_calls = 2
    tiles = WIDE_RX * (B // WEAK_TILE_SAMPLES)
    assert tiles > ORDER_ROUND_TILES and (512 * (B // WEAK_TILE_SAMPLES)) == ORDER_ROUND_TILES
    banks = {R2: _banks(n_rt=2, n_fleet=16)[R2][2:]}          # the weak-rich fleet: weak frames of known aircraft
    streams, plants = [], []
    for r in range(WIDE_RX):
        s, p = _stream(r, n_calls, R2, banks)
        streams.append(s)
        plants.append(p)
    every = {f for p in plants for _, f in p}
    rng = np.random.default_rng(31)
    orders = [[int(r) for r in rng.permutation(WIDE_RX)] for _ in range(n_calls)]
    kw = dict(recover=True, weak_preambles=True)
    with api.ReceiverPool(WIDE_RX, max_batch=WIDE_RX, **kw) as pool:
        for k, ids in enumerate(orders):
            pool.ingest(ids, _upload_views([streams[r][k * BUF: (k + 1) * BUF] for r in ids], k == 0))
        dec = gpu_decoder_factory(**kw)
        weak_at = [[0, 0] for _ in range(n_calls)]              # weak recoveries of pairs 480-511 and 512-519
        n_msgs = n_weak = 0
        for r in range(WIDE_RX):
            dec.reset()
            dec.process(streams[r])
            got = pool.take(r)
            _same(got, dec.take_messages(), r)
            assert pool.buffers(r) == n_calls
            assert pool.stats(r) == dec.stats() and pool.recovery_stats(r) == dec.recovery_stats(), r
            assert pool.weak_recovery_stats(r) == dec.weak_recovery_stats(), r
            _planted(got, plants[r], n_calls, every)
            n_msgs += len(got)
            for m in got:
                if m.recovered == 2:
                    n_weak += 1
                    k = _buffer_of(m)
                    i = orders[k].index(r)
                    if 480 <= i < 512:
                        weak_at[k][0] += 1
                    elif i >= 512:
                        weak_at[k][1] += 1
    print(f"\npool scale: {WIDE_RX} receivers, {tiles} strided weak tiles per call, {n_msgs} messages, "
          f"{n_weak} weak recoveries, by call (pairs 480-511, 512-519): {weak_at}")
    assert all(a > 0 and b > 0 for a, b in weak_at), weak_at
