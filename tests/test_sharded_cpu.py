"""CPU (-m "not gpu"): the multi-GPU host logic over gloo, world size 2.

The device half is replaced by the checker's candidate records (oracle_scan_candidates); what is
under test is the product's sharding plan, the record gather and the stream-ordered resolve on
rank 0 (dump1090_b200/sharded.py + modes_resolver_*)."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import checker as C
import streams as S
from dump1090_b200 import api, sharded, synth


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, nsamples, seed, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        data = synth.random_traffic(nsamples, nsamples // 700, seed)
        total_buffers = data.size // api.BUFFER_BYTES + 1
        plan = sharded.shard_plan(total_buffers, world)
        first, count = plan[rank]
        # stand-in for the device half: this rank's candidates, shard-local positions
        cands = C.oracle_scan_candidates(data)
        arr = np.frombuffer(b"".join(bytes(c) for c in cands), dtype=api.CANDIDATE_DTYPE).copy()
        mine = arr[((arr["t"] >> 17) >= first) & ((arr["t"] >> 17) < first + count)].copy()
        mine["t"] -= first << 17
        # two tiles per shard to exercise the tile walk
        half = mine.size // 2
        tiles = np.array([(0, half), (half, mine.size - half)], dtype=api.TILE_DTYPE)
        c_t = torch.from_numpy(mine.view(np.uint8).reshape(-1).copy()) if mine.size else torch.zeros(0, dtype=torch.uint8)
        t_t = torch.from_numpy(tiles.view(np.uint8).reshape(-1).copy())
        gathered = sharded.gather_records(c_t, t_t, mine.size, dist)
        if rank == 0:
            res = api.Resolver()
            res.set_output_array(100000)
            sharded.resolve_gathered(res, gathered, plan)
            n = res.output_count()
            lines = [res._out[i].raw_line() for i in range(n)]
            exp, exp_stats = C.oracle_decode(data)
            q.put((lines == [m.hexline() for m in exp], list(res.stats().values()) == exp_stats, n))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("nsamples,seed", [(600000, 31), (262144 * 2 + 1000, 32)])
def test_two_rank_gather_and_resolve(nsamples, seed, checker_libs):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, nsamples, seed, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=240)
        assert p.exitcode == 0
    same_lines, same_stats, n = q.get(timeout=10)
    assert same_lines and same_stats and n > 0


def _tiled(sel, n_buffers):
    """One tile per TILE_SAMPLES positions, like the scan kernel."""
    g = (sel["t"] + 2) // api.TILE_SAMPLES
    nt = api.tiles_for(n_buffers)
    cnt = np.bincount(g, minlength=nt).astype(np.uint32)
    t = np.zeros(nt, dtype=api.TILE_DTYPE)
    t["count"] = cnt
    t["offset"] = np.concatenate([[0], np.cumsum(cnt)[:-1]])
    return t


def _wrong_guess_stream(nbuf):
    """An address announced only early in the first shard and used by an address/parity reply much
    later: missing from the tail-based first guess of the next shard's cache (see test_host_logic)."""
    me = bytes([0x58, 0xC3, 0x82, 0xD6, 0x90, 0xC8, 0xAC])
    a, b = 0x4840D6, 0x3C6444
    frames = [(131072 + 5000, synth.make_frame(17, 5, a.to_bytes(3, "big") + me), 80.0, 0.3, 0.0)]
    for k in range(nbuf):
        frames.append((131072 * k + 40000, synth.make_frame(17, 5, b.to_bytes(3, "big") + me), 70.0, 1.1, 0.0))
    frames.append((131072 * (nbuf // 2 + 2) + 9000, synth.make_frame(4, 0, bytes([0x01, 0x85, 0x10]), icao_for_ap=a), 75.0, 0.7, 0.0))
    frames.append((131072 * (nbuf - 4) + 9000, synth.make_frame(5, 0, bytes([0x02, 0x20, 0x31]), icao_for_ap=b), 75.0, 0.2, 0.0))
    return synth.synth_stream(131072 * nbuf, frames, seed=9)


def _dist_worker(rank, world, port, kind, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        if kind.startswith("wrong_guess"):
            data = _wrong_guess_stream(24)
            total_buffers = 24
        elif kind.startswith("chain"):
            data = S.chain(kind)
            total_buffers = data.size // api.BUFFER_BYTES + 1
        else:
            data = synth.random_traffic(131072 * 9 + 5000, 1500, 77, n_aircraft=20)
            total_buffers = data.size // api.BUFFER_BYTES + 1
        plan = sharded.shard_plan(total_buffers, world)
        first, count = plan[rank]
        cands = C.oracle_scan_candidates(data, drop_eof=1 if kind.startswith("wrong_guess") else 0)
        arr = np.frombuffer(b"".join(bytes(c) for c in cands), dtype=api.CANDIDATE_DTYPE).copy()
        mine = arr[((arr["t"] >> 17) >= first) & ((arr["t"] >> 17) < first + count)].copy()
        mine["t"] -= first << 17
        res = api.Resolver()
        res.set_output_array(100000)
        xchg = sharded.ShmExchange(dist) if kind.endswith("_shm") else None
        info = sharded.resolve_distributed(res, mine, _tiled(mine, count), first, dist, exchange=xchg)
        assert set(info["ms"]) == {"tail", "exchange", "tentative", "commit"} and all(v >= 0 for v in info["ms"].values())
        if xchg:
            assert np.array_equal(xchg.all_gather(np.full(7, rank, dtype=np.uint32))[:, 0], np.arange(world))
            xchg.close()
        n = res.output_count()
        lines = [res._out[i].raw_line() for i in range(n)]
        pos = [int(res._out[i].sample_pos) for i in range(n)]
        everything = [None] * world
        dist.all_gather_object(everything, (lines, pos, list(res.stats().values()), info["rounds"]))
        if rank == 0:
            exp, exp_stats = C.oracle_decode(data, drop_eof=1 if kind.startswith("wrong_guess") else 0)
            got_lines = [l for part in everything for l in part[0]]
            got_pos = [x for part in everything for x in part[1]]
            got_stats = [sum(part[2][i] for part in everything) for i in range(8)]
            q.put((got_lines == [m.hexline() for m in exp], got_pos == [m.sample_pos for m in exp], got_stats == exp_stats,
                   everything[0][3], len(got_lines)))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world,kind", [(2, "traffic"), (3, "traffic"), (2, "wrong_guess"), (3, "traffic_shm"), (2, "wrong_guess_shm"),
                                        (2, "chain_evict"), (3, "chain_df4")])
def test_every_rank_resolves_its_own_shard(world, kind, checker_libs):
    """sharded.resolve_distributed over gloo: ranks exchange 4 KiB address caches only, never records,
    and the concatenation of their messages is exactly the sequential decode — also when the first
    guess of a shard's starting cache is wrong (then a second round is needed, and taken), and on a
    chain through the address cache where every shard's outcome depends on the previous shard's."""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_dist_worker, args=(r, world, port, kind, q)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=300)
        assert p.exitcode == 0
    same_lines, same_pos, same_stats, rounds, n = q.get(timeout=10)
    assert same_lines and same_pos and same_stats and n > 0
    assert rounds == 2 if kind.startswith("wrong_guess") else 1 <= rounds <= world


def test_shard_plan_and_carry():
    assert sharded.shard_plan(10, 4) == [(0, 3), (3, 3), (6, 2), (8, 2)]
    assert sharded.shard_plan(2, 4) == [(0, 1), (1, 1), (2, 0), (2, 0)]
    stream = (np.arange(3 * api.BUFFER_BYTES) % 251).astype(np.uint8)
    assert sharded.carry_before(stream, 0) is None
    c = sharded.carry_before(stream, 2)
    assert len(c) == api.CARRY_BYTES and c == bytes(stream[2 * api.BUFFER_BYTES - api.CARRY_BYTES: 2 * api.BUFFER_BYTES])


def test_bind_near_gpu_is_best_effort():
    """No GPU (or no sysfs entry) must not raise: the helper reports and leaves the affinity alone."""
    import os
    from dump1090_b200 import sharded
    before = os.sched_getaffinity(0)
    info = sharded.bind_near_gpu(0)
    assert "numa_node" in info and "cpus" in info
    import torch
    if not torch.cuda.is_available():
        assert info["cpus"] is None and os.sched_getaffinity(0) == before


def _xchg_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import time
        x = sharded.ShmExchange(dist, max_words=64)
        rng = np.random.default_rng(100 + rank)
        ok = True
        for s in range(400):
            if rng.random() < 0.2:
                time.sleep(float(rng.random()) * 2e-3)                    # ranks drift apart by whole exchanges' worth of time
            n = 1 + (s * 7) % 64                                          # every rank the same size in one exchange
            got = x.all_gather(np.full(n, 1000 * s + rank, dtype=np.uint32))
            ok &= got.shape == (world, n) and all(np.all(got[r] == 1000 * s + r) for r in range(world))
        x.close()
        q.put(bool(ok))
    finally:
        dist.destroy_process_group()


def test_shm_exchange_keeps_ranks_in_step():
    """Two rows per rank and one wait per exchange: no rank may read a row that its owner has already
    rewritten for a later exchange, however the ranks drift."""
    world = 3
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_xchg_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=300)
        assert p.exitcode == 0
    assert all(q.get(timeout=10) for _ in range(world))
