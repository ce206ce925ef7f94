"""Receiver-pool buffers fed from device memory (modes_pool_submit_device / modes_pool_ingest_device, CUDA
tensors in ReceiverPool.ingest / submit).

Every GPU contract case feeds one pool each call's buffers from host memory and another the same bytes from
device memory, in the same calls, and asks for the same output record for record: every message's bytes, the
receiver of each message in the shared output array, statistics, buffers(r), and the level, spectrum,
recovery and weak records.  The gather launch that fills the device-fed 2 MHz pairs is checked byte for byte
through a device harness of its own against a numpy model.  CPU tests check the exports and how ReceiverPool
sends each kind of input."""
from __future__ import annotations

import ctypes
import subprocess
import types

import numpy as np
import pytest

import checker as C
from dump1090_b200 import api
from test_pool import _schedule
from test_pool_input_format import (FLAG_SETS, KINDS, N_CALLS, SWITCHES, _mixed, _pool, _want_buffers,
                                    full_world)  # noqa: F401  (full_world: a fixture)

ROOT = C.ROOT
DSHIM = ROOT / "tests" / "_build" / "libgather_pool_device.so"
BUF = api.BUFFER_BYTES
CARRY = api.CARRY_BYTES
OUT_CAP = 200_000


# ---------------------------------------------------------------- CPU


def test_symbols_exported():
    header = (ROOT / "include" / "modes_b200.h").read_text()
    for name, args in (("modes_pool_submit_device", "(modes_pool *p, const uint32_t *receivers, const void *const *d_iq, size_t n);"),
                       ("modes_pool_ingest_device", "(modes_pool *p, const uint32_t *receivers, const void *const *d_iq, size_t n,")):
        assert name in api.EXPORTS
        assert f"int  {name}{args}" in header
        assert hasattr(api.lib(), name)
    assert api.lib().modes_pool_submit_device(None, None, None, 0) == -1
    assert api.lib().modes_pool_ingest_device(None, None, None, 0, ctypes.cast(None, api.POOL_SINK_FN), None) == -1


class _Lib:
    """Records the pool calls a ReceiverPool makes."""

    def __init__(self):
        self.calls = []

    def modes_pool_ingest(self, h, ids, ptrs, n, fn, user):
        self.calls.append(("host", n))
        return 0

    def modes_pool_submit(self, h, ids, ptrs, n):
        self.calls.append(("host", n))
        return 0

    def modes_pool_ingest_device(self, h, ids, ptrs, n, fn, user):
        self.calls.append(("device", [ptrs[i] for i in range(n)]))
        return 0

    def modes_pool_submit_device(self, h, ids, ptrs, n):
        self.calls.append(("device", [ptrs[i] for i in range(n)]))
        return 0

    def modes_pool_collect(self, h, fn, user):
        return 0


class _Device(types.SimpleNamespace):
    def __str__(self):
        return f"cuda:{self.index}"


class _Tensor:
    """What ReceiverPool reads of a CUDA tensor."""

    is_cuda = True

    def __init__(self, ptr, shape, itemsize, index=0, contiguous=True):
        self.ptr, self.shape, self.size, self.contig = ptr, tuple(shape), itemsize, contiguous
        self.device = _Device(index=index)

    def data_ptr(self):
        return self.ptr

    def dim(self):
        return len(self.shape)

    def numel(self):
        return int(np.prod(self.shape))

    def element_size(self):
        return self.size

    def is_contiguous(self):
        return self.contig

    def contiguous(self):
        return _Tensor(0x900000, self.shape, self.size, self.device.index)


@pytest.fixture
def stub(monkeypatch):
    L = _Lib()
    synced = []
    monkeypatch.setattr(api, "lib", lambda: L)
    monkeypatch.setattr(api, "_sync_stream", lambda t: synced.append(t.data_ptr()))
    pool = object.__new__(api.ReceiverPool)
    pool._h, pool.n, pool._fn = 1, 3, None
    pool.cfg = types.SimpleNamespace(device=0)
    pool._bytes = [BUF, 2 * BUF, BUF]
    yield pool, L, synced
    pool._h = None


def test_dispatch(stub):
    pool, L, synced = stub
    pool.ingest([0, 1], [np.zeros(BUF, np.uint8), np.zeros(2 * BUF, np.uint8)])
    assert L.calls == [("host", 2)] and not synced
    L.calls.clear()
    pool.ingest([1, 0], [_Tensor(0x100000, [BUF], 2), _Tensor(0x200000, [BUF // 4], 4, contiguous=False)])
    assert L.calls == [("device", [0x100000, 0x900000])] and synced == [0x100000]
    L.calls.clear()
    pool.submit([2, 0], _Tensor(0x400000, [2, BUF // 2], 2))                # the rows of one 2-D tensor
    assert L.calls == [("device", [0x400000, 0x400000 + BUF])]
    assert len(pool._inflight) == 1
    pool.collect()
    assert not pool._inflight


def test_device_refusals_before_the_pool(stub):
    pool, L, synced = stub
    with pytest.raises(ValueError, match="cuda:1"):
        pool.ingest([0], [_Tensor(0x100000, [BUF], 1, index=1)])
    with pytest.raises(ValueError, match="mixes"):
        pool.ingest([0, 2], [_Tensor(0x100000, [BUF], 1), np.zeros(BUF, np.uint8)])
    with pytest.raises(ValueError, match="mixes"):
        pool.submit([0, 2], [np.zeros(BUF, np.uint8), _Tensor(0x100000, [BUF], 1)])
    with pytest.raises(ValueError, match="input format takes"):
        pool.ingest([1], [_Tensor(0x100000, [BUF], 1)])
    with pytest.raises(ValueError, match="input format takes"):
        pool.submit([0, 1], _Tensor(0x100000, [2, BUF], 1))
    with pytest.raises(ValueError, match="one row per receiver"):
        pool.submit([0, 2], _Tensor(0x100000, [3, BUF], 1))
    assert not L.calls and not synced


# ---------------------------------------------------------------- GPU: the gather launch


@pytest.fixture(scope="module")
def dshim():
    subprocess.run(["make", "-s", "dshim"], cwd=ROOT, check=True)
    lib = ctypes.CDLL(str(DSHIM))
    lib.gpool_gather.restype = ctypes.c_int
    lib.gpool_gather.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p,
                                 ctypes.c_size_t, ctypes.c_void_p, ctypes.c_uint32]
    lib.gpool_error.restype = ctypes.c_char_p
    return lib


GATHER_JOB = np.dtype([(f, np.int64) for f in ("in_off", "data_off", "carry_in_off", "carry_out_off", "pad_tail_off")])


@pytest.mark.gpu
def test_gather_pool_kernel_equals_model(dshim):
    """One launch of 260 jobs (more than a full max_batch = 256 call makes): UC8 buffers from the callers'
    memory (random, rail 0/255 and no-signal bytes) and buffers already in their pairs (16-bit receivers,
    converted), fresh streams and carries read from either half, every pad tail, data buffer and carry slot
    between sentinel bytes; no byte outside them changes."""
    rng = np.random.default_rng(23)
    n_in, n_jobs, gap, sentinel = 12, 260, 64, 0xC3
    bufs = [rng.integers(0, 256, BUF, dtype=np.uint8) for _ in range(n_in)]
    bufs[1] = rng.choice(np.array([0, 255], np.uint8), BUF)                # the rails
    bufs[2] = np.full(BUF, 127, np.uint8)                                  # no signal
    bufs[3][-CARRY:] = rng.choice(np.array([0, 255], np.uint8), CARRY)
    src = np.concatenate(bufs)
    # carries: [half][job] slots at a pitch of CARRY + gap, sentinels between them
    cpitch = CARRY + gap
    carry = np.full(2 * n_jobs * cpitch + gap, sentinel, np.uint8)
    slot = lambda h, i: gap + (h * n_jobs + i) * cpitch                    # noqa: E731
    for h in range(2):
        for i in range(n_jobs):
            carry[slot(h, i): slot(h, i) + CARRY] = rng.integers(0, 256, CARRY, dtype=np.uint8)
    # pairs: [gap][pad tail][gap'][data], data 16-byte aligned, in a shuffled order
    tail_to_data = CARRY + gap + (-(CARRY + gap)) % 16
    ppitch = tail_to_data + BUF + gap
    out = np.full(n_jobs * ppitch + gap, sentinel, np.uint8)
    order = rng.permutation(n_jobs)
    jobs = np.zeros(n_jobs, GATHER_JOB)
    want_out, want_carry = out.copy(), carry.copy()
    kinds = {"caller": 0, "converted": 0, "fresh": 0, "half0": 0, "half1": 0}
    for i in range(n_jobs):
        tail = gap + int(order[i]) * ppitch
        data = tail + tail_to_data
        k = int(rng.integers(0, n_in))
        if i % 3 == 2:                                                     # already converted into its pair
            out[data: data + BUF] = bufs[k]
            in_off = -1
            kinds["converted"] += 1
        else:
            in_off = k * BUF
            kinds["caller"] += 1
        buf = bufs[k]
        h = int(rng.integers(0, 2))
        fresh = i % 5 == 0
        kinds["fresh" if fresh else f"half{h}"] += 1
        jobs[i] = (in_off, data, -1 if fresh else slot(h, i), slot(1 - h, i), tail)
        want_out[data: data + BUF] = buf
        want_out[tail: tail + CARRY] = 127 if fresh else carry[slot(h, i): slot(h, i) + CARRY]
        want_carry[slot(1 - h, i): slot(1 - h, i) + CARRY] = buf[-CARRY:]
    assert min(kinds.values()) > 20, kinds
    got_out, got_carry = out.copy(), carry.copy()
    rc = dshim.gpool_gather(src.ctypes.data, src.size, got_carry.ctypes.data, got_carry.size, got_out.ctypes.data,
                            got_out.size, jobs.ctypes.data, n_jobs)
    assert rc == 0, dshim.gpool_error().decode()
    bad = np.flatnonzero(got_out != want_out)
    assert bad.size == 0, (bad[:5], bad.size)
    bad = np.flatnonzero(got_carry != want_carry)
    assert bad.size == 0, (bad[:5], bad.size)
    # a bad request runs nothing
    jobs[0]["data_off"] += 4
    assert dshim.gpool_gather(src.ctypes.data, src.size, got_carry.ctypes.data, got_carry.size, got_out.ctypes.data,
                              got_out.size, jobs.ctypes.data, n_jobs) == -1


# ---------------------------------------------------------------- GPU: the contract


def _device(rxs):
    import torch
    d = [torch.from_numpy(np.ascontiguousarray(rx.x)).cuda() for rx in rxs]
    torch.cuda.synchronize()
    return d


def _dbuf(rx, d, k):
    return d[k * rx.size: (k + 1) * rx.size]


def _feed(pool, rxs, calls, max_batch, src=None, mode="ingest"):
    """The calls' buffers from host memory (src None) or from each receiver's device copy (src).  mode:
    ingest; scribble (ingest, each buffer a copy of its own, overwritten once the call returns); pipelined
    (submit(k + 1) before collect(k))."""
    import torch
    nxt = [0] * len(rxs)
    pending = 0
    for ids in calls:
        for lo in range(0, len(ids), max_batch):
            part = ids[lo: lo + max_batch]
            if src is None:
                bufs = [rxs[r].buf(nxt[r]) for r in part]
            else:
                bufs = [_dbuf(rxs[r], src[r], nxt[r]) for r in part]
                if mode == "scribble":
                    bufs = [b.clone() for b in bufs]
            for r in part:
                nxt[r] += 1
            if mode == "pipelined":
                pool.submit(part, bufs)
                pending += 1
                if pending == 2:
                    pool.collect()
                    pending -= 1
                continue
            pool.ingest(part, bufs)
            if src is not None and mode == "scribble":
                for b in bufs:
                    b.random_(0, 256)
                torch.cuda.synchronize()
    for _ in range(pending):
        pool.collect()
    return nxt


def _results(pool, n, kw):
    count = pool.output_count()
    assert count <= OUT_CAP
    out = dict(array=[bytes(m) for m in pool._out[:count]], rx=pool._out_rx[:count].tolist())
    for r in range(n):
        d = dict(msgs=[bytes(m) for m in pool.take(r)], stats=pool.stats(r), buffers=pool.buffers(r))
        if kw.get("levels"):
            d["levels"] = pool.take_levels(r).tobytes()
        if kw.get("spectrum"):
            d["spectra"] = pool.take_spectra(r).tobytes()
        if kw.get("recover"):
            d["recovery"] = (pool.recovery_stats(r), pool.weak_recovery_stats(r))
        out[r] = d
    return out


def _compare(rxs, calls, max_batch, kw=None, mode="ingest", cfg=None):
    """A device-fed pool equals a host-fed one on the same calls; returns the host-fed results."""
    kw, cfg = kw or {}, cfg or {}
    src = _device(rxs)
    res = []
    for feed in (None, src):
        with _pool(rxs, max_batch=max_batch, **kw, **cfg) as pool:
            pool.set_output_array(OUT_CAP)
            _feed(pool, rxs, calls, max_batch, feed, "ingest" if feed is None else mode)
            res.append(_results(pool, len(rxs), kw))
    want, got = res
    assert got.keys() == want.keys()
    for k in want:
        assert got[k] == want[k], (k, kw, cfg, mode)
    return want


@pytest.mark.gpu
@pytest.mark.parametrize("kw", FLAG_SETS, ids=lambda k: "-".join(f"{a}{b}" for a, b in k.items()) or "default")
def test_mixed_pool_equals_host_fed(kw, checker_libs):
    """UC8, SC16 and SC16Q11 receivers (one at shift 2) at both rates, mixed in calls of at most 3 and out of
    lock step; under default flags also the oracle on each receiver's converted / resampled bytes."""
    rxs = _mixed()
    cfg = dict(fix_errors=kw.get("fix", 1), aggressive=kw.get("aggressive", 0), check_crc=kw.get("check_crc", 1))
    want = _compare(rxs, _schedule(len(rxs), N_CALLS, seed=6), 3, mode="scribble", cfg=cfg)
    for r, rx in enumerate(rxs):
        assert want[r]["buffers"] == _want_buffers(rx.rate), r
        if rx.fmt != "uc8":
            assert len(want[r]["msgs"]) > 20, r
    if kw:
        return
    with _pool(rxs, max_batch=3) as pool:
        _feed(pool, rxs, _schedule(len(rxs), N_CALLS, seed=6), 3, _device(rxs))
        for r, rx in enumerate(rxs):
            k = pool.buffers(r)
            msgs, stats = C.oracle_decode(rx.decoded(k), drop_eof=1)
            assert [m.raw_line() for m in pool.take(r)] == [m.hexline() for m in msgs], r
            assert list(pool.stats(r).values()) == stats, r


@pytest.mark.gpu
@pytest.mark.parametrize("sw", SWITCHES + [dict(spectrum=True), dict(carrier=True, signal=True),
                                           dict(signal=True, arrival=True, levels=True, spectrum=True, carrier=True,
                                                recover=True, weak_preambles=True)],
                         ids=["signal", "arrival", "levels", "recover", "weak", "spectrum", "carrier", "all"])
def test_every_switch_equals_host_fed(sw):
    """Each switch on its own, and all of them, with two batches in flight."""
    rxs = _mixed()
    want = _compare(rxs, _schedule(len(rxs), N_CALLS, seed=10), 4, kw=sw, mode="pipelined")
    if sw.get("levels"):
        assert any(len(want[r]["levels"]) for r in range(len(rxs)))
    if sw.get("spectrum"):
        assert any(len(want[r]["spectra"]) for r in range(len(rxs)))


@pytest.mark.gpu
def test_call_shapes(checker_libs):
    """A receiver in both batches in flight, a call in which no receiver completes a buffer, the rows of one
    2-D tensor against a list of tensors, and reset and refeed."""
    import torch
    rxs = _mixed()
    n = len(rxs)
    src = _device(rxs)
    # the first call of a 2.4 MS/s receiver alone completes nothing; both batches in flight name receiver 4
    calls = [[4], [4, 2, 0], [2, 5, 4, 1], [5, 4, 2, 0, 1, 3, 6], [0, 1, 2, 3, 4, 5, 6], [6, 3, 1, 0]]
    for mode in ("ingest", "pipelined"):
        res = []
        for feed in (None, src):
            with _pool(rxs, max_batch=n) as pool:
                pool.set_output_array(OUT_CAP)
                _feed(pool, rxs, calls[:1], n, feed, mode)
                if mode == "ingest":
                    assert pool.buffers(4) == 0 and pool.take(4) == []
                _feed(pool, rxs, calls[1:], n, feed, mode)
                res.append(_results(pool, n, {}))
        assert res[1] == res[0], mode
        assert min(res[0][r]["buffers"] for r in range(n)) >= 2
    # rows of one 2-D tensor (UC8, then int16 for the 16-bit receivers) equal a list of tensors
    u8 = [r for r in range(n) if rxs[r].fmt == "uc8"]
    w16 = [r for r in range(n) if rxs[r].fmt != "uc8"]
    res = []
    for shape in ("list", "rows"):
        with _pool(rxs, max_batch=n) as pool:
            for k in range(N_CALLS):
                for grp in (u8, w16[::-1]):
                    bufs = [_dbuf(rxs[r], src[r], k) for r in grp]
                    if shape == "rows":
                        block = torch.stack(bufs)
                        pool.ingest(grp, block if rxs[grp[0]].fmt == "uc8" else block.view(torch.int16))
                    else:
                        pool.ingest(grp, bufs)
            res.append([[bytes(m) for m in pool.take(r)] + [pool.stats(r), pool.buffers(r)] for r in range(n)])
    assert res[0] == res[1]
    # reset and refeed, also with the other kind of memory once reset
    with _pool(rxs, max_batch=n) as pool:
        for rx_id in (0, 4, 3):
            rx = rxs[rx_id]
            for feed in ("device", "host", "device"):
                pool.reset(rx_id)
                pool.take(rx_id)
                for k in range(3):
                    b = _dbuf(rx, src[rx_id], k) if feed == "device" else rx.buf(k)
                    pool.ingest([rx_id], [b])
                kb = pool.buffers(rx_id)
                assert kb == _want_buffers(rx.rate, 3), (rx_id, feed)
                lines = [m.hexline() for m in C.oracle_decode(rx.decoded(kb), drop_eof=1)[0]]
                assert [m.raw_line() for m in pool.take(rx_id)] == lines, (rx_id, feed)


@pytest.mark.gpu
def test_refusals():
    rxs = _mixed()
    src = _device(rxs)
    with _pool(rxs, max_batch=4) as pool:
        x = rxs[0].buf(0)
        with pytest.raises(RuntimeError, match="receiver 0: the bytes are in host memory"):
            pool.ingest_device_ptrs(np.array([0], np.uint32), (ctypes.c_void_p * 1)(x.ctypes.data))
        pinned = api.PinnedBuffer(BUF)
        try:
            with pytest.raises(RuntimeError, match="receiver 0: the bytes are in pinned host memory"):
                pool.submit_device_ptrs(np.array([0], np.uint32), (ctypes.c_void_p * 1)(pinned.ptr))
        finally:
            pinned.free()
        ptr, free = _managed(BUF)
        try:
            with pytest.raises(RuntimeError, match="receiver 2: the bytes are in managed memory"):
                pool.ingest_device_ptrs(np.array([0, 2], np.uint32), (ctypes.c_void_p * 2)(src[0].data_ptr(), ptr))
        finally:
            free(ptr)
        with pytest.raises(RuntimeError, match="receiver 1: null pointer"):
            pool.ingest_device_ptrs(np.array([0, 1], np.uint32), (ctypes.c_void_p * 2)(src[0].data_ptr(), None))
        with pytest.raises(RuntimeError, match="receiver 2: .* not 16-byte aligned"):
            pool.ingest_device_ptrs(np.array([0, 2], np.uint32),
                                    (ctypes.c_void_p * 2)(src[0].data_ptr(), src[2].data_ptr() + 4))
        with pytest.raises(ValueError, match="input format takes"):
            pool.ingest([2], [src[2][:BUF]])
        with pytest.raises(ValueError, match="mixes"):
            pool.ingest([0, 1], [src[0][:BUF], rxs[1].buf(0)])
        # nothing above started a stream: every receiver takes either kind of memory
        for r in range(len(rxs)):
            pool.set_input_rate(r, rxs[r].rate)
        # one kind of memory per receiver until reset
        pool.ingest([0, 1], [_dbuf(rxs[0], src[0], 0), _dbuf(rxs[1], src[1], 0)])
        pool.ingest([2], [rxs[2].buf(0)])
        with pytest.raises(RuntimeError, match="receiver 1 has a stream fed from device memory in progress"):
            pool.ingest([2, 1], [rxs[2].buf(1), rxs[1].buf(1)])
        with pytest.raises(RuntimeError, match="receiver 2 has a stream fed from host memory in progress"):
            pool.submit([0, 2], [_dbuf(rxs[0], src[0], 1), _dbuf(rxs[2], src[2], 1)])
        pool.ingest([1, 0], [_dbuf(rxs[1], src[1], 1), _dbuf(rxs[0], src[0], 1)])   # the refusals changed nothing
        assert pool.buffers(0) == 2
        pool.reset(1)
        pool.ingest([1], [rxs[1].buf(0)])


def _managed(nbytes):
    """(address, free) of managed memory from the CUDA runtime torch loads."""
    import torch  # noqa: F401  (loads the runtime)
    rt = ctypes.CDLL("libcudart.so.12")
    p = ctypes.c_void_p()
    assert rt.cudaMallocManaged(ctypes.byref(p), ctypes.c_size_t(nbytes), ctypes.c_uint(1)) == 0
    return p.value, lambda q: rt.cudaFree(ctypes.c_void_p(q))


@pytest.mark.gpu
@pytest.mark.skipif("not __import__('torch').cuda.device_count() > 1", reason="needs two GPUs")
def test_tensor_on_other_device():
    import torch
    t = torch.zeros(BUF, dtype=torch.uint8, device="cuda:1")
    with api.ReceiverPool(2) as pool:
        with pytest.raises(ValueError, match="cuda:1"):
            pool.ingest([0], [t])
        with pytest.raises(RuntimeError, match="memory of device 1"):
            pool.ingest_device_ptrs(np.array([0], np.uint32), (ctypes.c_void_p * 1)(t.data_ptr()))


# ---------------------------------------------------------------- GPU: at full batch size


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["ingest", "pipelined"])
def test_full_batch_equals_host_fed(mode, full_world):
    """256 receivers of all six format and rate combinations at max_batch = 256."""
    rxs, calls = full_world["rxs"], full_world["calls"]
    assert {(rx.fmt, rx.rate) for rx in rxs} == set(KINDS)
    want = _compare(rxs, calls, len(rxs), mode=mode)
    assert sum(len(want[r]["msgs"]) for r in range(len(rxs))) > 1000
