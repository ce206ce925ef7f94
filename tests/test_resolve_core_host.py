"""CPU check of the algorithm the device resolve runs (dump1090_b200/csrc/modes_resolve_core.cuh +
the buffer-parallel schedule of modes_resolve_gpu.cu): every reference buffer replayed on its own
from a guessed address cache, caches handed on slot by slot, wrong guesses repeated.  The host shim
(tests/host_shim/resolve_core_host.cpp, test infrastructure) must deliver exactly what the product's
sequential host resolver delivers, with the same statistics, on every stream and flag set."""
import ctypes
import subprocess

import numpy as np
import pytest

import checker as C
import streams as S
from dump1090_b200 import api, synth

SHIM = C.ROOT / "tests" / "_build" / "libresolve_core_host.so"


class Delivery(ctypes.Structure):
    _fields_ = [("t", ctypes.c_int64), ("pass_", ctypes.c_int32), ("crcok", ctypes.c_int32), ("phase_corrected", ctypes.c_int32),
                ("extra", ctypes.c_int32), ("extra_is_ap", ctypes.c_int32), ("pad", ctypes.c_int32)]


@pytest.fixture(scope="module")
def shim(checker_libs):
    subprocess.run(["make", "-s", "shim"], cwd=C.ROOT, check=True)
    lib = ctypes.CDLL(str(SHIM))
    lib.shim_resolve_buffers.restype = ctypes.c_long
    return lib


def _tiled(arr, n_buffers):
    g = (arr["t"] + 2) // api.TILE_SAMPLES
    nt = api.tiles_for(n_buffers)
    cnt = np.bincount(g, minlength=nt).astype(np.uint32)
    t = np.zeros(nt, dtype=api.TILE_DTYPE)
    t["count"] = cnt
    t["offset"] = np.concatenate([[0], np.cumsum(cnt)[:-1]])
    return t


def _streams():
    yield "modes1", C.modes1()
    yield "traffic", synth.random_traffic(131072 * 9 + 5000, 1500, 77, n_aircraft=20)
    yield "dense_fleet", synth.random_traffic(131072 * 30, 9000, 5, n_aircraft=60)
    yield "grid", synth.df17_grid(280000, 700, 5)
    yield "ties", S.tie_rich(11)
    yield "retry_at_j0", S.retry_at_buffer_start()
    yield from S.chain_streams()


STREAMS = dict(_streams())
_scans = {}


def _candidates(name, fix, aggressive):
    key = (name, fix, aggressive)
    if key not in _scans:
        _scans[key] = C.oracle_scan_candidates(STREAMS[name], fix=fix, aggressive=aggressive, cap=400000)
    return _scans[key]


FLAG_SETS = [dict(), dict(aggressive=1), dict(check_crc=0), dict(check_crc=0, aggressive=1), dict(fix=0)]


def _cases():
    """(flags, stream, max_rounds), named flags-stream for the rounds-until-settled runs and
    flags-stream-roundsN for the device's schedule."""
    for max_rounds in (0, 1, 2, 4):
        for name in STREAMS:
            for kw in FLAG_SETS:
                kid = "-".join(f"{a}{b}" for a, b in kw.items()) or "default"
                yield pytest.param(kw, name, max_rounds, id=f"{kid}-{name}" + (f"-rounds{max_rounds}" if max_rounds else ""))


@pytest.mark.parametrize("kw,name,max_rounds", list(_cases()))
def test_buffer_parallel_resolve_equals_sequential(kw, name, max_rounds, shim):
    """max_rounds = 0: guess and verify until nothing changes; 1, 2, 4: the device's schedule, that
    many rounds and then, if the caches are still changing, one replay in stream order."""
    data = STREAMS[name]
    nbuf = data.size // api.BUFFER_BYTES + 1
    cands = _candidates(name, kw.get("fix", 1), kw.get("aggressive", 0))
    arr = np.frombuffer(b"".join(bytes(c) for c in cands), dtype=api.CANDIDATE_DTYPE).copy()
    tiles = _tiled(arr, nbuf)
    # the rule: the product's sequential host resolver
    seq = api.Resolver(fix_errors=kw.get("fix", 1), aggressive=kw.get("aggressive", 0), check_crc=kw.get("check_crc", 1))
    seq.run(arr, tiles)
    want = seq.take_messages()
    cap = 2 * len(cands) + 16
    out = (Delivery * cap)()
    stats = (ctypes.c_int64 * 8)()
    start = np.zeros(1024, dtype=np.uint32)
    end = np.zeros(1024, dtype=np.uint32)
    rounds, fallback = ctypes.c_int(0), ctypes.c_int(0)
    n = shim.shim_resolve_buffers(arr.ctypes.data_as(ctypes.c_void_p), tiles.ctypes.data_as(ctypes.c_void_p),
                                  ctypes.c_size_t(tiles.size), ctypes.c_size_t(nbuf), int(kw.get("check_crc", 1)),
                                  start.ctypes.data_as(ctypes.c_void_p), out, ctypes.c_size_t(cap), stats,
                                  end.ctypes.data_as(ctypes.c_void_p), ctypes.byref(rounds), api.TILE_SAMPLES,
                                  max_rounds, ctypes.byref(fallback))
    assert n >= 0, "did not settle" if n == -2 else "the hand-over after the in-order replay found a wrong cache"
    assert n == len(want)
    assert list(stats) == list(seq.stats().values())
    by_t = {int(c.t): c for c in cands}
    for d, m in zip(out[:n], want):
        ev = by_t[d.t].passes[d.pass_]
        assert d.t - 238 == m.sample_pos and bytes(ev.msg) == bytes(m.msg)
        assert (d.crcok, d.phase_corrected) == (m.crcok, m.phase_corrected)
        if d.extra_is_ap:
            assert d.extra == (m.aa1 << 16) | (m.aa2 << 8) | m.aa3
        else:
            assert d.extra == m.iid
    assert np.array_equal(end, seq.get_cache())
    assert 1 <= rounds.value <= nbuf
    if max_rounds:
        assert rounds.value <= max_rounds
        if name.startswith("chain_"):
            assert fallback.value                                         # the in-order replay was taken, and exact
    else:
        assert not fallback.value
        if name.startswith("chain_") and nbuf > 8:
            assert rounds.value > 4                                       # the chain defeats the device's fixed rounds
