"""CPU check of the per-candidate evaluation that the frame-evaluation kernels run one thread per
candidate (dump1090_b200/csrc/modes_eval_serial.cuh: the single walk of eval_fused_kernel, whole and
half windows, and the two-pass codings of eval_serial_kernel): the same header is compiled for the host
(tests/host_shim/, test infrastructure only) and fed the oracle's candidate positions; the
evaluated records — both attempts, frame bytes, gate/CRC/repair verdicts — must equal the
oracle's byte for byte.  The GPU parity tests check the kernel itself."""
import ctypes
import subprocess

import numpy as np
import pytest

import checker as C
from dump1090_b200 import api, synth
import repair_corpus as R
import streams as S

SHIM = C.ROOT / "tests" / "_build" / "libeval_serial_host.so"


@pytest.fixture(scope="module")
def shim(checker_libs):
    subprocess.run(["make", "-s", "shim"], cwd=C.ROOT, check=True)
    lib = ctypes.CDLL(str(SHIM))
    lib.shim_eval_candidates.restype = ctypes.c_int
    lib.shim_eval_candidates.argtypes = [ctypes.c_void_p, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_uint32,
                                         ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    return lib


def _streams():
    yield "modes1", C.modes1()
    for seed in (1, 2, 3):
        yield f"traffic{seed}", synth.random_traffic(300000, 400, seed)
    yield "grid", synth.df17_grid(280000, 700, 5)
    yield "ties", S.tie_rich(11)
    yield "ties_weak", S.tie_rich(12, levels=(0, 0, 1, 3, 30))
    yield "retry_at_j0", S.retry_at_buffer_start()
    yield "repair0", R.repair_stream(0.0)                              # tests/repair_corpus.py
    yield "repair_frac", R.repair_stream(R.RETRY_FRAC)


STREAMS = dict(_streams())


def _evaluate(shim, data, fix, aggressive, lean):
    exp = C.oracle_scan_candidates(data, fix=fix, aggressive=aggressive, cap=400000)
    want = np.frombuffer(b"".join(bytes(c) for c in exp), dtype=api.CANDIDATE_DTYPE)
    nbuf = data.size // api.BUFFER_BYTES + 1
    virt = np.full(480 + nbuf * api.BUFFER_BYTES, 127, dtype=np.uint8)   # halo (initial carry: no signal) + whole buffers
    virt[480: 480 + data.size] = data
    v = (want["t"] + 2).astype(np.uint32)
    got = np.zeros(want.size, dtype=api.CANDIDATE_DTYPE)
    rc = shim.shim_eval_candidates(virt.ctypes.data, virt.size // 2, v.ctypes.data, v.size, fix, aggressive, lean,
                                   got.ctypes.data)
    assert rc == 0
    return got.view(np.uint8).reshape(-1, 56), want.view(np.uint8).reshape(-1, 56)


@pytest.mark.parametrize("name", list(STREAMS))
@pytest.mark.parametrize("fix,aggressive", [(1, 0), (1, 1), (0, 0)])
@pytest.mark.parametrize("lean", [0, 1, 2, 3], ids=["two_pass", "two_pass_lean", "fused", "fused_halves"])
def test_serial_evaluation_matches_oracle(name, fix, aggressive, lean, shim):
    got, want = _evaluate(shim, STREAMS[name], fix, aggressive, lean)
    assert want.shape[0] > (200 if name != "retry_at_j0" else 10)
    bad = np.nonzero((got != want).any(axis=1))[0]
    assert bad.size == 0, f"{bad.size} of {want.shape[0]} records differ, first at {bad[0]}: {got[bad[0]].tolist()} != {want[bad[0]].tolist()}"


@pytest.mark.parametrize("lean", [0, 1, 2, 3], ids=["two_pass", "two_pass_lean", "fused", "fused_halves"])
def test_serial_evaluation_random_alphabets(lean, shim):
    """Many small streams with random amplitude alphabets, preamble jitter and noise levels: weak
    and saturated pairs, long indefinite runs, every gate outcome."""
    total = 0
    for case, levels, data in S.random_alphabet_cases():
        for fix, aggressive in ((1, 1), (0, 0)):
            got, want = _evaluate(shim, data, fix, aggressive, lean)
            total += want.shape[0]
            bad = np.nonzero((got != want).any(axis=1))[0]
            assert bad.size == 0, f"case {case} levels {levels}: {bad.size} of {want.shape[0]} records differ"
    assert total > 5000
