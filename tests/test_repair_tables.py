"""CPU (-m "not gpu"): the CRC repair's tables and the repair itself, exhaustively.

The reference repairs a frame by looking its syndrome up in a sorted table of every 1- and 2-bit
error pattern over positions 5..111 (bitErrorTable, fixBitErrors: dump1090.c:795-894).  The kernels
replace the search with two hash tables (fix_hash, pair_hash: dump1090_b200/csrc/modes_tables.cpp)
and rely on the code's low-weight structure to do so.  Here:
  * the reference's table, read through ctypes, equals an independent construction, and the
    structure the kernels rely on holds (no pair shares a single's syndrome; the low-weight
    codewords that make miscorrections are counted);
  * the product's tables return every entry and reject every other syndrome;
  * serial::crc_and_fix (compiled for the host, tests/host_shim/) repairs all 2^24 syndromes of a
    long and a short frame, with and without `aggressive`, exactly as a model built on the
    reference's own table does, and the model equals fixBitErrors itself on the corpus and on
    random syndromes.
"""
import ctypes
import itertools
import subprocess
import time

import numpy as np
import pytest

import checker as C
import repair_corpus as R
from dump1090_b200 import synth

needs_ref = pytest.mark.skipif(not C.have_ref(), reason="oracle/_ref not built")

SHIM = C.ROOT / "tests" / "_build" / "libeval_serial_host.so"
PAIR_SLOTS = 1 << 14
SWEEP_CHUNK = 1 << 20
# struct modes_frame_eval (include/modes_b200.h)
FRAME_EVAL = np.dtype([("msg", "u1", 14), ("msgtype", "u1"), ("flags", "u1"), ("errorbit", "u1"), ("nfixed", "u1"),
                       ("crc", "<u4")], align=True)


@pytest.fixture(scope="module")
def shim(checker_libs):
    subprocess.run(["make", "-s", "shim"], cwd=C.ROOT, check=True)
    lib = ctypes.CDLL(str(SHIM))
    p = ctypes.c_void_p
    lib.shim_tables.argtypes = [p, p, p]
    lib.shim_build_bit_syndromes.argtypes = [p]
    lib.shim_build_fix_hash.argtypes = [p, p]
    lib.shim_build_pair_hash.argtypes = [p, p]
    lib.shim_probe.argtypes = [p, ctypes.c_uint32, p, p]
    lib.shim_probe.restype = None
    lib.shim_crc_and_fix.argtypes = [p, ctypes.c_uint64, ctypes.c_int, ctypes.c_int, p]
    return lib


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _product_tables(shim):
    syn = np.zeros(112, dtype=np.uint32)
    fix = np.zeros(256, dtype=np.uint32)
    pair = np.zeros(PAIR_SLOTS, dtype=np.uint32)
    assert shim.shim_tables(_ptr(syn), _ptr(fix), _ptr(pair)) == 0
    return syn, fix, pair


def _independent_table():
    """(syndrome, bits, pos0, pos1) of every 1- and 2-bit pattern over positions 5..111, sorted."""
    syn = R.bit_syndromes()
    rows = [(syn[p], 1, p, -1) for p in range(5, 112)]
    rows += [(syn[p] ^ syn[q], 2, p, q) for p, q in itertools.combinations(range(5, 112), 2)]
    return np.array(sorted(rows), dtype=np.int64)


# ---- the code and the tables ----------------------------------------------------------------

def test_code_structure():
    """The numbers the repair paths rely on, recomputed from the generator."""
    assert bin(synth.GENERATOR).count("1") == 16           # even weight: (x + 1) divides it, every codeword has even weight
    syn = R.bit_syndromes()
    singles = {syn[p] for p in range(5, 112)}
    pairs = [syn[p] ^ syn[q] for p, q in itertools.combinations(range(5, 112), 2)]
    assert len(singles) == 107 and len(set(pairs)) == 5671
    assert not singles & set(pairs)                        # no pair aliases a single
    assert R.codewords(4, range(112)) == []                # so no weight-2 or weight-4 codeword anywhere
    long6 = R.long_codewords6()
    assert len(long6) == 224
    assert sum(min(c) >= 5 for c in long6) == 155          # 4-bit errors alias a pair, 5-bit errors a single
    assert sum(min(c) < 5 for c in long6) == 69            # touch the DF field
    assert R.codewords(6, range(56, 112)) == []            # short frames: no weight 6 ...
    assert len(R.short_codewords8()) == 236                # ... but 236 of weight 8 (6- and 7-bit errors alias)


@needs_ref
def test_reference_table_equals_independent_construction(checker_libs):
    tab = C.ref_error_table()
    assert tab.shape == (5778, 4)
    assert np.unique(tab[:, 0]).size == 5778 and np.all(np.diff(tab[:, 0]) > 0)
    assert np.array_equal(tab, _independent_table())


def test_bit_syndromes_equal_reference(shim, checker_libs):
    syn, _, _ = _product_tables(shim)
    assert syn.tolist() == list(R.bit_syndromes())
    assert [int(syn[p]) for p in range(88, 112)] == [1 << (111 - p) for p in range(88, 112)]
    if C.have_ref():
        assert syn[:88].tolist() == C.ref_checksum_table()[:88]


def test_hashes_return_entries_and_reject_everything_else(shim):
    """fix_hash and pair_hash probed with every 24-bit syndrome."""
    syn = R.bit_syndromes()
    want_single = np.full(1 << 24, -1, dtype=np.int32)
    want_pair = np.full(1 << 24, -1, dtype=np.int32)
    for p in range(5, 112):
        want_single[syn[p]] = p
    for p, q in itertools.combinations(range(5, 112), 2):
        want_pair[syn[p] ^ syn[q]] = p
    s = np.arange(1 << 24, dtype=np.uint32)
    single = np.empty(s.size, dtype=np.int32)
    first = np.empty(s.size, dtype=np.int32)
    shim.shim_probe(_ptr(s), s.size, _ptr(single), _ptr(first))
    assert np.array_equal(single, want_single)
    assert np.array_equal(first, want_pair)


def test_pair_table_refuses_a_pair_that_aliases_a_single(shim):
    syn = np.array(R.bit_syndromes(), dtype=np.uint32)
    out = np.zeros(PAIR_SLOTS, dtype=np.uint32)
    assert shim.shim_build_pair_hash(_ptr(syn), _ptr(out)) == 1
    bad = syn.copy()
    bad[7] = bad[5] ^ bad[6]                               # pair (5, 6) now has single 7's syndrome
    assert shim.shim_build_pair_hash(_ptr(bad), _ptr(out)) == 0
    fix = np.zeros(256, dtype=np.uint32)
    assert shim.shim_build_fix_hash(_ptr(bad), _ptr(fix)) == 1    # the singles alone are still distinct


# ---- the model of the repair, against the reference's own fixBitErrors ------------------------

@needs_ref
def test_model_equals_fix_bit_errors(checker_libs):
    table = C.ref_error_table()
    frames = R.frames_array()
    rng = np.random.default_rng(24)
    rand = np.zeros((2 << 16, 14), dtype=np.uint8)
    rand[: 1 << 16] = np.frombuffer(R.BASES["df17b"], dtype=np.uint8)
    rand[1 << 16:, :7] = np.frombuffer(R.BASES["df11b"], dtype=np.uint8)
    s = rng.integers(1, 1 << 24, size=2 << 16)
    for k in range(3):
        rand[: 1 << 16, 11 + k] ^= (s[: 1 << 16] >> (16 - 8 * k)).astype(np.uint8)
        rand[1 << 16:, 4 + k] ^= (s[1 << 16:] >> (16 - 8 * k)).astype(np.uint8)
    assert np.array_equal(R.syndromes(rand), s)
    n_fixed = {1: 0, 2: 0}
    for frames_ in (frames, rand):
        s_ = R.syndromes(frames_)
        bits = R.nbits_of_array(frames_[:, 0] >> 3)
        for maxfix in (1, 2):
            ok, nb, p0, p1 = R.table_lookup(table, s_, bits, maxfix)
            for i in range(frames_.shape[0]):
                got, n, pos = C.ref_fix_bit_errors(frames_[i].tobytes(), int(bits[i]), maxfix)
                want = [int(p0[i]), int(p1[i])][: int(nb[i])]
                assert (n, pos) == (int(nb[i]), want), (i, n, pos, want)
                assert got == synth.flip_bits(frames_[i].tobytes(), want)
                n_fixed[n] = n_fixed.get(n, 0) + 1
    print(f"model == fixBitErrors: {n_fixed[1]} single-bit and {n_fixed[2]} two-bit repairs")
    assert n_fixed[1] > 5000 and n_fixed[2] > 40000


# ---- exhaustive sweep of serial::crc_and_fix -------------------------------------------------

def compare_sweep(got_msg, got_crc, got_errorbit, got_nfixed, want):
    """Mismatch count and first mismatch of a sweep chunk against model_repair's answer."""
    w_msg, w_crc, w_err, w_nf = want
    bad = (got_msg != w_msg).any(axis=1) | (got_crc != w_crc) | (got_errorbit != (w_err & 0xFF)) | (got_nfixed != w_nf)
    return np.flatnonzero(bad)


@needs_ref
@pytest.mark.parametrize("aggressive", [0, 1])
@pytest.mark.parametrize("base", ["df17a", "df11a"])
def test_serial_crc_and_fix_sweeps_every_syndrome(base, aggressive, shim, checker_libs):
    table = C.ref_error_table()
    t0 = time.perf_counter()
    counts = np.zeros(3, dtype=np.int64)
    for s, frames in R.sweep_chunks(R.BASES[base], SWEEP_CHUNK):
        out = np.zeros(s.size, dtype=FRAME_EVAL)
        assert shim.shim_crc_and_fix(_ptr(frames), s.size, 1, aggressive, _ptr(out)) == 0
        want = R.model_repair(table, frames, 1, aggressive, s)
        raw = out.view(np.uint8).reshape(-1, 24)
        bad = compare_sweep(raw[:, :14], out["crc"], out["errorbit"], out["nfixed"], want)
        assert bad.size == 0, f"{bad.size} syndromes differ, first S = {s[bad[0]]:#08x}: " \
                              f"{raw[bad[0]].tolist()} vs {want[0][bad[0]].tolist()} crc {want[1][bad[0]]} " \
                              f"errorbit {want[2][bad[0]]} nfixed {want[3][bad[0]]}"
        counts += np.bincount(want[3], minlength=3)
    nbits = 8 * len(R.BASES[base])
    print(f"{base} aggressive={aggressive}: {counts[1]} single-bit, {counts[2]} two-bit repairs of 2^24 "
          f"syndromes in {time.perf_counter() - t0:.1f} s")
    assert counts[1] == (107 if nbits == 112 else 56)             # every single inside the frame and the table
    assert counts[2] == (0 if not aggressive else 5671 if nbits == 112 else 1540)
