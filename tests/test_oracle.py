"""CPU (-m "not gpu"): pin the oracle restatement against the reference and the golden fixtures."""
import ctypes
import hashlib

import numpy as np
import pytest

import checker as C
import golden_util as G
from dump1090_b200 import synth

FLAG_SETS = [dict(), dict(aggressive=1), dict(fix=0), dict(check_crc=0), dict(check_crc=0, aggressive=1),
             dict(drop_eof=1), dict(fix=0, drop_eof=1), dict(check_crc=0, aggressive=1, drop_eof=1)]

# line count and md5 of the --raw output of the reference on checker.modes1() (the stored head of modes1.bin)
MODES1_PINS = {
    (): (147, "f23b14fbd58d"), (("drop_eof", 1),): (119, "896cf3d1da7e"),
    (("aggressive", 1),): (147, "f23b14fbd58d"), (("fix", 0),): (147, "a8c3b59364d7"),
    (("drop_eof", 1), ("fix", 0)): (119, "896cf3d1da7e"), (("check_crc", 0),): (359, "5c32e315e805"),
    (("aggressive", 1), ("check_crc", 0)): (385, "5c0d8b9ab062"),
    (("aggressive", 1), ("check_crc", 0), ("drop_eof", 1)): (308, "412617cf2a6d"),
}


def _md5_lines(msgs):
    return hashlib.md5("".join(m.hexline() + "\n" for m in msgs).encode()).hexdigest()[:12]


def _fields(msgs):
    return [C.msg_fields(m) for m in msgs]


needs_ref = pytest.mark.skipif(not C.have_ref(), reason="oracle/_ref not built")


@pytest.mark.parametrize("kw", FLAG_SETS, ids=str)
def test_oracle_modes1_pins(kw, checker_libs):
    msgs, _ = C.oracle_decode(C.modes1(), **kw)
    key = tuple(sorted(kw.items()))
    if key in MODES1_PINS:
        assert (len(msgs), _md5_lines(msgs)) == MODES1_PINS[key]


def test_oracle_modes1_stats_pins(checker_libs):
    # the reference's stat counters (single-bit fixes are double counted by the reference: 2 -> 4)
    _, st = C.oracle_decode(C.modes1())
    assert st == [261, 125, 256, 145, 111, 2, 4, 0]
    _, st = C.oracle_decode(C.modes1(), fix=0)
    assert st[:5] == [261, 126, 256, 147, 109]
    msgs, _ = C.oracle_decode(C.modes1())
    hist = {}
    for m in msgs:
        hist[m.msgtype] = hist.get(m.msgtype, 0) + 1
    assert hist == {0: 9, 4: 2, 5: 4, 11: 43, 17: 79, 20: 7, 21: 3}


@needs_ref
@pytest.mark.parametrize("kw", FLAG_SETS, ids=str)
def test_oracle_equals_reference_modes1(kw, checker_libs):
    r, rs = C.ref_decode(C.modes1(), **kw)
    o, os_ = C.oracle_decode(C.modes1(), **kw)
    assert _fields(r) == _fields(o)
    assert rs == os_


@needs_ref
@pytest.mark.parametrize("seed", [11, 12, 13])
@pytest.mark.parametrize("kw", [dict(), dict(aggressive=1), dict(check_crc=0, aggressive=1)], ids=str)
def test_oracle_equals_reference_synthetic(seed, kw, checker_libs):
    data = synth.random_traffic(200000 + 7777 * seed, 300, seed, sigma=1.0 + seed % 3)
    r, rs = C.ref_decode(data, **kw)
    o, os_ = C.oracle_decode(data, **kw)
    assert _fields(r) == _fields(o)
    assert rs == os_


@pytest.mark.parametrize("name,cid", G.CASES)
def test_oracle_equals_golden(name, cid, checker_libs):
    doc = G.load(name)
    case = doc["cases"][cid]
    data = G.make_input(doc)
    msgs, st = C.oracle_decode(data, **case["flags"])
    assert _fields(msgs) == case["messages"]
    assert st == case["stats"]


def test_magnitude_pins(checker_libs):
    # kernel-level pins for checker.modes1()
    m = C.oracle_magnitude(C.modes1())
    assert m.size == 163840 and int(m.astype(np.int64).sum()) == 938262314 and int(m.max()) == 64913
    assert hashlib.sha256(m.astype("<u2").tobytes()).hexdigest().startswith("c8afd162f16f9d3f")


@needs_ref
def test_magnitude_equals_reference(checker_libs):
    buf = np.full(262620, 127, dtype=np.uint8)
    d = C.modes1()
    buf[476: 476 + 262144] = d[:262144]
    out = np.empty(131310, dtype=np.uint16)
    C.ref_lib().ref_magnitude(buf.ctypes.data_as(ctypes.c_void_p), out.ctypes.data_as(ctypes.c_void_p))
    assert np.array_equal(out, C.oracle_magnitude(buf))


def test_candidate_pins(checker_libs):
    # positions passing all preamble tests, every j, no skip
    cands = C.oracle_scan_candidates(C.modes1())
    t = np.array([c.t for c in cands], dtype=np.int64)
    per_buffer = [int(((t >> 17) == k).sum()) for k in range(3)]
    assert per_buffer == [215, 52, 0]
    pos = t - 238
    assert pos[:5].tolist() == [794, 1918, 2552, 4196, 4235]
    assert hashlib.sha256(pos.astype("<i8").tobytes()).hexdigest().startswith("63573bbb8af89e26")


def test_known_answer_frames(checker_libs):
    # README.md:151 and dump1090.c:2460: both have syndrome 0
    lib = C.oracle_lib()
    lib.oracle_checksum.restype = ctypes.c_uint32
    for hx in ("8D451E8B99019699C00B0A81F36E", "8D4B969699155600E87406F5B69F"):
        b = bytes.fromhex(hx)
        assert lib.oracle_checksum(b, 112) == 0
        assert synth.modes_parity(b[:11]) == int.from_bytes(b[11:], "big")
        for bit in (5, 40, 111):
            assert lib.oracle_checksum(synth.flip_bits(b, [bit]), 112) != 0


@needs_ref
def test_crc_table_matches_reference(checker_libs):
    # a single set data bit b has checksum == the reference's table entry b
    tab = (ctypes.c_uint32 * 112)()
    C.oracle_lib().oracle_crc_table(tab)
    ref = C.ref_lib()
    ref.ref_checksum.restype = ctypes.c_uint32
    for b in range(88):
        msg = bytearray(14)
        msg[b >> 3] = 0x80 >> (b & 7)
        assert ref.ref_checksum(bytes(msg), 112) == tab[b]
    assert tab[87] == 0xFFF409 and all(tab[b] == 0 for b in range(88, 112))


def test_magnitude_is_strictly_monotone_in_squared_amplitude(checker_libs):
    """The scan kernel compares squared amplitudes instead of magnitudes; that is exact
    iff round(360*sqrt(n)) is strictly increasing over reachable n = i*i+q*q."""
    lut = (ctypes.c_uint16 * 16641)()
    C.oracle_lib().oracle_maglut(lut)
    by_n = {}
    for i in range(129):
        for q in range(129):
            by_n.setdefault(i * i + q * q, set()).add(lut[i * 129 + q])
    assert all(len(v) == 1 for v in by_n.values())
    ns = sorted(by_n)
    ms = [next(iter(by_n[n])) for n in ns]
    assert all(a < b for a, b in zip(ms, ms[1:]))
    assert max(ms) == 65167


@needs_ref
def test_decode_bytes_matches_reference(checker_libs):
    rng = synth.Counter(99)
    ref, orc = C.ref_lib(), C.oracle_lib()
    for k in range(300):
        df = [17, 17, 18, 11, 4, 5, 20, 21, 0, 16][k % 10]
        body = bytes(rng.below(256) for _ in range(10 if df >= 16 else 3))
        frame = synth.make_frame(df, rng.below(8), body)
        flips = [rng.below(len(frame) * 8) for _ in range(k % 3)]
        frame = synth.flip_bits(frame, flips).ljust(14, b"\0")
        for aggressive in (0, 1):
            a, b = C.Msg(), C.Msg()
            ref.ref_decode_bytes(frame, 1, aggressive, ctypes.byref(a))
            orc.oracle_decode_bytes(frame, 1, aggressive, ctypes.byref(b))
            assert C.msg_fields(a) == C.msg_fields(b)
