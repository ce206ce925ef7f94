"""-m gpu: the device CRC repair against the reference, exhaustively on the hex door and on the air.

The hex door (modes_decode_frames: eval_frames_kernel's warp crc_and_fix, which has no CPU build)
sees every 24-bit syndrome of a long and a short frame, with and without `aggressive`, and the
whole repair corpus (tests/repair_corpus.py) with the address cache carried through the batch.
The corpus on the air (repair_stream) goes through the whole decoder and is compared with the
reference's own decode, not only with the oracle; test_gpu_parity.py and test_gpu_resolve.py run
the same streams through every frame-evaluation kernel and the device resolve."""
import ctypes
import time

import numpy as np
import pytest

import checker as C
import repair_corpus as R
from dump1090_b200 import api
from test_repair_oracle import FIX_SETS, STREAMS, check_coverage, check_invariants

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not C.have_ref(), reason="oracle/_ref not built")]

CHUNK = 1 << 18
MSG_BYTES = ctypes.sizeof(api.Message)
# least coverage of a repair stream's messages per (fix, aggressive): see test_repair_oracle
STREAM_FLOORS = {
    (1, 0): dict(single=2000, pair=0, miscorrection=2500, df11_df_bit=80, iid=100),
    (1, 1): dict(single=2000, pair=45000, miscorrection=11000, df11_df_bit=600, iid=50),
    (0, 0): dict(single=0, pair=0, miscorrection=0, df11_df_bit=0, iid=150),
}


def _column(raw, name):
    off = getattr(C.Msg, name).offset
    return raw[:, off: off + 4].copy().view(np.int32).ravel()


@pytest.mark.parametrize("aggressive", [0, 1])
@pytest.mark.parametrize("base", ["df17a", "df11a"])
def test_hex_door_sweeps_every_syndrome(base, aggressive, gpu_decoder_factory, checker_libs):
    """base ^ S for every S != 0 (S = 0 would announce the address, and later DF11 residuals
    below 80 would then be accepted with an interrogator id): bytes, crc, crcok and errorbit."""
    table = C.ref_error_table()
    dec = gpu_decoder_factory(fix_errors=1, aggressive=aggressive)
    t0 = time.perf_counter()
    nfixed = np.zeros(3, dtype=np.int64)
    for s, frames in R.sweep_chunks(R.BASES[base], CHUNK, with_zero=False):
        out = dec.decode_frames(frames)
        raw = np.frombuffer(out, dtype=np.uint8).reshape(-1, MSG_BYTES)
        w_msg, w_crc, w_err, w_nf = R.model_repair(table, frames, 1, aggressive, s)
        crc, crcok, err = _column(raw, "crc"), _column(raw, "crcok"), _column(raw, "errorbit")
        bad = np.flatnonzero((raw[:, :14] != w_msg).any(axis=1) | (crc != w_crc) | (crcok != (w_crc == 0)) | (err != w_err))
        assert bad.size == 0, f"{bad.size} syndromes differ, first S = {s[bad[0]]:#08x}: {raw[bad[0], :14].tolist()} " \
                              f"crc {crc[bad[0]]} errorbit {err[bad[0]]} vs {w_msg[bad[0]].tolist()} {w_crc[bad[0]]} {w_err[bad[0]]}"
        nfixed += np.bincount(w_nf, minlength=3)
    print(f"hex door {base} aggressive={aggressive}: {nfixed[1]} single-bit, {nfixed[2]} two-bit repairs of "
          f"2^24 - 1 syndromes in {time.perf_counter() - t0:.1f} s")
    long_ = len(R.BASES[base]) == 14
    assert nfixed[1] == (107 if long_ else 56)
    assert nfixed[2] == (0 if not aggressive else 5671 if long_ else 1540)


@pytest.mark.parametrize("fix,aggressive", FIX_SETS)
def test_hex_door_corpus_equals_reference(fix, aggressive, gpu_decoder_factory, checker_libs):
    """The whole corpus in one batch through a fresh context: every field as the reference's
    decodeModesMessage gives it, the address cache carried from frame to frame (the iid block)."""
    items = R.corpus()
    frames = R.frames_array(items)
    want = C.ref_decode_frames(frames, fix=fix, aggressive=aggressive)
    got = gpu_decoder_factory(fix_errors=fix, aggressive=aggressive).decode_frames(frames)
    bad = [i for i in range(len(items)) if C.msg_fields(got[i]) != C.msg_fields(want[i])]
    assert not bad, f"{len(bad)} frames differ, first {items[bad[0]][1]}: {C.msg_fields(got[bad[0]])} != {C.msg_fields(want[bad[0]])}"
    check_invariants(items, got)
    check_coverage(items, got, fix, aggressive, "hex door")


@pytest.mark.parametrize("name", list(STREAMS))
@pytest.mark.parametrize("kw", [dict(), dict(aggressive=1), dict(fix=0), dict(check_crc=0, aggressive=1)],
                         ids=lambda k: "-".join(f"{a}{b}" for a, b in k.items()) or "default")
def test_repair_stream_decode_equals_reference(name, kw, gpu_decoder_factory, checker_libs):
    """The decoder on the air against the reference's own decode: lines, fields and statistics
    (single_bit_fix and two_bits_fix included)."""
    data = STREAMS[name]()
    want, want_stats = C.ref_decode(data, cap=400000, **kw)
    dec = gpu_decoder_factory(fix_errors=kw.get("fix", 1), aggressive=kw.get("aggressive", 0),
                              check_crc=kw.get("check_crc", 1))
    got = dec.decode(data)
    assert [m.raw_line() for m in got] == [m.hexline() for m in want]
    assert [C.msg_fields(m) for m in got] == [C.msg_fields(m) for m in want]
    assert list(dec.stats().values()) == want_stats
    items = R.corpus()
    slot_items = [items[(m.sample_pos - 40 + R.SLOT // 2) // R.SLOT] for m in got]
    cov = R.coverage(slot_items, got)
    print(f"{name} {kw}: {cov}, stats single_bit_fix {want_stats[6]} two_bits_fix {want_stats[7]}")
    floors = STREAM_FLOORS[(kw.get("fix", 1), kw.get("aggressive", 0))]
    low = {k: (cov[k], v) for k, v in floors.items() if cov[k] < v}
    assert not low, f"coverage below its floor (got, floor): {low}"
