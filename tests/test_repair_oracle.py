"""CPU (-m "not gpu"): the oracle's CRC repair and address cache against the reference on the repair
corpus (tests/repair_corpus.py), frame by frame through decodeModesMessage and on the air through
the whole demodulator, with the phase-corrected retry carrying repairs."""
import numpy as np
import pytest

import checker as C
import repair_corpus as R
from test_oracle import FLAG_SETS

needs_ref = pytest.mark.skipif(not C.have_ref(), reason="oracle/_ref not built")

FIX_SETS = [(1, 0), (1, 1), (0, 0), (0, 1)]
# least coverage of the corpus per (fix, aggressive): single-bit repairs, two-bit repairs,
# miscorrections, DF11 frames repaired in their DF field, interrogator-id acceptances
MIN_COVERAGE = {
    (1, 0): dict(single=3500, pair=0, miscorrection=2800, df11_df_bit=90, iid=120),
    (1, 1): dict(single=3500, pair=45000, miscorrection=11000, df11_df_bit=600, iid=50),
    (0, 0): dict(single=0, pair=0, miscorrection=0, df11_df_bit=0, iid=150),
    (0, 1): dict(single=0, pair=0, miscorrection=0, df11_df_bit=0, iid=150),
}
STREAMS = {"repair0": lambda: R.repair_stream(0.0), "repair_frac": lambda: R.repair_stream(R.RETRY_FRAC)}


def check_coverage(items, msgs, fix, aggressive, what):
    cov = R.coverage(items, msgs)
    print(f"{what} fix={fix} aggressive={aggressive}: {cov}")
    low = {k: (cov[k], v) for k, v in MIN_COVERAGE[(fix, aggressive)].items() if cov[k] < v}
    assert not low, f"coverage below its floor (got, floor): {low}"
    if not fix:
        assert cov["single"] == cov["pair"] == 0
    if not aggressive:
        assert cov["pair"] == 0
    return cov


def check_invariants(items, msgs):
    """What holds whatever the flags: controls, 3-bit errors and long frames flipped into DF 17/18
    are never repaired; a repaired frame always passes its CRC."""
    for (f, label), m in zip(items, msgs):
        kind, base = label.split("/")[:2]
        never = kind == "flip3" or (kind == "dfbit" and not base.startswith("src11")) or \
            (base.startswith("df") and base[:4] not in ("df11", "df17", "df18"))
        if never:
            assert m.errorbit == -1, label
        if m.errorbit != -1:
            assert m.crcok and m.crc == 0, label


@needs_ref
@pytest.mark.parametrize("fix,aggressive", FIX_SETS)
def test_corpus_oracle_equals_reference(fix, aggressive, checker_libs):
    """oracle_decode_frames == ref_decode_frames on every corpus frame, the address cache carried
    through the batch: every field and the repaired bytes; the oracle's fix counters count the
    reference's repairs."""
    items = R.corpus()
    frames = R.frames_array(items)
    r = C.ref_decode_frames(frames, fix=fix, aggressive=aggressive)
    o, os_ = C.oracle_decode_frames(frames, fix=fix, aggressive=aggressive)
    bad = [i for i in range(len(items)) if C.msg_fields(r[i]) != C.msg_fields(o[i])]
    assert not bad, f"{len(bad)} frames differ, first {items[bad[0]][1]}: {C.msg_fields(r[bad[0]])} != {C.msg_fields(o[bad[0]])}"
    check_invariants(items, r)
    cov = check_coverage(items, r, fix, aggressive, "corpus")
    assert os_ == [0] * 6 + [cov["single"], cov["pair"]]       # the oracle counts the reference's repairs


@needs_ref
@pytest.mark.parametrize("name", list(STREAMS))
@pytest.mark.parametrize("kw", FLAG_SETS, ids=str)
def test_repair_stream_oracle_equals_reference(name, kw, checker_libs):
    data = STREAMS[name]()
    r, rs = C.ref_decode(data, cap=400000, **kw)
    o, os_ = C.oracle_decode(data, cap=400000, **kw)
    assert [C.msg_fields(m) for m in r] == [C.msg_fields(m) for m in o]
    assert rs == os_
    if kw.get("fix", 1):
        assert rs[6] > 3000 and (rs[7] > 40000) == bool(kw.get("aggressive", 0))


def test_repair_stream_retries_carry_repairs(checker_libs):
    """On repair_stream(0) every repair happens in the first attempt; with the fractional offset
    a share of them happens only in the phase-corrected retry (pass[1])."""
    for frac, want_retry in ((0.0, False), (R.RETRY_FRAC, True)):
        cands = C.oracle_scan_candidates(R.repair_stream(frac), fix=1, aggressive=1, cap=400000)
        p1 = np.array([[c.passes[k].nfixed for k in (0, 1)] for c in cands])
        print(f"frac {frac}: {len(cands)} candidates, repairs in pass[0]: {(p1[:, 0] > 0).sum()}, "
              f"in pass[1]: {(p1[:, 1] > 0).sum()} ({(p1[:, 1] == 1).sum()} single, {(p1[:, 1] == 2).sum()} two-bit)")
        assert (p1[:, 0] > 0).sum() > 45000
        if want_retry:
            assert (p1[:, 1] == 1).sum() >= 10 and (p1[:, 1] == 2).sum() >= 2000
        else:
            assert (p1[:, 1] > 0).sum() == 0
