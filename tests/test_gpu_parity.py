"""-m gpu: the CUDA path, through the C ABI, against the oracle (bit-exact)."""
import numpy as np
import pytest

import checker as C
from dump1090_b200 import api, synth

pytestmark = pytest.mark.gpu

FLAG_SETS = [dict(), dict(aggressive=1), dict(fix=0), dict(check_crc=0), dict(check_crc=0, aggressive=1),
             dict(drop_eof=1), dict(fix=0, drop_eof=1)]


import streams as S

# all frame-evaluation kernels: thread per candidate with both attempts in one walk (whole or half
# windows staged), thread per candidate with two passes (two codings of the per-bit loops), warp per candidate
EVAL_VARIANTS = ["serial", "warp", "lean", "fused", "fused2"]


def _dec_kw(kw):
    return dict(fix_errors=kw.get("fix", 1), aggressive=kw.get("aggressive", 0), check_crc=kw.get("check_crc", 1),
                drop_eof_buffer=kw.get("drop_eof", 0))


def _fields(msgs):
    return [C.msg_fields(m, with_pos=True) for m in msgs]


def _streams():
    yield "modes1", C.modes1()
    for seed in (1, 2, 3):
        yield f"traffic{seed}", synth.random_traffic(300000, 400, seed)
    yield "grid", synth.df17_grid(280000, 700, 5)


def _nasty_streams():
    """Demodulator corner cases (tests/streams.py): tri-state first bits and copied-bit runs, weak
    pairs, and first attempts that fail exactly at j == 0 of a buffer (dump1090.c:1660)."""
    yield "ties", S.tie_rich(11)
    yield "ties_weak", S.tie_rich(12, levels=(0, 0, 1, 3, 30))
    yield "retry_at_j0", S.retry_at_buffer_start()


STREAMS = dict(_streams())
NASTY = dict(_nasty_streams())
ALL_STREAMS = {**STREAMS, **NASTY}


@pytest.mark.parametrize("name", list(STREAMS))
@pytest.mark.parametrize("kw", FLAG_SETS, ids=lambda k: "-".join(f"{a}{b}" for a, b in k.items()) or "default")
def test_decode_matches_oracle(name, kw, gpu_decoder_factory, checker_libs):
    data = STREAMS[name]
    exp, exp_stats = C.oracle_decode(data, **kw)
    dec = gpu_decoder_factory(**_dec_kw(kw))
    got = dec.decode(data)
    assert [m.raw_line() for m in got] == [m.hexline() for m in exp]
    assert _fields(got) == _fields(exp)
    assert list(dec.stats().values()) == exp_stats


def _check_candidates(data, aggressive, dec):
    import torch
    nbuf = data.size // api.BUFFER_BYTES + 1
    padded = np.full(nbuf * api.BUFFER_BYTES, 127, dtype=np.uint8)
    padded[: data.size] = data
    exp = C.oracle_scan_candidates(data, fix=1, aggressive=aggressive, cap=400000)
    exp_arr = np.frombuffer(b"".join(bytes(c) for c in exp), dtype=api.CANDIDATE_DTYPE)
    d = torch.from_numpy(padded).cuda()
    dec.detect_device(d.data_ptr(), nbuf)
    cands, tiles = dec.detect_fetch(nbuf)
    order = np.concatenate([np.arange(o, o + c) for o, c in tiles] or [np.zeros(0, int)]).astype(int)
    assert cands.size == exp_arr.size
    # compare raw record bytes (numpy does not preserve struct padding across fancy indexing)
    got = cands.view(np.uint8).reshape(-1, 56)[order]
    want = exp_arr.view(np.uint8).reshape(-1, 56)
    assert np.array_equal(got[:, :8], want[:, :8]), "candidate positions differ"
    bad = np.nonzero((got != want).any(axis=1))[0]
    assert bad.size == 0, f"{bad.size} of {want.shape[0]} records differ, first at {bad[0]}: {got[bad[0]].tolist()} != {want[bad[0]].tolist()}"
    return want.shape[0]


@pytest.mark.parametrize("name", list(ALL_STREAMS))
@pytest.mark.parametrize("aggressive", [0, 1])
@pytest.mark.parametrize("variant", EVAL_VARIANTS)
def test_candidates_match_oracle(name, aggressive, variant, gpu_decoder_factory, checker_libs, monkeypatch):
    """Scan + frame-evaluation kernels: candidate set and both evaluated passes, record for record.
    All frame-evaluation kernels (thread per candidate, the default; warp per candidate; thread per
    candidate with the leaner per-bit loops), incl. the tie-rich streams and the j == 0 retries."""
    monkeypatch.setenv("MODES_EVAL_VARIANT", variant)
    _check_candidates(ALL_STREAMS[name], aggressive, gpu_decoder_factory(aggressive=aggressive))


@pytest.mark.parametrize("variant", EVAL_VARIANTS)
def test_candidates_random_alphabets(variant, gpu_decoder_factory, checker_libs, monkeypatch):
    """24 small streams with random amplitude alphabets, noise and saturation through the kernels
    themselves (the same cases the host shim checks on CPU)."""
    monkeypatch.setenv("MODES_EVAL_VARIANT", variant)
    total = 0
    decs = {a: gpu_decoder_factory(aggressive=a) for a in (0, 1)}
    for case, levels, data in S.random_alphabet_cases():
        for aggressive in (1, 0):
            total += _check_candidates(data, aggressive, decs[aggressive])
    assert total > 5000


@pytest.mark.parametrize("name", list(NASTY))
@pytest.mark.parametrize("kw", [dict(), dict(aggressive=1), dict(check_crc=0, aggressive=1)],
                         ids=lambda k: "-".join(f"{a}{b}" for a, b in k.items()) or "default")
def test_nasty_streams_decode(name, kw, gpu_decoder_factory, checker_libs):
    data = NASTY[name]
    exp, exp_stats = C.oracle_decode(data, cap=400000, **kw)
    dec = gpu_decoder_factory(**_dec_kw(kw))
    got = dec.decode(data)
    assert [m.raw_line() for m in got] == [m.hexline() for m in exp]
    assert _fields(got) == _fields(exp)
    assert list(dec.stats().values()) == exp_stats


def test_magnitude_matches_oracle(gpu_decoder_factory, checker_libs):
    dec = gpu_decoder_factory()
    data = C.modes1()
    assert np.array_equal(dec.magnitude(data), C.oracle_magnitude(data))
    # every (I, Q) byte pair
    allpairs = np.stack(np.meshgrid(np.arange(256), np.arange(256), indexing="ij"), -1).astype(np.uint8).ravel()
    assert np.array_equal(dec.magnitude(allpairs), C.oracle_magnitude(allpairs))


def test_chunked_feed_is_invariant(gpu_decoder_factory, checker_libs):
    data = C.modes1()
    dec = gpu_decoder_factory(max_batch_bytes=api.BUFFER_BYTES)
    whole = [m.raw_line() for m in dec.decode(data)]
    for chunk in (1000, 262144, 300001):
        assert [m.raw_line() for m in dec.decode(data, chunk=chunk)] == whole
    assert len(whole) == 147
