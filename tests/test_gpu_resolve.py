"""-m gpu: modes_config.gpu_resolve = 1 — the order-dependent half (retry/skip state machine, ICAO
address cache, statistics) replayed on the device, one warp per reference buffer, instead of on
the host (SURVEY.md §8(f) item 4).  Same messages, fields and statistics as the oracle and as the
host resolve, whatever the batch size (the address cache is handed from batch to batch on the GPU)."""
import hashlib

import numpy as np
import pytest

import checker as C
import repair_corpus as R
import streams as S
from dump1090_b200 import api, synth

pytestmark = pytest.mark.gpu

FLAG_SETS = [dict(), dict(aggressive=1), dict(fix=0), dict(check_crc=0), dict(check_crc=0, aggressive=1), dict(drop_eof=1)]


def _dec_kw(kw):
    return dict(fix_errors=kw.get("fix", 1), aggressive=kw.get("aggressive", 0), check_crc=kw.get("check_crc", 1),
                drop_eof_buffer=kw.get("drop_eof", 0))


def _streams():
    yield "modes1", C.modes1()
    yield "traffic", synth.random_traffic(131072 * 9 + 5000, 1500, 77, n_aircraft=20)
    yield "dense_fleet", synth.random_traffic(131072 * 30, 9000, 5, n_aircraft=60)
    yield "grid", synth.df17_grid(280000, 700, 5)
    yield "ties", S.tie_rich(11)
    yield "retry_at_j0", S.retry_at_buffer_start()
    # a preamble every 60 samples: within the documented density, but with check_crc = 0 nearly every
    # candidate delivers both attempts
    yield "dense_ties", S.tie_rich(21, n_frames=17800, levels=(0, 40, 100), period=60)
    yield from S.chain_streams()
    yield "repair0", R.repair_stream(0.0)                              # tests/repair_corpus.py
    yield "repair_frac", R.repair_stream(R.RETRY_FRAC)


STREAMS = dict(_streams())


@pytest.mark.parametrize("name", list(STREAMS))
@pytest.mark.parametrize("kw", FLAG_SETS, ids=lambda k: "-".join(f"{a}{b}" for a, b in k.items()) or "default")
def test_device_resolve_matches_oracle(name, kw, gpu_decoder_factory, checker_libs):
    data = STREAMS[name]
    exp, exp_stats = C.oracle_decode(data, cap=400000, **kw)
    dec = gpu_decoder_factory(gpu_resolve=1, **_dec_kw(kw))
    got = dec.decode(data)
    assert [m.raw_line() for m in got] == [m.hexline() for m in exp]
    assert [C.msg_fields(m, with_pos=True) for m in got] == [C.msg_fields(m, with_pos=True) for m in exp]
    assert list(dec.stats().values()) == exp_stats


def _batch_cases():
    """(batch buffers, stream), named by the batch size (0: the default) and the stream unless it is
    the traffic stream."""
    for name in ["traffic"] + list(S.CHAINS):
        for b in (1, 3, 8, 64, 0):
            bid = str(b) if b else "default"
            yield pytest.param(b, name, id=bid if name == "traffic" else f"{bid}-{name}")


@pytest.mark.parametrize("batch_buffers,name", list(_batch_cases()))
def test_device_resolve_cache_crosses_batches(batch_buffers, name, gpu_decoder_factory, checker_libs):
    """Small batches: an address announced in one batch validates address/parity replies in later
    ones — the cache is handed from batch to batch on the device, across the two pipeline slots.
    The chains (tests/streams.address_chain) also run through whole batches longer than the fixed
    rounds of guessing (batch_buffers >= 8, the default size)."""
    if name == "traffic":
        data = synth.random_traffic(131072 * 21 + 999, 5000, 13, n_aircraft=25)
    else:
        data = STREAMS[name]
    exp, st = C.oracle_decode(data, cap=100000)
    assert any(m.msgtype in (0, 4, 5, 16, 20, 21) for m in exp) or name == "chain_df11_iid"
    dec = gpu_decoder_factory(gpu_resolve=1, max_batch_bytes=batch_buffers * api.BUFFER_BYTES)
    for chunk in (None, 300001):
        got = dec.decode(data, chunk=chunk)
        assert [m.raw_line() for m in got] == [m.hexline() for m in exp]
        assert [C.msg_fields(m, with_pos=True) for m in got] == [C.msg_fields(m, with_pos=True) for m in exp]
        assert list(dec.stats().values()) == st


def test_device_resolve_full_size_equals_host_resolve(gpu_decoder_factory, checker_libs):
    """BASELINE.json configs[1] size: the 481 691 messages of the tiled capture, device resolve vs host resolve."""
    data = synth.tile_to(C.modes1(), 1 << 30)
    digests = []
    for gpu in (0, 1):
        dec = gpu_decoder_factory(fix_errors=0, gpu_resolve=gpu)
        out = dec.set_output_array(700000)
        dec.reset(); dec.rearm_output(); dec.process(data); dec.finish()
        n = dec.output_count()
        a = np.frombuffer(out, dtype=np.uint8, count=n * 200).reshape(n, 200)
        digests.append((n, hashlib.sha256(a.tobytes()).hexdigest(), dec.stats()))
        dec.set_output_array(0)
    assert digests[0][0] == 481691
    assert digests[0] == digests[1]
