"""-m gpu: a slot's batches alternate between two counter sets, each zeroed by the scan of the batch
before it, and the count reaches the host without a copy.  A batch denser than the candidate buffers
(one candidate per 64 samples) is repeated on the other set: its records must equal those of a batch
that had room, whatever ran on the slot before it and after it, on the detect path (where
modes_detect_publish_count copies the set of the batch just queued) and in a two-slot streaming decode."""
import numpy as np
import pytest

import checker as C
from dump1090_b200 import api, synth

pytestmark = pytest.mark.gpu

BUF = api.BUFFER_BYTES
NS = BUF // 2
NBUF = 4


def periodic_preambles(nsamples):
    """A preamble every 15 samples: about four times the default candidate capacity."""
    hi = np.tile(np.array([1, 0, 1, 0, 0, 0, 0, 1, 0, 1, 0, 0, 0, 0, 0], np.uint8), -(-nsamples // 15))[:nsamples]
    out = np.full(2 * nsamples, 127, np.uint8)
    out[0::2] = 127 + 100 * hi
    return out


def canonical(cands, tiles):
    """Records in position order (the scan lists tiles in no fixed order) and the per-tile counts."""
    return cands[np.argsort(cands["t"], kind="stable")].tobytes(), tiles["count"].tobytes()


def test_detect_batches_alternate_counter_sets(gpu_decoder_factory):
    import torch
    sparse = synth.random_traffic(NS * NBUF, 120 * NBUF, 31)[: NBUF * BUF]
    dense = periodic_preambles(NBUF * NS)
    carry = bytes(sparse[-api.CARRY_BYTES:])
    d = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in (("sparse", sparse), ("dense", dense))}

    # with room: caller-supplied buffers five times the default capacity
    cap = NBUF * NS // 8
    recs = torch.zeros(cap * 56, dtype=torch.uint8, device="cuda")
    tiles = torch.zeros(api.tiles_for(NBUF) * 8, dtype=torch.uint8, device="cuda")
    roomy = gpu_decoder_factory()
    want = {}
    for k in d:
        roomy.detect_device(d[k].data_ptr(), NBUF, carry, recs.data_ptr(), cap, tiles.data_ptr())
        want[k] = canonical(*roomy.detect_fetch(NBUF))
    default_cap = NBUF * NS // 64 + 4096
    assert len(want["dense"][0]) // 56 > default_cap > len(want["sparse"][0]) // 56

    # default buffers: the first dense batch overflows and is repeated; batches are queued back to back
    dec = gpu_decoder_factory()
    pub = torch.zeros(4, dtype=torch.int32, device="cuda")
    launches = []
    for k in ("sparse", "dense", "sparse", "dense", "dense", "sparse"):
        before = dec.launch_count()
        dec.detect_device(d[k].data_ptr(), NBUF, carry)
        dec.publish_count(pub.data_ptr())
        got = canonical(*dec.detect_fetch(NBUF))
        launches.append(dec.launch_count() - before)
        assert got == want[k], k
        torch.cuda.synchronize()
        assert int(pub[0]) == len(got[0]) // 56, k
    assert launches == [2, 4, 2, 2, 2, 2], "the first dense batch alone is repeated"

    # queued without waiting: only the last batch's count is read
    for k in ("dense", "sparse", "dense"):
        dec.detect_device(d[k].data_ptr(), NBUF, carry)
    assert canonical(*dec.detect_fetch(NBUF)) == want["dense"]


@pytest.mark.parametrize("batch_buffers", [1, 2])
def test_stream_overflow_on_one_slot(batch_buffers, gpu_decoder_factory, checker_libs):
    """Sparse and dense batches on the two slots of a streaming decode: the batches that overflow are
    repeated on their own slot's other set, and the decode equals the oracle, fresh and grown."""
    data = np.concatenate([synth.random_traffic(NS * 3, 360, 8)[: 3 * BUF], periodic_preambles(3 * NS + 5000),
                           synth.fleet_at(8, 1500, 2008)[0]])
    exp, st = C.oracle_decode(data, check_crc=0, cap=400000)
    dec = gpu_decoder_factory(check_crc=0, max_batch_bytes=batch_buffers * BUF)
    for _ in range(2):
        got = dec.decode(data)
        assert [m.raw_line() for m in got] == [m.hexline() for m in exp]
        assert list(dec.stats().values()) == st
