"""-m gpu: a decode context's buffers grow on demand and are released once.  The hex door's staging
grows without touching the device resolve's address cache; a context that has grown for a dense
stream decodes as a fresh one does; a multi-GPU front counts the launches of its GPUs where they
happen, a repeated batch included."""
import numpy as np
import pytest

import checker as C
from dump1090_b200 import api, synth

pytestmark = pytest.mark.gpu

BUF = api.BUFFER_BYTES
NS = BUF // 2                             # samples per buffer
ALL_FEATURES = dict(signal=True, arrival=True, levels=True, recover=True, weak_preambles=True)


def traffic():
    return synth.random_traffic(NS * 9 + 5000, 1500, 77, n_aircraft=20)


def sparse_buffers(n):
    """n whole buffers of ordinary traffic."""
    data = synth.random_traffic(NS * n, 120 * n, 31)
    assert data.size == n * BUF
    return data


def periodic_preambles(nsamples):
    """A preamble every 15 samples: more candidates than the default capacity (one per 64 samples)."""
    hi = np.tile(np.array([1, 0, 1, 0, 0, 0, 0, 1, 0, 1, 0, 0, 0, 0, 0], np.uint8), -(-nsamples // 15))[:nsamples]
    out = np.full(2 * nsamples, 127, np.uint8)
    out[0::2] = 127 + 100 * hi
    return out


def weak_windows(n_buffers, seed=5):
    """A window every 30 samples that passes the weak-preamble test and fails the reference's: more weak
    positions than a context's first weak list (one per 512 samples + 4096) holds."""
    rng = np.random.default_rng(seed)
    amps = np.zeros(30)
    amps[[0, 2, 7, 9]] = 40
    amps[3] = 45                                                          # the reference's test fails
    for i, bit in enumerate([1, 0, 0, 1, 0]):                             # DF 18
        amps[16 + 2 * i + (1 - bit)] = 30
    data = np.full(n_buffers * BUF, 127, np.uint8)
    for s in range(0, n_buffers * NS - 30, 30):
        data[2 * s: 2 * s + 60: 2] = (127 + amps + rng.integers(0, 2, 30)).astype(np.uint8)
    return data


def dense_stream():
    return np.concatenate([periodic_preambles(4 * NS), weak_windows(4), synth.fleet_at(8, 1500, 2008)[0]])


def outcome(dec, data):
    """Everything a decode with every switch on reports."""
    got = dec.decode(data)
    return ([bytes(m) for m in got], dec.stats(), dec.recovery_stats(), dec.weak_recovery_stats(),
            dec.take_levels().tobytes())


def test_hex_door_then_device_resolve(gpu_decoder_factory, checker_libs):
    """The hex door's staging grows twice between decodes with the device resolve; every decode still
    equals the oracle, and the hex door equals that of a context with the host resolve."""
    data = traffic()
    exp, exp_stats = C.oracle_decode(data, cap=400000)
    frames = np.resize(np.array([list(m.msg) for m in exp], np.uint8), (5000, 14))
    dec = gpu_decoder_factory(gpu_resolve=1)
    host = gpu_decoder_factory()

    def decode_both():
        got = dec.decode(data)
        assert [m.raw_line() for m in got] == [m.hexline() for m in exp]
        assert [C.msg_fields(m, with_pos=True) for m in got] == [C.msg_fields(m, with_pos=True) for m in exp]
        assert list(dec.stats().values()) == exp_stats
        host.decode(data)                     # the same address cache for the next hex-door call

    decode_both()
    for n in (1, 100, 5000):
        got = dec.decode_frames(frames[:n])
        assert bytes(got) == bytes(host.decode_frames(frames[:n])), n
        decode_both()
    dec.close()


@pytest.mark.parametrize("max_batch_bytes", [0, 2 * BUF], ids=["one_batch", "two_buffer_batches"])
def test_growth_across_features(max_batch_bytes, gpu_decoder_factory, checker_libs):
    """One context with every switch on decodes a sparse stream, a stream that overflows its candidate
    and weak lists, and the sparse stream again: each as a fresh context does."""
    sparse, dense = traffic(), dense_stream()
    # the dense stream's whole buffers, as one batch, overflow both lists
    nbuf = dense.size // BUF
    probe = gpu_decoder_factory()
    probe.detect_host(np.ascontiguousarray(dense[: nbuf * BUF]).ctypes.data, nbuf, None)
    probe.weak_device()
    assert probe.detect_wait() > nbuf * NS // 64 + 4096
    assert probe.weak_fetch()[0] > nbuf * NS // 512 + 4096
    cfg = dict(ALL_FEATURES, max_batch_bytes=max_batch_bytes)
    dec = gpu_decoder_factory(**cfg)
    for data in (sparse, dense, sparse):
        assert outcome(dec, data) == outcome(gpu_decoder_factory(**cfg), data)


def test_multi_gpu_launch_count(gpu_decoder_factory, checker_libs):
    """With one-buffer batches dealt to two GPU contexts (on one device, reused round-robin), a sparse
    stream costs two launches per buffer, the EOF buffer included; a batch repeated after an overflow
    costs more."""
    n = 5
    sparse = sparse_buffers(n)
    dec = gpu_decoder_factory(n_gpus=2, max_batch_bytes=BUF)
    one = gpu_decoder_factory(max_batch_bytes=BUF)
    before = dec.launch_count()
    got = dec.decode(sparse)
    assert dec.launch_count() - before == 2 * (n + 1)
    assert [bytes(m) for m in got] == [bytes(m) for m in one.decode(sparse)]
    dense = np.concatenate([periodic_preambles(NS * 2 + 5000), synth.fleet_at(8, 1500, 2008)[0]])
    before = dec.launch_count()
    got = dec.decode(dense)
    assert dec.launch_count() - before > 2 * (dense.size // BUF + 1), "no repeated batch was counted"
    assert [bytes(m) for m in got] == [bytes(m) for m in one.decode(dense)]
