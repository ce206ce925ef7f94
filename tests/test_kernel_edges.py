"""The recovery (K6), signal (K4) and level (K5) kernels on the constructed edge cases that their host
builds (tests/host_shim/) already pass.

The host builds compile the plain-loop branches of the core headers and replace the recovery warp's
arg-min rounds, solution count, owner-lane ballot and mask shuffle with a sort and a loop; decoded
streams rarely or never reach AMBIGUOUS records, solutions owned by lanes 1..31, all-equal windows, the
signal pass's two record lengths, its capacity clamp or the second trip of its grid-stride loop.  So
here the same corpora (tests/edge_corpora.py) run through the shipped kernels, through the device
harness tests/device_shim/kernels_device.cu (linked against the product's own objects) and through
the public entry points, and every record is compared byte for byte with the numpy restatements:
recover_model.restate, test_signal.expected_signal and test_levels.buffer_sums."""
import ctypes
import subprocess

import numpy as np
import pytest

import checker as C
import edge_corpora as E
import recover_model as R
import test_levels as TL
import test_signal as TS
from dump1090_b200 import api, synth

pytestmark = pytest.mark.gpu

ROOT = C.ROOT
DSHIM = ROOT / "tests" / "_build" / "libkernels_device.so"
BUF = api.BUFFER_BYTES
NS = BUF // 2                             # samples per buffer
HALO = 240                                # virtual samples before the body: 2 unused + 238 carried
LAST_J = 131069                           # the last position the scan visits in a buffer
OUT_SENTINEL = 0x5A                       # dev_recover fills its output with it before the launch
MAX_WARPS_PER_SM = 64                     # sm_90: a one-wave grid has at most this many warps per SM
FOUND, AMBIGUOUS, INELIGIBLE = api.RECOVER_FOUND, api.RECOVER_AMBIGUOUS, api.RECOVER_INELIGIBLE


@pytest.fixture(scope="module")
def dshim():
    subprocess.run(["make", "-s", "dshim"], cwd=ROOT, check=True)
    lib = ctypes.CDLL(str(DSHIM))
    u32, p = ctypes.c_uint32, ctypes.c_void_p
    lib.dev_error.restype = ctypes.c_char_p
    lib.dev_sm_count.restype = ctypes.c_int
    lib.dev_recover.argtypes = [p, u32, p, p, u32, u32, u32, p]
    lib.dev_signal.argtypes = [p, u32, p, p, u32, u32, u32]
    lib.dev_sweeps.argtypes = [p]
    assert lib.dev_sm_count() > 0, lib.dev_error()
    return lib


# ---------------------------------------------------------------- batches and placements


class Batch:
    """A batch of n_buffers buffers as the kernels address it: the virtual sample array of the carry
    block (2 unused samples, then the 238 carried) followed by the body, as I/Q bytes."""

    def __init__(self, n_buffers):
        self.n_buffers = n_buffers
        self.virt = np.full(2 * (HALO + n_buffers * NS), 127, dtype=np.uint8)

    def put(self, t, win):
        """The window of record t: its 224 samples from virtual index t + 18 on."""
        v = 2 * (int(t) + 18)
        self.virt[v: v + win.size] = win

    def args(self):
        body, carry = self.virt[2 * HALO:], self.virt[4: 2 * HALO]
        return body, carry


def placements(n, placement):
    """Batches (n_buffers, window indices, t) that place windows 0..n-1 of a corpus, none overlapping."""
    if placement in ("even", "odd"):                                      # mid-buffer, both sample alignments
        t = 1000 + (placement == "odd") + 226 * np.arange(n)
        return [(int(t[-1] + 2) // NS + 1, np.arange(n), t)]
    if placement == "carry":                                              # the window starts in the carry block
        return [(1, np.array([k]), np.array([(37 * k) % 222])) for k in range(n)]
    if placement == "last_j":                                             # j = 131069 of every buffer of a batch
        out = []
        for s in range(0, n, 8):
            idx = np.arange(s, min(n, s + 8))
            out.append((idx.size, idx, NS * np.arange(idx.size) + LAST_J))
        return out
    raise ValueError(placement)


PLACEMENTS = ["even", "odd", "carry", "last_j"]


def batch_of(wins, n_buffers, idx, t):
    b = Batch(n_buffers)
    for i, ti in zip(idx, t):
        b.put(ti, wins[i])
    return b


def dev_recover(lib, batch, t, capacity=None, counter=None):
    t = np.ascontiguousarray(t, dtype=np.int64)
    out = np.zeros(t.size, dtype=api.RECOVERED_DTYPE)
    body, carry = batch.args()
    rc = lib.dev_recover(body.ctypes.data, batch.n_buffers, carry.ctypes.data, t.ctypes.data, t.size,
                         t.size if capacity is None else capacity, t.size if counter is None else counter,
                         out.ctypes.data)
    assert rc == 0, lib.dev_error()
    return out


def dev_signal(lib, batch, records, capacity=None, counter=None):
    recs = np.ascontiguousarray(records).copy()
    body, carry = batch.args()
    rc = lib.dev_signal(body.ctypes.data, batch.n_buffers, carry.ctypes.data, recs.ctypes.data, recs.size,
                        recs.size if capacity is None else capacity, recs.size if counter is None else counter)
    assert rc == 0, lib.dev_error()
    return recs


def assert_same(got, want, what):
    assert got.size == want.size, what
    for f in ("msg", "status", "nflips", "signal", "pad"):
        d = got[f] != want[f]
        bad = np.flatnonzero(d.any(axis=1) if d.ndim > 1 else d)
        assert bad.size == 0, f"{what}: field {f} differs at {bad[:5].tolist()}"


def test_harness_refuses_windows_outside_the_batch(dshim):
    """Nothing runs for a window outside [0, 240 + N) or a capacity beyond the arrays."""
    b = Batch(1)
    body, carry = b.args()
    out = np.zeros(2, dtype=api.RECOVERED_DTYPE)
    recs = np.zeros(2, dtype=api.CANDIDATE_DTYPE)
    for t in ((0, NS - 1), (0, -1), (NS + 5, 0)):
        tt = np.array(t, dtype=np.int64)
        assert dshim.dev_recover(body.ctypes.data, 1, carry.ctypes.data, tt.ctypes.data, 2, 2, 2, out.ctypes.data) != 0
        recs["t"] = tt
        assert dshim.dev_signal(body.ctypes.data, 1, carry.ctypes.data, recs.ctypes.data, 2, 2, 2) != 0
    tt = np.array([0, NS - 2], dtype=np.int64)                            # the last window that fits
    assert dshim.dev_recover(body.ctypes.data, 1, carry.ctypes.data, tt.ctypes.data, 2, 2, 2, out.ctypes.data) == 0
    assert dshim.dev_recover(body.ctypes.data, 1, carry.ctypes.data, tt.ctypes.data, 2, 3, 2, out.ctypes.data) != 0
    assert dshim.dev_recover(body.ctypes.data, 0, carry.ctypes.data, tt.ctypes.data, 2, 2, 2, out.ctypes.data) != 0


# ---------------------------------------------------------------- recovery records


@pytest.fixture(scope="module")
def recover_corpora():
    c = dict(E.recover_random_windows())
    c["frames"] = E.recover_frame_windows()[0]
    c["confident"] = E.recover_confident_windows()
    c["ambiguity"] = E.recover_ambiguity_windows()
    return {k: (np.ascontiguousarray(v, dtype=np.uint8).reshape(-1, 448), E.restated(v)) for k, v in c.items()}


def owner_lanes(wins, rec):
    """The high five subset bits of each FOUND record's solution (the warp lane that owns it), from
    the record's flips and the ten positions of the definition."""
    m = R.magnitudes(wins.reshape(-1)).reshape(-1, 224)
    a, c = m[:, 0::2], m[:, 1::2]
    hard = np.packbits((a > c).astype(np.uint8), axis=1)
    keys = (np.abs(a - c)[:, 5:112] << 7) | np.arange(5, 112)[None, :]
    pos = np.sort(keys, axis=1)[:, :api.RECOVER_BITS] & 127
    flipped = np.unpackbits(hard ^ rec["msg"], axis=1)
    lanes = []
    for r in np.flatnonzero(rec["status"] == FOUND):
        mask = sum(1 << k for k in range(api.RECOVER_BITS) if flipped[r, pos[r, k]])
        assert int(flipped[r].sum()) == bin(mask).count("1") == int(rec["nflips"][r])
        lanes.append(mask >> 5)
    return np.array(lanes, dtype=np.int64)


@pytest.mark.parametrize("placement", PLACEMENTS)
def test_recovery_records_on_constructed_corpora(placement, dshim, recover_corpora):
    got = {}
    for name, (wins, want) in recover_corpora.items():
        rec = np.zeros(len(wins), dtype=api.RECOVERED_DTYPE)
        for nb, idx, t in placements(len(wins), placement):
            rec[idx] = dev_recover(dshim, batch_of(wins, nb, idx, t), t)
        assert_same(rec, want, f"{name}, {placement}")
        got[name] = rec
    # the corpora reached the branches only the device compiles
    amb = got["ambiguity"]
    assert ((amb["status"] == AMBIGUOUS) & (amb["nflips"] == 3)).sum() >= 155
    lanes = np.concatenate([owner_lanes(recover_corpora[n][0], got[n]) for n in got])
    assert (lanes > 0).sum() >= 80 and (lanes == 0).sum() >= 100            # solved by lanes 1..31 and by lane 0
    for df in (17, 18):
        assert (got[f"all_equal_df{df}"]["status"] != INELIGIBLE).all()
    assert (got["confident"]["status"][40:] == INELIGIBLE).all()


def test_recovery_capacity_and_volume(dshim, recover_corpora):
    wins = np.concatenate([recover_corpora["frames"][0], recover_corpora["ambiguity"][0]])
    want = np.concatenate([recover_corpora["frames"][1], recover_corpora["ambiguity"][1]])
    (nb, idx, t), = placements(len(wins), "odd")
    b = batch_of(wins, nb, idx, t)
    n = t.size
    for capacity, counter in ((n, n), (n // 3, n + 1000), (n // 3, 2 ** 32 - 1), (n, 17), (n, 0), (0, n)):
        got = dev_recover(dshim, b, t, capacity, counter)
        k = min(capacity, counter)
        assert_same(got[:k], want[:k], (capacity, counter))
        assert (got.view(np.uint8).reshape(n, 20)[k:] == OUT_SENTINEL).all(), (capacity, counter)
    # the same windows under many t, shuffled: the grid-stride loop makes several trips
    rng = np.random.default_rng(21)
    reps = -(-4 * MAX_WARPS_PER_SM * dshim.dev_sm_count() // n)
    sel = rng.permutation(np.tile(np.arange(n), reps))
    got = dev_recover(dshim, b, t[sel])
    assert got.size > 4 * MAX_WARPS_PER_SM * dshim.dev_sm_count()
    assert_same(got, want[sel], "volume")


# ---------------------------------------------------------------- signal fields

COMBOS = np.array([(56, 112), (112, 56), (0, 112), (56, 0), (0, 0)])     # bits of attempt 0 / 1 (0: not decoded)
SHORT_DF = np.array([0, 4, 5, 11, 15, 22, 24, 31, 128, 255], dtype=np.uint8)
LONG_DF = np.array([16, 17, 18, 19, 20, 21], dtype=np.uint8)


@pytest.fixture(scope="module")
def signal_corpus():
    """All signal windows, and the signal of each for 56 and 112 bits."""
    wins = np.concatenate([w for _, w in E.signal_windows(np.random.default_rng(77))])
    mag = TS.magnitudes(wins.reshape(-1))
    pos = 224 * np.arange(len(wins)) - 16                                  # pos + 16: the window's first sample
    sig = {b: TS.expected_signal(mag, pos, np.full(len(wins), b)) for b in (56, 112)}
    assert sig[112].max() == 65167 and sig[112].min() == 0
    return wins, sig


def signal_records(rng, t, combos):
    """Candidate records at t, random bytes elsewhere, with the attempts decoded as 56- or 112-bit
    frames or not at all (0)."""
    n = t.size
    recs = np.frombuffer(rng.integers(0, 256, n * 56, dtype=np.uint8).tobytes(), dtype=api.CANDIDATE_DTYPE).copy()
    recs["t"] = t
    b = recs.view(np.uint8).reshape(n, 56)
    for k in (0, 1):
        bits = combos[:, k]
        b[:, 22 + 24 * k] = np.where(bits == 112, rng.choice(LONG_DF, n), rng.choice(SHORT_DF, n))
        flags = b[:, 23 + 24 * k]
        b[:, 23 + 24 * k] = np.where(bits > 0, flags | api.EVAL_DECODED, flags & ~np.uint8(api.EVAL_DECODED))
    return recs


def expected_records(before, widx, combos, sig, limit=None):
    """The records after the pass: halfwords 13 / 25 (pass[k].signal) of decoded attempts set, every
    other byte as before; records from `limit` on untouched."""
    want = before.copy()
    h = want.view(np.uint16).reshape(want.size, 28)
    n = want.size if limit is None else min(limit, want.size)
    for k in (0, 1):
        bits = combos[:n, k]
        val = np.where(bits == 112, sig[112][widx[:n]], sig[56][widx[:n]])
        sel = np.flatnonzero(bits > 0)
        h[sel, 13 + 12 * k] = val[sel]
    return want


def assert_records_equal(got, want, what):
    g, w = got.view(np.uint8).reshape(-1, 56), want.view(np.uint8).reshape(-1, 56)
    bad = np.flatnonzero((g != w).any(axis=1))
    assert bad.size == 0, f"{what}: {bad.size} records differ, first {bad[:5].tolist()}"


@pytest.mark.parametrize("placement", PLACEMENTS)
def test_signal_fields_on_constructed_corpora(placement, dshim, signal_corpus):
    wins, sig = signal_corpus
    rng = np.random.default_rng(len(placement))
    n_dec = 0
    for nb, idx, t in placements(len(wins), placement):
        b = batch_of(wins, nb, idx, t)
        # every window under every attempt combination, in a shuffled order
        order = rng.permutation(idx.size * len(COMBOS))
        widx, combos = np.repeat(idx, len(COMBOS))[order], np.tile(COMBOS, (idx.size, 1))[order]
        recs = signal_records(rng, np.repeat(t, len(COMBOS))[order], combos)
        got = dev_signal(dshim, b, recs)
        assert_records_equal(got, expected_records(recs, widx, combos, sig), placement)
        n_dec += int((combos > 0).sum())
    assert n_dec == 6 * len(wins)


def test_signal_capacity_and_second_trip(dshim, signal_corpus):
    wins, sig = signal_corpus
    rng = np.random.default_rng(5)
    (nb, idx, t), = placements(len(wins), "odd")
    b = batch_of(wins, nb, idx, t)
    n = 4 * len(wins)
    widx = rng.integers(0, len(wins), n)
    combos = COMBOS[rng.integers(0, len(COMBOS), n)]
    recs = signal_records(rng, t[widx], combos)
    for capacity, counter in ((n // 3, n + 5), (n // 3, 2 ** 32 - 1), (n, 100), (n, 0), (0, n)):
        got = dev_signal(dshim, b, recs, capacity, counter)
        assert_records_equal(got, expected_records(recs, widx, combos, sig, min(capacity, counter)), (capacity, counter))
    # more records than 32 per warp of a full wave: the grid-stride loop comes back
    n = 32 * MAX_WARPS_PER_SM * dshim.dev_sm_count() * 5 // 2
    widx = rng.integers(0, len(wins), n)
    combos = COMBOS[rng.integers(0, len(COMBOS), n)]
    recs = signal_records(rng, t[widx], combos)
    assert_records_equal(dev_signal(dshim, b, recs), expected_records(recs, widx, combos, sig), "second trip")


# ---------------------------------------------------------------- the core headers' device build


def test_exhaustive_sweeps_of_the_device_arithmetic(dshim):
    out = np.zeros(4, dtype=np.uint64)
    assert dshim.dev_sweeps(out.ctypes.data) == 0, dshim.dev_error()
    assert out[0] == 0, f"isqrt32: {int(out[0])} wrong, first at x = {int(out[1])}"
    assert out[2] == 0, f"sample words: {int(out[2])} wrong, first at w = {int(out[3]):#010x}"


# ---------------------------------------------------------------- the level kernel


def level_records(bufs):
    want = np.zeros(len(bufs), dtype=api.LEVEL_DTYPE)
    for k, b in enumerate(bufs):
        want[k]["buffer"], want[k]["n_samples"] = k, NS
        want[k]["clipped"], want[k]["sum_mag"], want[k]["sum_power"], want[k]["peak"] = TL.buffer_sums(b)
    return want


def test_levels_on_constructed_buffers(gpu_decoder_factory):
    import torch
    rng = np.random.default_rng(31)
    i, q = np.meshgrid(np.arange(256), np.arange(256), indexing="ij")
    pairs = np.stack([i.ravel(), q.ravel()], axis=1).astype(np.uint8)     # all 65536 (I, Q) samples
    # sample p of rotation r sits in slot (p + r) % 8 of a 16-byte load: rotations 0..7 over 4 buffers
    bufs = [np.concatenate([np.roll(pairs, 2 * b, axis=0), np.roll(pairs, 2 * b + 1, axis=0)]).reshape(-1) for b in range(4)]
    # 254 and 1 are flagged by the cheap rail test and never clipped, in every byte lane
    rails = [rng.choice(np.array([1, 254], dtype=np.uint8), size=BUF), np.full(BUF, 254, np.uint8), np.full(BUF, 1, np.uint8)]
    rails += [np.roll(np.tile(np.array([254, 1, 127, 127], dtype=np.uint8), NS // 2), s) for s in range(4)]
    bufs += rails + [b for _, b in E.level_buffers(rng)]
    want = level_records(bufs)
    assert (want["clipped"][4: 4 + len(rails)] == 0).all() and want["clipped"][:4].tolist() == [2 * 1020] * 4
    dec = gpu_decoder_factory()
    flat = torch.from_numpy(np.concatenate(bufs)).cuda()
    dec.levels_device(flat.data_ptr(), len(bufs))
    TL.assert_records(dec.levels_fetch(), want, "constructed buffers")
    # more buffers than resident CTAs (3 per SM), at the pool's stride of two buffers; pads on the rail
    n = 512
    assert n > 3 * torch.cuda.get_device_properties(0).multi_processor_count
    kinds = [lambda: rng.integers(0, 256, BUF, dtype=np.uint8),
             lambda: rng.choice(np.array([0, 1, 126, 127, 128, 254, 255], dtype=np.uint8), size=BUF),
             lambda: np.clip(rng.normal(127, 1 + rng.integers(0, 40), size=BUF).round(), 0, 255).astype(np.uint8),
             lambda: rng.choice(np.array([1, 127, 254], dtype=np.uint8), size=BUF)]
    many = [kinds[k % 4]() for k in range(n)]
    strided = np.zeros((2 * n, BUF), dtype=np.uint8)
    strided[1::2] = np.stack(many)
    d = torch.from_numpy(strided.reshape(-1)).cuda()
    dec.levels_device(d.data_ptr() + BUF, n, 2 * BUF)
    TL.assert_records(dec.levels_fetch(), level_records(many), "512 buffers at stride 2")


# ---------------------------------------------------------------- end to end through the scan


def _scannable(pos):
    j = (pos + 238) % NS
    return pos >= 0 and j < NS - 2


def planted_stream(wins, n_buffers, seed):
    """A stream of n_buffers buffers (+ a short tail) with the windows planted behind preambles
    (pulses at 0, 2, 7, 9; samples 4-5 and 11-14 quiet).  Some preambles sit at the first positions of
    a buffer (their window straddles the seam) or at the last position the scan visits in a buffer.
    Returns (stream, planted positions)."""
    rng = np.random.default_rng(seed)
    special = []
    for k in range(1, n_buffers):
        if k % 2:
            special.append(NS * k - 238 + [0, 1, 7, 100, 221][(k // 2) % 5])
        else:
            special.append(NS * k - 238 - (NS - LAST_J))                  # j = 131069 of buffer k - 1
    limit = NS * n_buffers
    pos, cur = [], 0
    while len(pos) + len(special) < len(wins):
        if cur + 240 > limit:
            raise ValueError("windows do not fit")
        if _scannable(cur) and all(cur + 240 <= s or s + 240 <= cur for s in special):
            pos.append(cur)
            cur += 240 + int(rng.integers(0, 600))
        else:
            cur += 1
    pos = np.array(sorted(pos + special[: len(wins)]), dtype=np.int64)
    data = np.full(2 * limit + 1000, 127, dtype=np.uint8)
    s = data.reshape(-1, 2)
    for p, w in zip(pos, wins):
        s[p + np.array([0, 2, 7, 9]), 0] = 227
        data[2 * (p + 16): 2 * (p + 16) + 448] = w
    return data, pos


def _padded(data):
    nbuf = data.size // BUF + 1
    p = np.full(nbuf * BUF, 127, dtype=np.uint8)
    p[: data.size] = data
    return p, nbuf


def _check_records(data, cands, rec, planted, what):
    t = cands["t"]
    missing = set(planted.tolist()) - set((t - 238).tolist())
    assert not missing, f"{what}: no candidate at {sorted(missing)[:5]}"
    assert_same(rec, R.restate_records(data, t), what)
    mag = TS.magnitudes(data)
    decoded = 0
    for k in (0, 1):
        p = cands["p"][:, k]
        dec = (p["flags"] & api.EVAL_DECODED) != 0
        bits = np.where((p["msgtype"] >= 16) & (p["msgtype"] <= 21), 112, 56)
        want = np.where(dec, TS.expected_signal(mag, t - 238, bits), 0)
        assert np.array_equal(p["signal"].astype(np.int64), want), (what, k)
        decoded += int(dec.sum())
    assert decoded > 0


def test_planted_corpus_through_the_scan(gpu_decoder_factory, recover_corpora):
    wins = np.concatenate([w for w, _ in recover_corpora.values()])
    data, planted = planted_stream(wins, 12, 41)
    padded, nbuf = _padded(data)
    # one batch
    dec = gpu_decoder_factory(aggressive=1, signal=True)
    launches = dec.launch_count()
    dec.detect_host(padded.ctypes.data, nbuf, None)
    dec.recover_device()
    cands, _ = dec.detect_fetch(nbuf)
    rec = dec.recover_fetch()
    assert dec.launch_count() - launches == 4
    _check_records(data, cands, rec, planted, "one batch")
    # one buffer per batch, each with the previous buffer's last 238 samples as its carry
    parts_c, parts_r = [], []
    for k in range(nbuf):
        buf = np.ascontiguousarray(padded[k * BUF: (k + 1) * BUF])
        dec.detect_host(buf.ctypes.data, 1, padded[k * BUF - api.CARRY_BYTES: k * BUF].tobytes() if k else None)
        dec.recover_device()
        c, _ = dec.detect_fetch(1)
        parts_r.append(dec.recover_fetch())
        c["t"] += NS * k
        parts_c.append(c)
    cands_b, rec_b = np.concatenate(parts_c), np.concatenate(parts_r)
    assert sorted(cands_b["t"].tolist()) == sorted(cands["t"].tolist())
    _check_records(data, cands_b, rec_b, planted, "one buffer per batch")
    ts = (planted + 238) % NS
    assert (ts < 222).sum() >= 5 and (ts == LAST_J).sum() >= 5


# ---------------------------------------------------------------- a repeated batch


def test_recovery_and_signal_after_a_repeated_batch(gpu_decoder_factory, checker_libs):
    """A stream dense enough to overflow the candidate buffers makes the decode repeat the batch with
    larger buffers; the recovery records and signal fields equal the restatements all the same."""
    data = np.concatenate([TL._periodic([1, 0, 1, 0, 0, 0, 0, 1, 0, 1, 0, 0, 0, 0, 0], NS * 2 + 5000),
                           synth.fleet_at(8, 1500, 2008)[0]])
    padded, nbuf = _padded(data)
    dec = gpu_decoder_factory(check_crc=0, signal=True)
    launches = dec.launch_count()
    dec.detect_host(padded.ctypes.data, nbuf, None)
    dec.recover_device()
    cands, _ = dec.detect_fetch(nbuf)
    rec = dec.recover_fetch()
    assert dec.launch_count() - launches > 4, "the batch was not repeated"
    _check_records(data, cands, rec, np.zeros(0, dtype=np.int64), "repeated batch")
    assert (rec["status"] != INELIGIBLE).sum() > 100
    # the streaming decode, one buffer per batch: the CPU path's messages, signals as restated
    kw = dict(check_crc=0)
    cpu = R.cpu_decode(data, kw, signal=True)
    on = gpu_decoder_factory(recover=True, signal=True, max_batch_bytes=BUF, **R.flag_cfg(kw))
    got = on.decode(data)
    assert on.launch_count() > 4 * (data.size // BUF + 1), "no batch was repeated"
    assert len(got) == len(cpu[0]) and on.recovery_stats() == cpu[2] and on.stats() == cpu[1]
    for g, w in zip(got, cpu[0]):
        if w.recovered:
            assert bytes(g) == bytes(w)
        else:
            c = g.copy()
            c.signal = 0
            assert bytes(c) == bytes(w)
    TS._assert_signals([m for m in got if not m.recovered], data)
    assert cpu[2]["delivered"] > 0
