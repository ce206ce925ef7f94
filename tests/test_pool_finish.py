"""Finite captures through the receiver pool (modes_pool_finish / modes_pool_finish_device): after a receiver is
finished with its tail, everything the pool delivered for it equals the single-stream decode of all its bytes,
the EOF buffer included unless drop_eof_buffer is set.

CPU tests check the finish schedule (tests/pool_finish_model.py) against the streaming models and modes_finish's
rule, the refusals that need no device, the exports, and the C host's --pool refusals.  GPU tests check the
contract against the oracle and the single stream, device-fed tails, the edge shapes, the C host's --pool and
api.decode_captures."""
import copy
import ctypes
import subprocess

import numpy as np
import pytest

import checker as C
import input_format_model as M
import pool_finish_model as FM
import resample_model as RM
from dump1090_b200 import api, synth

ROOT = C.ROOT
EXE = ROOT / "dump1090-b200"
BUF = api.BUFFER_BYTES
B = api.BUFFER_SAMPLES
R2, R24 = 2_000_000, 2_400_000
FLAG_SETS = [dict(), dict(aggressive=1), dict(fix=0), dict(check_crc=0)]   # test_pool's four
DEFAULT_SHIFT = {"uc8": None, "sc16": 8, "sc16q11": 4}


# ---------------------------------------------------------------- CPU: the schedule


def _tails(rate, fmt, n_calls):
    full = FM.buffer_bytes(fmt)
    t = {0, 1, 2, 3, 4, 5, 1001, 1002, 77_777, full - 1, full}
    t0 = FM.two_pair_tails(rate, fmt, n_calls)
    if t0 is not None:
        t |= {t0, max(t0 - 1, 0), min(t0 + 1, full)}
    return sorted(t)


@pytest.mark.parametrize("rate", [R2, R24])
@pytest.mark.parametrize("fmt", ["uc8", "sc16"])
def test_finish_schedule_is_the_streaming_finish(rate, fmt):
    """For every receiver state of 0-12 calls and tails of 0-5 bytes, odd and even lengths, a full buffer and
    the lengths about the first that makes two pairs: the model's pairs are the buffers the streaming models
    (16-bit conversion, then the resampler at 2.4 MS/s) have not yet decoded whole, up to modes_finish's EOF
    buffer; at most one is whole and it goes in batch 1."""
    full = FM.buffer_bytes(fmt)
    conv = M.Streaming(8) if fmt != "uc8" else None
    rs = RM.Streaming() if rate == R24 else None
    emitted, piece = 0, np.full(full, 127, np.uint8)
    two = 0
    for c in range(13):
        submitted, in_total = FM.state_after(rate, c)
        assert submitted == emitted // B, c
        for t in _tails(rate, fmt, c):
            cv, r2 = copy.deepcopy(conv), copy.deepcopy(rs)
            tail = piece[:t]
            uc8 = cv.feed(tail) if cv else tail
            if r2 is not None:                             # finish_held's rule: the EOF buffer holds sample N_out
                total = emitted + (r2.feed(uc8).size + r2.finish().size) // 2
                eof = total // B
            else:                                          # modes_finish: the EOF buffer is the bytes pending
                pending = uc8.size if t < full else 0
                eof = emitted // B + (t == full)
                total = eof * B + (pending + 1) // 2
            for drop in (False, True):
                pairs = FM.finish_pairs(rate, fmt, submitted, in_total, t, drop)
                last = eof + (0 if drop else 1)
                assert [b for _, b, _ in pairs] == list(range(submitted, last)), (c, t, drop)
                whole = [p for p in pairs if p[0] == 1]
                assert len(whole) <= 1 and all(p[2] == B for p in whole), (c, t)
                if not drop:
                    assert pairs[-1] == (2, eof, total - eof * B), (c, t)
            if len(FM.finish_pairs(rate, fmt, submitted, in_total, t)) == 2:
                two += 1
                t0 = FM.two_pair_tails(rate, fmt, c)
                assert t0 is not None and t >= t0, (c, t)
        # the next whole buffer
        uc8 = conv.feed(piece) if conv else piece
        emitted += (rs.feed(uc8).size if rs else uc8.size) // 2
    assert two > 0                                   # a full tail at 2 MHz; several states at 2.4 MS/s
    if rate == R2:
        assert FM.two_pair_tails(rate, fmt, 3) == full


def test_refusals_without_a_device():
    with api.ReceiverPool(3, max_batch=2) as pool:
        pool.set_input_format(2, "sc16")
        with pytest.raises(ValueError, match="at most 262144"):
            pool.finish([0], [np.zeros(BUF + 1, np.uint8)])
        with pytest.raises(ValueError, match="at most 524288"):
            pool.finish([2], [np.zeros(2 * BUF + 1, np.uint8)])
        with pytest.raises(RuntimeError, match="out of range"):
            pool.finish([3], [np.zeros(5, np.uint8)])
        with pytest.raises(RuntimeError, match="listed twice"):
            pool.finish([1, 1], [np.zeros(5, np.uint8)] * 2)
        with pytest.raises(RuntimeError, match="created for 2"):
            pool.finish([0, 1, 2], [np.zeros(5, np.uint8)] * 3)
        with pytest.raises(ValueError, match="tails for"):
            pool.finish([0, 1], [np.zeros(5, np.uint8)])
        # the C call refuses a tail longer than the receiver's buffer itself, before any device is touched
        L = api.lib()
        for r, n in ((0, BUF + 1), (2, 2 * BUF + 1)):
            tail = np.zeros(n, np.uint8)
            ids = np.array([r], np.uint32)
            sizes = np.array([n], np.uintp)
            ptrs = (ctypes.c_void_p * 1)(tail.ctypes.data)
            assert L.modes_pool_finish(pool._h, api._ptr(ids), ptrs, api._ptr(sizes), 1, api.POOL_SINK_FN(0), None) == -1
            assert "more than its buffer" in L.modes_pool_last_error(pool._h).decode()
        ids = np.array([0], np.uint32)
        sizes = np.array([7], np.uintp)
        ptrs = (ctypes.c_void_p * 1)(None)
        assert L.modes_pool_finish(pool._h, api._ptr(ids), ptrs, api._ptr(sizes), 1, api.POOL_SINK_FN(0), None) == -1
        assert "null pointer" in L.modes_pool_last_error(pool._h).decode()


def test_symbols_exported():
    L = api.lib()
    for s in ("modes_pool_finish", "modes_pool_finish_device"):
        assert s in api.EXPORTS
        assert hasattr(L, s)
    out = subprocess.run(["nm", "-D", "--defined-only", str(ROOT / "dump1090_b200" / "libmodes_b200.so")],
                         capture_output=True, text=True, check=True).stdout
    assert " modes_pool_finish\n" in out and " modes_pool_finish_device\n" in out


@pytest.mark.parametrize("flags,named", [
    (["--beast"], "--beast"), (["--sbs"], "--sbs"), (["--aircraft-json"], "--aircraft-json"),
    (["--levels"], "--levels"), (["--spectrum"], "--spectrum"), (["--carrier"], "--carrier"),
    (["--recover"], "--recover"), (["--recover-weak"], "--recover-weak"), (["--gpu-resolve"], "--gpu-resolve"),
    (["--gpus", "2"], "--gpus"), (["--chunk", "4096"], "--chunk"), (["--input-offset", "0"], "--input-offset"),
    (["--beast", "--arrival"], "--beast")])
def test_host_pool_refuses_unsupported_flags(flags, named, tmp_path):
    f = tmp_path / "a.bin"
    f.write_bytes(bytes(1000))
    r = subprocess.run([str(EXE), "--pool", "--ifile", str(f), "--ifile", str(f), *flags], capture_output=True, text=True)
    assert r.returncode == 1 and r.stdout == ""
    assert f"--pool cannot be combined with {named}" in r.stderr


def test_host_pool_refuses_stdin_and_rates(tmp_path):
    f = tmp_path / "a.bin"
    f.write_bytes(bytes(1000))
    r = subprocess.run([str(EXE), "--pool", "--ifile", str(f), "--ifile", "-"], capture_output=True, text=True)
    assert r.returncode == 1 and "--ifile - (stdin)" in r.stderr
    for rate in ("4000000", "10000000"):
        r = subprocess.run([str(EXE), "--pool", "--ifile", str(f), "--sample-rate", rate], capture_output=True, text=True)
        assert r.returncode == 1 and "--pool takes --sample-rate 2000000 or 2400000" in r.stderr
    r = subprocess.run([str(EXE), "--pool", "--ifile", str(tmp_path / "missing.bin")], capture_output=True, text=True)
    assert r.returncode == 1 and "Opening data file" in r.stderr


# ---------------------------------------------------------------- GPU: the contract


class Rx:
    """A receiver's finite capture: n_whole buffers and a tail of `tail` bytes of its format at its rate."""

    def __init__(self, fmt, rate, n_whole, tail, seed, shift=None, snr=16):
        self.fmt, self.rate, self.shift = fmt, rate, shift
        self.full = FM.buffer_bytes(fmt)
        self.n_whole, self.tail = n_whole, tail
        nbytes = n_whole * self.full + tail
        s = shift if shift is not None else DEFAULT_SHIFT[fmt]
        samples = nbytes // (2 if fmt == "uc8" else 4) + 1
        nframes = samples * R2 // rate // 400 + 3
        if fmt == "uc8" and rate == R2:
            x = synth.random_traffic(samples, samples // 700 + 3, seed=seed)
        elif fmt == "uc8":
            x = synth.fleet_at_rate(snr, nframes, seed, sample_rate=rate)[0]
        else:
            x = synth.fleet_at_rate(snr, nframes, seed, sample_rate=rate, dtype="sc16", scale=float(1 << s))[0]
        assert x.size >= nbytes
        self.x = np.ascontiguousarray(x[:nbytes])

    def buf(self, k):
        return self.x[k * self.full: (k + 1) * self.full]

    def tail_bytes(self):
        return self.x[self.n_whole * self.full:]

    def decoded(self):
        """The 2 MHz bytes of the whole stream (N_out samples)."""
        y = self.x if self.fmt == "uc8" else M.convert(self.x, self.shift if self.shift is not None else DEFAULT_SHIFT[self.fmt])
        return RM.resample(y) if self.rate == R24 else y

    def buffers(self, drop=False):
        """modes_pool_buffers after the finish."""
        submitted, in_total = FM.state_after(self.rate, self.n_whole)
        return submitted + len(FM.finish_pairs(self.rate, self.fmt, submitted, in_total, self.tail, drop))


def _seven():
    """2 MHz and 2.4 MS/s, UC8, SC16 and SC16Q11, with tails of a whole buffer, odd, 16-bit partial samples,
    and the 2.4 MS/s tails that make two pairs."""
    t24 = FM.two_pair_tails(R24, "uc8", 4)
    t24s = FM.two_pair_tails(R24, "sc16q11", 7)
    return [Rx("uc8", R2, 3, 77_777, seed=101),
            Rx("uc8", R24, 4, t24 + 1001, seed=31, snr=20),
            Rx("sc16", R2, 2, 2 * BUF - 2, seed=41, snr=14),
            Rx("sc16q11", R2, 4, 2 * BUF, seed=42, snr=20),
            Rx("sc16", R24, 3, 100_003, seed=43, snr=20),
            Rx("sc16q11", R24, 7, t24s + 6, seed=44, snr=14),
            Rx("sc16q11", R2, 2, 1, seed=45, shift=2, snr=10)]


def _pool(rxs, **kw):
    pool = api.ReceiverPool(len(rxs), **kw)
    for r, rx in enumerate(rxs):
        pool.set_input_rate(r, rx.rate)
        pool.set_input_format(r, rx.fmt, rx.shift)
    return pool


def _feed(pool, rxs, max_batch, seed, device=False, tails=None):
    """Every receiver's whole buffers, not in lock step, in calls of up to max_batch receivers; then every
    receiver finished with its tail (tails: other tails, as arrays or tensors), in calls of up to max_batch."""
    rng = np.random.default_rng(seed)
    nxt = [0] * len(rxs)
    dev = None
    if device:
        import torch
        dev = [torch.from_numpy(rx.x).cuda() for rx in rxs]
    while any(nxt[r] < rx.n_whole for r, rx in enumerate(rxs)):
        ids = [r for r, rx in enumerate(rxs) if nxt[r] < rx.n_whole and rng.random() < 0.7]
        rng.shuffle(ids)
        for lo in range(0, len(ids), max_batch):
            part = ids[lo: lo + max_batch]
            src = [(dev[r] if device else rxs[r].x)[nxt[r] * rxs[r].full: (nxt[r] + 1) * rxs[r].full] for r in part]
            pool.ingest(part, src)
            for r in part:
                nxt[r] += 1
    order = list(range(len(rxs)))
    rng.shuffle(order)
    for lo in range(0, len(order), max_batch):
        part = order[lo: lo + max_batch]
        pool.finish(part, [tails[r] if tails is not None else rxs[r].tail_bytes() for r in part])


def _same(got, want, what):
    assert len(got) == len(want), (what, len(got), len(want))
    for k, (g, w) in enumerate(zip(got, want)):
        assert bytes(g) == bytes(w), (what, k, g.raw_line(), w.raw_line())


def _single(rx, **kw):
    return api.Decoder(input_rate=rx.rate, input_format=rx.fmt, input_shift=rx.shift, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("drop", [0, 1], ids=["eof", "drop_eof"])
@pytest.mark.parametrize("kw", FLAG_SETS, ids=lambda k: "-".join(f"{a}{b}" for a, b in k.items()) or "default")
def test_finished_pool_equals_oracle(kw, drop, checker_libs):
    rxs = _seven()
    cfg = dict(fix_errors=kw.get("fix", 1), aggressive=kw.get("aggressive", 0), check_crc=kw.get("check_crc", 1),
               drop_eof_buffer=drop)
    with _pool(rxs, max_batch=5, **cfg) as pool:
        _feed(pool, rxs, 5, seed=6)
        for r, rx in enumerate(rxs):
            assert pool.buffers(r) == rx.buffers(drop), r
            msgs, stats = C.oracle_decode(rx.decoded(), drop_eof=drop, **kw)
            got = pool.take(r)
            assert len(got) > 10, r
            assert [m.raw_line() for m in got] == [m.hexline() for m in msgs], f"receiver {r}"
            assert [C.msg_fields(m, with_pos=True) for m in got] == [C.msg_fields(m, with_pos=True) for m in msgs], r
            assert list(pool.stats(r).values()) == stats, f"receiver {r}"


SWITCHES = [dict(signal=True), dict(arrival=True, signal=True), dict(carrier=True), dict(levels=True),
            dict(spectrum=True), dict(recover=True), dict(recover=True, weak_preambles=True)]


@pytest.mark.gpu
@pytest.mark.parametrize("sw", SWITCHES, ids=["signal", "arrival", "carrier", "levels", "spectrum", "recover", "weak"])
def test_every_switch_equals_single_stream(sw):
    rxs = _seven()
    with _pool(rxs, max_batch=5, **sw) as pool:
        _feed(pool, rxs, 5, seed=10)
        for r, rx in enumerate(rxs):
            with _single(rx, **sw) as dec:
                _same(pool.take(r), dec.decode(rx.x), (sw, r))
                assert pool.stats(r) == dec.stats(), (sw, r)
                assert pool.buffers(r) == rx.buffers(), (sw, r)
                if sw.get("levels"):
                    lv = pool.take_levels(r)
                    assert list(lv["buffer"]) == list(range(pool.buffers(r))), r
                    assert lv["n_samples"][-1] == (rx.decoded().size + 1) // 2 % B, r
                    assert np.array_equal(lv, dec.take_levels()), r
                if sw.get("spectrum"):
                    sp = pool.take_spectra(r)
                    assert len(sp) == pool.buffers(r), r
                    assert np.array_equal(sp, dec.take_spectra()), r
                if sw.get("recover"):
                    assert pool.recovery_stats(r) == dec.recovery_stats(), r
                    assert pool.weak_recovery_stats(r) == dec.weak_recovery_stats(), r


def _odd_tails(rxs):
    """Odd tails for every receiver, shorter than its buffer."""
    return [rx.x[rx.n_whole * rx.full:][: (rx.tail if rx.tail % 2 else rx.tail - 1) if rx.tail else 0] for rx in rxs]


def _at_end(t, torch):
    """The bytes t in a CUDA tensor that ends where they end, 16-byte aligned."""
    pad = 16 * 3
    a = torch.empty(pad + t.size, dtype=torch.uint8, device="cuda")
    v = a[pad:]
    if t.size:
        v.copy_(torch.from_numpy(np.ascontiguousarray(t)))
    assert v.data_ptr() % 16 == 0 and v.data_ptr() + t.size == a.data_ptr() + a.numel()
    return v


@pytest.mark.gpu
@pytest.mark.parametrize("sw", [dict(), dict(signal=True, levels=True, spectrum=True, carrier=True, recover=True)],
                         ids=["plain", "switches"])
def test_device_fed_equals_host_fed(sw):
    import torch
    rxs = _seven()
    tails = _odd_tails(rxs)
    assert all(t.size % 2 == 1 for t in tails)
    with _pool(rxs, max_batch=5, **sw) as host, _pool(rxs, max_batch=5, **sw) as devp:
        _feed(host, rxs, 5, seed=12, tails=tails)
        _feed(devp, rxs, 5, seed=12, device=True, tails=[_at_end(t, torch) for t in tails])
        torch.cuda.synchronize()
        for r in range(len(rxs)):
            got = devp.take(r)
            assert got, r
            _same(got, host.take(r), ("device", r))
            assert devp.stats(r) == host.stats(r), r
            assert devp.buffers(r) == host.buffers(r), r
            if sw:
                assert np.array_equal(devp.take_levels(r), host.take_levels(r)), r
                assert np.array_equal(devp.take_spectra(r), host.take_spectra(r)), r
                assert devp.recovery_stats(r) == host.recovery_stats(r), r


@pytest.mark.gpu
def test_never_fed_and_empty_tails():
    """A capture shorter than one buffer, a 0-byte capture, and a 0-byte tail after whole buffers, at both
    rates and formats, with levels (the EOF record counts its real samples)."""
    rxs = [Rx("uc8", R2, 0, 100_001, seed=61), Rx("sc16", R24, 0, 300_001, seed=62), Rx("uc8", R24, 0, 0, seed=63),
           Rx("sc16q11", R2, 0, 0, seed=64), Rx("uc8", R2, 2, 0, seed=65), Rx("sc16", R24, 3, 0, seed=66),
           Rx("uc8", R24, 6, 0, seed=67)]
    with _pool(rxs, max_batch=len(rxs), levels=True) as pool:
        _feed(pool, rxs, len(rxs), seed=14)
        for r, rx in enumerate(rxs):
            with _single(rx, levels=True) as dec:
                _same(pool.take(r), dec.decode(rx.x), r)
                assert pool.stats(r) == dec.stats(), r
                lv = pool.take_levels(r)
                assert np.array_equal(lv, dec.take_levels()), r
                assert len(lv) == pool.buffers(r) == rx.buffers(), r
                assert lv["n_samples"][-1] == (rx.decoded().size + 1) // 2 % B, r


@pytest.mark.gpu
def test_finish_refusals_reset_and_restart():
    a = Rx("uc8", R2, 2, 5_001, seed=71)
    b = Rx("sc16", R24, 3, 12_345, seed=72)
    with api.ReceiverPool(2) as pool:
        pool.submit([0], [a.buf(0)])
        with pytest.raises(RuntimeError, match="in flight"):
            pool.finish([1], [np.zeros(3, np.uint8)])
        pool.collect()
        pool.ingest([0], [a.buf(1)])
        pool.finish([0, 1], [a.tail_bytes(), np.zeros(0, np.uint8)])
        with pytest.raises(RuntimeError, match="after modes_pool_finish; call modes_pool_reset first"):
            pool.ingest([0], [a.buf(0)])
        with pytest.raises(RuntimeError, match="after modes_pool_finish; call modes_pool_reset first"):
            pool.submit([1], [a.buf(0)])
        with pytest.raises(RuntimeError, match="after modes_pool_finish; call modes_pool_reset first"):
            pool.finish([0], [np.zeros(1, np.uint8)])
        for r in range(2):
            with pytest.raises(RuntimeError, match="in progress"):
                pool.set_input_rate(r, R24)
            with pytest.raises(RuntimeError, match="in progress"):
                pool.set_input_format(r, "sc16")
        with _single(a) as dec:
            _same(pool.take(0), dec.decode(a.x), "first stream")
        # a new stream after reset, at another rate and format
        pool.reset(0)
        pool.set_input_rate(0, R24)
        pool.set_input_format(0, "sc16")
        for k in range(b.n_whole):
            pool.ingest([0], [b.buf(k)])
        pool.finish([0], [b.tail_bytes()])
        with _single(b) as dec:
            _same(pool.take(0), dec.decode(b.x), "second stream")
            assert pool.stats(0) == dec.stats()
        assert pool.buffers(0) == b.buffers()


@pytest.mark.gpu
def test_one_finish_of_256_receivers():
    """One finish naming 256 receivers of all six rate/format kinds at max_batch = 256, the tails of every
    length class (0, odd, partial 16-bit samples, whole buffers, two pairs)."""
    kinds = [(f, r) for f in ("uc8", "sc16", "sc16q11") for r in (R2, R24)]
    base = {k: Rx(k[0], k[1], 4, 0, seed=80 + i) for i, k in enumerate(kinds)}
    rxs = []
    for i in range(256):
        fmt, rate = kinds[i % 6]
        full = FM.buffer_bytes(fmt)
        n_whole = (i // 6) % 3
        t0 = FM.two_pair_tails(rate, fmt, n_whole)
        tail = [0, 1, 3, full - 1, full, 4 * (i + 7) + 2, t0 if t0 is not None else 99][(i // 18) % 7]
        rx = copy.copy(base[(fmt, rate)])
        rx.n_whole, rx.tail = n_whole, tail
        rx.x = base[(fmt, rate)].x[: n_whole * full + tail]
        rxs.append(rx)
    decs = {k: _single(base[k], signal=True) for k in kinds}
    try:
        with _pool(rxs, max_batch=256, signal=True) as pool:
            for k in range(2):
                ids = [r for r, rx in enumerate(rxs) if rx.n_whole > k]
                pool.ingest(ids, [rxs[r].buf(k) for r in ids])
            pool.finish(list(range(256)), [rx.tail_bytes() for rx in rxs])
            for r, rx in enumerate(rxs):
                _same(pool.take(r), decs[(rx.fmt, rx.rate)].decode(rx.x), r)
                assert pool.stats(r) == decs[(rx.fmt, rx.rate)].stats(), r
                assert pool.buffers(r) == rx.buffers(), r
    finally:
        for d in decs.values():
            d.close()


# ---------------------------------------------------------------- GPU: the C host and decode_captures


def _run(args):
    r = subprocess.run([str(EXE), *args], capture_output=True, check=True)
    return r.stdout


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,rate", [("uc8", R2), ("sc16", R24)], ids=["uc8-2M", "sc16-2.4M"])
def test_host_pool_equals_single_runs(fmt, rate, tmp_path):
    rxs = [Rx(fmt, rate, 2, 12_345, seed=91), Rx(fmt, rate, 0, 99_999, seed=92), Rx(fmt, rate, 3, 0, seed=93)]
    files = []
    for i, rx in enumerate(rxs):
        f = tmp_path / f"c{i}.bin"
        rx.x.tofile(f)
        files.append(str(f))
    base = ["--sample-rate", str(rate), "--iformat", fmt.upper()]
    for out in (["--raw", "--stats"], [], ["--raw"], ["--onlyaddr"]):
        for drop in ([], ["--drop-eof-buffer"]):
            single = b"".join(_run(["--ifile", f, *base, *out, *drop]) for f in files)
            pooled = _run(["--pool", *sum((["--ifile", f] for f in files), []), *base, *out, *drop])
            assert pooled == single, (out, drop)
            assert single, (out, drop)


@pytest.mark.gpu
def test_decode_captures_equals_decoder(tmp_path):
    rxs = [Rx("uc8", R2, 2, 333, seed=95), Rx("uc8", R2, 0, 0, seed=96), Rx("uc8", R2, 1, 131_071, seed=97),
           Rx("uc8", R2, 3, BUF - 1, seed=98)]
    f = tmp_path / "a.bin"
    rxs[0].x.tofile(f)
    caps = [str(f), rxs[1].x, rxs[2].x, rxs[3].x]
    got = api.decode_captures(caps, max_batch=3, signal=True)
    with api.Decoder(signal=True) as dec:
        for r, rx in enumerate(rxs):
            _same(got[r], dec.decode(rx.x), r)
    rxs = [Rx("sc16", R24, 2, 7_777, seed=99), Rx("sc16", R24, 5, 0, seed=100), Rx("sc16", R24, 0, 1_001, seed=102)]
    got = api.decode_captures([rx.x for rx in rxs], input_rate=R24, input_format="sc16", max_batch=2, drop_eof_buffer=1)
    with api.Decoder(input_rate=R24, input_format="sc16", drop_eof_buffer=1) as dec:
        for r, rx in enumerate(rxs):
            _same(got[r], dec.decode(rx.x), ("sc16", r))
