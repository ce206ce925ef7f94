"""Streams fed from device memory (modes_process_device, CUDA tensors in Decoder.process / decode).

Every GPU case feeds one decoder the stream's bytes from device memory and another the same bytes from
host memory, in the same call sizes, and asks for the same output: messages with every field and
sample_pos, statistics, and the level, spectrum, recovery and weak records.  The calls are whole streams
and random odd sizes, so the device pointers start at every alignment mod 16 and calls split buffers,
samples and 16-bit values.
"""
from __future__ import annotations

import types

import numpy as np
import pytest

import checker as C
import input_format_model as IF
import test_input_decimation as TD
import test_input_rate as TR
from dump1090_b200 import api, synth

BUF = api.BUFFER_BYTES
B = api.BUFFER_SAMPLES
FORMATS = {"uc8": None, "sc16": 8, "sc16q11": 4}                 # the shift each 16-bit stream is written at
RATES = (2_000_000, 2_400_000, 4_000_000, 6_000_000, 8_000_000, 10_000_000)
SILENCE = {"uc8": 127, "sc16": 0, "sc16q11": 0}

_inputs = {}


def stream(hz: int, fmt: str, offset: int = 0) -> np.ndarray:
    """A few buffers of random traffic at the rate, sent `offset` Hz off centre, written in the format
    (16-bit: values that convert back to the UC8 bytes at the format's default shift)."""
    key = (hz, fmt, offset)
    if key not in _inputs:
        if offset:
            x, _ = synth.fleet_at_rate(18, 1200, 14, sample_rate=hz, carrier_hz=float(offset))
        elif hz == 2_000_000:
            x = synth.random_traffic(3 * B + 12_345, 400, 11)
        elif hz == 2_400_000:
            x = TR.traffic24(4 * B + 777, 500, 12)
        else:
            x = TD.traffic_at(hz // 2_000_000, "uc8", 3 * B * (hz // 2_000_000) + 999, 13)
        _inputs[key] = x if fmt == "uc8" else IF.to_sc16(x, FORMATS[fmt])
    return _inputs[key]


def max_offset(hz: int) -> int:
    return hz // 2 - 1_000_000 if hz >= 4_000_000 else 0


def odd_sizes(n: int, seed: int, hi: int = 300_000) -> list:
    rng = np.random.default_rng(seed)
    out, left = [], n
    while left:
        k = min(int(rng.integers(0, hi)) | 1, left)
        out.append(k)
        left -= k
    return out


def feed_host(dec, x: np.ndarray, sizes) -> None:
    dec.reset()
    off = 0
    for n in sizes:
        dec.process(x[off: off + n])
        off += n
    dec.finish()


def feed_device(dec, x: np.ndarray, sizes, scribble: bool = False) -> None:
    """The stream from one device copy at its offsets; scribble: each call from its own tensor, overwritten
    with random bytes as soon as the call returns."""
    import torch
    d = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    torch.cuda.synchronize()
    dec.reset()
    off = 0
    for n in sizes:
        if scribble:
            t = d[off: off + n].clone()
            torch.cuda.synchronize()
            dec.process_device_ptr(t.data_ptr(), n)
            t.random_(0, 256)
            torch.cuda.synchronize()
        else:
            dec.process_device_ptr(d.data_ptr() + off, n)
        off += n
    dec.finish()


def results(dec, kw) -> dict:
    r = dict(msgs=[TR.fields(m) for m in dec.take_messages()], stats=dec.stats())
    if kw.get("levels"):
        r["levels"] = dec.take_levels().tobytes()
    if kw.get("spectrum"):
        r["spectra"] = dec.take_spectra().tobytes()
    if kw.get("recover"):
        r["recovery"] = (dec.recovery_stats(), dec.weak_recovery_stats())
    return r


def make(hz, fmt, offset=0, **kw):
    return api.Decoder(input_rate=hz, input_format=fmt, input_offset=offset, **kw)


def compare(hz, fmt, offset, x, size_sets, scribble=False, **kw):
    """The device-fed decoder equals the host-fed one for each call-size list; returns the host results."""
    wants = []
    with make(hz, fmt, offset, **kw) as host, make(hz, fmt, offset, **kw) as dev:
        for sizes in size_sets:
            feed_host(host, x, sizes)
            want = results(host, kw)
            feed_device(dev, x, sizes, scribble)
            got = results(dev, kw)
            assert got.keys() == want.keys()
            for k in want:
                assert got[k] == want[k], (hz, fmt, offset, kw, k, len(sizes))
            wants.append(want)
    return wants


# ---------------------------------------------------------------- GPU: the contract


CONTRACT = [(hz, fmt, 0) for hz in RATES for fmt in FORMATS] + \
           [(hz, fmt, s * max_offset(hz)) for hz, fmt, s in ((4_000_000, "uc8", 1), (6_000_000, "sc16", -1),
                                                              (8_000_000, "sc16q11", 1), (10_000_000, "sc16", -1))]


@pytest.mark.gpu
@pytest.mark.parametrize("drop", (0, 1))
@pytest.mark.parametrize("hz,fmt,offset", CONTRACT)
def test_contract(hz, fmt, offset, drop):
    x = stream(hz, fmt, offset)
    wants = compare(hz, fmt, offset, x, [[x.size], odd_sizes(x.size, hz // 1000 + offset // 1000 + drop)],
                    drop_eof_buffer=drop)
    assert len(wants[0]["msgs"]) > 10, (hz, fmt)


@pytest.mark.gpu
@pytest.mark.parametrize("hz,fmt", [(2_000_000, "uc8"), (10_000_000, "sc16")])
def test_contract_oracle(checker_libs, hz, fmt):
    """The host-fed and device-fed decode equal the oracle on the model's 2 MHz bytes."""
    x = stream(hz, fmt)
    y = x if hz == 2_000_000 else TD.decimated(x, hz // 2_000_000, fmt)
    for drop in (0, 1):
        want = compare(hz, fmt, 0, x, [odd_sizes(x.size, 5 + drop)], drop_eof_buffer=drop)[0]
        ora, ora_st = C.oracle_decode(y, drop_eof=drop)
        with api.Decoder(drop_eof_buffer=drop) as d2:
            msgs = d2.decode(y)
        assert [TR.fields(m) for m in msgs] == want["msgs"]
        assert [m.raw_line() for m in msgs] == [m.hexline() for m in ora]
        assert [m.sample_pos for m in msgs] == [m.sample_pos for m in ora]
        assert list(want["stats"].values()) == ora_st


SWITCHES = [dict(signal=True, arrival=True), dict(levels=True, spectrum=True),
            dict(levels=True, spectrum=True, drop_eof_buffer=1), dict(recover=True, weak_preambles=True),
            dict(gpu_resolve=1)]
SWITCH_CASES = [(2_000_000, "uc8", 0), (2_400_000, "uc8", 0), (10_000_000, "sc16", max_offset(10_000_000))]


@pytest.mark.gpu
@pytest.mark.parametrize("hz,fmt,offset", SWITCH_CASES)
def test_switches(hz, fmt, offset):
    x = stream(hz, fmt, offset)
    for kw in SWITCHES:
        wants = compare(hz, fmt, offset, x, [[x.size], odd_sizes(x.size, 7)], **kw)
        assert len(wants[0]["msgs"]) > 10
        if kw.get("levels"):
            assert len(wants[0]["levels"]) and len(wants[0]["spectra"])


@pytest.mark.gpu
@pytest.mark.parametrize("hz,fmt,offset", SWITCH_CASES)
def test_multi_gpu(hz, fmt, offset):
    """n_gpus=2 with one-buffer batches: every other batch is copied to the second GPU's slot (with one
    physical GPU, the same device again)."""
    x = stream(hz, fmt, offset)
    compare(hz, fmt, offset, x, [[x.size], odd_sizes(x.size, 9)], n_gpus=2, max_batch_bytes=BUF, levels=True,
            spectrum=True, recover=True, signal=True)


@pytest.mark.gpu
@pytest.mark.parametrize("hz,fmt,offset", SWITCH_CASES)
def test_no_read_after_return(hz, fmt, offset):
    x = stream(hz, fmt, offset)
    compare(hz, fmt, offset, x, [odd_sizes(x.size, 3), odd_sizes(x.size, 4, hi=3 * BUF)], scribble=True,
            levels=True, spectrum=True)


@pytest.mark.gpu
def test_tensor_dispatch():
    """Decoder.process and decode take a CUDA tensor of any dtype as its raw bytes."""
    import torch
    x = stream(10_000_000, "sc16")
    v = torch.from_numpy(x.view(np.int16).copy()).cuda()                 # int16 SC16 I/Q, as a radio hands it over
    with make(10_000_000, "sc16") as host, make(10_000_000, "sc16") as dev:
        want = [TR.fields(m) for m in host.decode(x)]
        assert [TR.fields(m) for m in dev.decode(v)] == want
        assert [TR.fields(m) for m in dev.decode(v, chunk=100_003)] == want
        pair = v.view(-1, 2)[:, :1].expand(-1, 2)                       # not contiguous: copied first
        raw = pair.contiguous().cpu().numpy().view(np.uint8)
        assert [TR.fields(m) for m in dev.decode(pair)] == [TR.fields(m) for m in host.decode(raw)]
        dev.reset()
        dev.process(v[: v.numel() // 2])
        dev.process(v[v.numel() // 2:])
        dev.finish()
        assert [TR.fields(m) for m in dev.take_messages()] == want
        assert [TR.fields(m) for m in dev.decode(x)] == want              # numpy still takes the host path


# ---------------------------------------------------------------- GPU: lifecycle and refusals


@pytest.mark.gpu
@pytest.mark.parametrize("hz,fmt", [(2_000_000, "uc8"), (2_400_000, "uc8"), (6_000_000, "sc16q11")])
def test_lifecycle(hz, fmt):
    import torch
    x = stream(hz, fmt)
    d = torch.from_numpy(x).cuda()
    with make(hz, fmt) as host, make(hz, fmt) as dev:
        want = [TR.fields(m) for m in host.decode(x)]
        # reset mid-stream, then a new device-fed stream; zero-byte calls, with and without a pointer
        dev.reset()
        dev.process_device_ptr(d.data_ptr(), BUF + 1001)
        dev.reset()
        dev.process_device_ptr(0, 0)
        dev.process_device_ptr(d.data_ptr(), 0)
        dev.process_device_ptr(d.data_ptr(), x.size)
        dev.process_device_ptr(d.data_ptr() + x.size, 0)
        dev.finish()
        assert [TR.fields(m) for m in dev.take_messages()] == want
        # finish with an empty, a partial and a whole pending buffer (at 2 MHz UC8: of the EOF buffer)
        for n in (0, 1, 2 * BUF - 3, 2 * BUF):
            for drop in (0, 1):
                with make(hz, fmt, drop_eof_buffer=drop) as h, make(hz, fmt, drop_eof_buffer=drop) as g:
                    feed_host(h, x[:n], [n])
                    feed_device(g, x[:n], [n])
                    assert results(g, {}) == results(h, {}), (hz, fmt, n, drop)


@pytest.mark.gpu
def test_refusals():
    import torch
    x = stream(2_000_000, "uc8")[: 3 * BUF]
    d = torch.from_numpy(x).cuda()
    with api.Decoder() as dec:
        with pytest.raises(RuntimeError, match="in host memory"):
            dec.process_device_ptr(x.ctypes.data, x.size)
        pinned = api.PinnedBuffer(4096)
        try:
            with pytest.raises(RuntimeError, match="in pinned host memory"):
                dec.process_device_ptr(pinned.ptr, 4096)
        finally:
            pinned.free()
        with pytest.raises(RuntimeError, match="null pointer"):
            dec.process_device_ptr(0, 16)
        # one kind of memory per stream
        dec.reset()
        dec.process_device_ptr(d.data_ptr(), 1000)
        with pytest.raises(RuntimeError, match="in progress"):
            dec.process(x[1000:2000])
        dec.finish()
        dec.reset()
        dec.process(x[:1000])
        with pytest.raises(RuntimeError, match="in progress"):
            dec.process_device_ptr(d.data_ptr() + 1000, 1000)
        dec.finish()
        dec.reset()                                                     # each refusal left the decoder usable
        with api.Decoder() as h:
            assert [TR.fields(m) for m in dec.decode(d)] == [TR.fields(m) for m in h.decode(x)]


@pytest.mark.gpu
@pytest.mark.skipif("not __import__('torch').cuda.device_count() > 1", reason="needs two GPUs")
def test_tensor_on_other_device():
    import torch
    t = torch.zeros(BUF, dtype=torch.uint8, device="cuda:1")
    with api.Decoder(device=0) as dec:
        with pytest.raises(ValueError, match="cuda:1"):
            dec.process(t)
        with pytest.raises(RuntimeError, match="memory of device 1"):
            dec.process_device_ptr(t.data_ptr(), BUF)


# ---------------------------------------------------------------- GPU: past 2^32 output samples

SILENT_CHUNK = 256 << 20


@pytest.mark.gpu
@pytest.mark.parametrize("hz,fmt,offset", [(2_000_000, "uc8", 0), (10_000_000, "sc16", -max_offset(10_000_000))])
def test_long_stream(hz, fmt, offset):
    """A silent prefix that ends past 2^32 output samples (at 10 MS/s SC16 past 2^34 input samples, where
    the shift's phase has wrapped), then traffic: the device-fed decode equals the host-fed one given the
    same prefix and traffic, message for message with sample_pos."""
    import torch
    m = hz // 2_000_000
    bps = 2 if fmt == "uc8" else 4
    prefix = (2 ** 32 // B + 2) * B * m * bps                           # bytes: whole 2 MHz buffers
    x = stream(hz, fmt, offset)
    sizes = odd_sizes(x.size, 21)
    kw = dict(signal=True, arrival=True)
    with make(hz, fmt, offset, **kw) as host, make(hz, fmt, offset, **kw) as dev:
        buf = api.PinnedBuffer(SILENT_CHUNK)
        try:
            buf.array[:] = SILENCE[fmt]
            host.reset()
            left = prefix
            while left:
                n = min(SILENT_CHUNK - 1, left)                          # odd calls: the prefix splits samples
                host.process_ptr(buf.ptr, n)
                left -= n
        finally:
            buf.free()
        silent = torch.full((SILENT_CHUNK,), SILENCE[fmt], dtype=torch.uint8, device="cuda")
        d = torch.from_numpy(x).cuda()
        torch.cuda.synchronize()
        dev.reset()
        left = prefix
        while left:
            n = min(SILENT_CHUNK - 1, left)
            dev.process_device_ptr(silent.data_ptr(), n)
            left -= n
        assert not host.take_messages() and not dev.take_messages()
        off = 0
        for n in sizes:
            host.process(x[off: off + n])
            dev.process_device_ptr(d.data_ptr() + off, n)
            off += n
        host.finish()
        dev.finish()
        want, got = results(host, kw), results(dev, kw)
        assert len(want["msgs"]) > 10
        assert want["msgs"][0][[f for f, _ in api.Message._fields_].index("sample_pos")] > 2 ** 32
        assert got == want


# ---------------------------------------------------------------- CPU


def test_symbol_exported():
    assert "modes_process_device" in api.EXPORTS
    header = (C.ROOT / "include" / "modes_b200.h").read_text()
    assert "int  modes_process_device(modes_ctx *ctx, const void *d_iq, size_t nbytes);" in header
    assert hasattr(api.lib(), "modes_process_device")
    assert api.lib().modes_process_device(None, None, 0) == -1


class _Lib:
    """Records the process calls a Decoder makes."""

    def __init__(self):
        self.calls = []

    def modes_process(self, h, p, n):
        self.calls.append(("host", n))
        return 0

    def modes_process_device(self, h, p, n):
        self.calls.append(("device", p.value, n))
        return 0

    def modes_finish(self, h):
        return 0

    def modes_reset(self, h):
        return 0


class _Tensor:
    """What Decoder reads of a CUDA tensor."""

    is_cuda = True

    def __init__(self, ptr, numel, itemsize, index=0, contiguous=True):
        self.ptr, self.n, self.size, self.contig = ptr, numel, itemsize, contiguous
        self.device = types.SimpleNamespace(index=index)

    def data_ptr(self):
        return self.ptr

    def numel(self):
        return self.n

    def element_size(self):
        return self.size

    def is_contiguous(self):
        return self.contig

    def contiguous(self):
        return _Tensor(0x9000, self.n, self.size, self.device.index)


@pytest.fixture
def stub(monkeypatch):
    L = _Lib()
    synced = []
    monkeypatch.setattr(api, "lib", lambda: L)
    monkeypatch.setattr(api, "_sync_stream", lambda t: synced.append(t.data_ptr()))
    dec = object.__new__(api.Decoder)
    dec._h = 1
    dec.cfg = types.SimpleNamespace(device=0)
    dec._collector = types.SimpleNamespace(messages=[])
    yield dec, L, synced
    dec._h = None


def test_dispatch(stub):
    dec, L, synced = stub
    dec.process(np.zeros(10, np.uint8))
    dec.process(b"\x7f" * 7)
    dec.process(np.zeros(5, np.int16))                                  # numpy: its values as bytes, as before
    assert L.calls == [("host", 10), ("host", 7), ("host", 5)] and not synced
    L.calls.clear()
    dec.process(_Tensor(0x1000, 6, 2))
    dec.process(_Tensor(0x2000, 6, 2, contiguous=False))
    assert L.calls == [("device", 0x1000, 12), ("device", 0x9000, 12)]
    assert synced == [0x1000, 0x9000]
    L.calls.clear()
    dec.decode(_Tensor(0x4000, 10, 4), chunk=15)
    assert L.calls == [("device", 0x4000, 15), ("device", 0x400f, 15), ("device", 0x401e, 10)]
    L.calls.clear()
    dec.decode(np.zeros(40, np.uint8), chunk=15)
    assert L.calls == [("host", 15), ("host", 15), ("host", 10)]


def test_other_device_refused(stub):
    dec, L, synced = stub
    with pytest.raises(ValueError, match="cuda:0"):
        dec.process(_Tensor(0x1000, 6, 2, index=1))
    with pytest.raises(ValueError, match="cuda:0"):
        dec.decode(_Tensor(0x1000, 6, 2, index=1))
    assert not L.calls and not synced
