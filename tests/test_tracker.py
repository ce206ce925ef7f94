"""SURVEY.md §8(f) item 3: the aircraft tracker (modes_tracker_*, pure host code) against the
reference's own interactiveReceiveData / decodeCPR / decodeCPRSurface / modesSendSBSOutput /
aircraftsToJson, driven message by message with the same explicit clock.  Positions are compared
bit for bit (doubles), text byte for byte.  The reference's answers are replayed from
tests/golden/tracker_ref.tape.gz (gzipped JSON); `MODES_RECORD_REFERENCE=1 python -m pytest tests/test_tracker.py`
records them anew from oracle/_ref (built by `make oracle` where the reference's sources are found)."""
import ctypes
import gzip
import json
import math
import os
from pathlib import Path

import numpy as np
import pytest

import checker as C
from dump1090_b200 import api, synth


TAPE = Path(__file__).resolve().parent / "golden" / "tracker_ref.tape.gz"
RECORD = os.environ.get("MODES_RECORD_REFERENCE") == "1"
_tapes = {}


class _Aircraft(tuple):
    """A recorded struct aircraft: as_tuple() and the position fields the tests read."""
    def as_tuple(self):
        return tuple(self)

    addr = property(lambda self: self[0])
    lat = property(lambda self: self[12])
    lon = property(lambda self: self[13])


def _enc(v):
    if hasattr(v, "as_tuple"):
        return {"a": [x.decode("latin1") if isinstance(x, bytes) else x for x in v.as_tuple()]}
    if isinstance(v, (list, tuple)):
        return [_enc(x) for x in v]
    return v


def _dec(v):
    if isinstance(v, dict):
        return _Aircraft(x.encode("latin1") if i in (1, 2) else x for i, x in enumerate(v["a"]))
    if isinstance(v, list):
        return tuple(_dec(x) for x in v)
    return v


class _Reference:
    """The reference's tracker door: its answers in call order, from the tape (or, recording, from oracle/_ref)."""

    def __init__(self, name):
        self.name, self.k = name, 0
        if RECORD:
            _tapes[name] = []
        else:
            if not _tapes:
                with gzip.open(TAPE, "rb") as f:
                    _tapes.update(json.loads(f.read().decode()))
            self.tape = _tapes[name]

    def _ask(self, call):
        if RECORD:
            v = call()
            _tapes[self.name].append(_enc(v))
            return v
        self.k += 1
        return _dec(self.tape[self.k - 1])

    def tracker(self, check_crc=1):
        ref, ask = (C.RefTracker(check_crc) if RECORD else None), self._ask

        class T:
            update = staticmethod(lambda m, now: ask(lambda: ref.update(m, now)))
            aircraft = staticmethod(lambda: list(ask(lambda: ref.aircraft())))
            reference = staticmethod(lambda: ask(lambda: ref.reference()))
            json = staticmethod(lambda metric=0: ask(lambda: ref.json(metric)))
            expire = staticmethod(lambda now, ttl: ask(lambda: ref.expire(now, ttl)))
            table = staticmethod(lambda now, metric, rows: ask(lambda: C.ref_track_table(now, metric, rows)))
        return T

    def cpr_nl(self, lat):
        return self._ask(lambda: C.ref_cpr_nl(lat))


@pytest.fixture
def reference(request):
    yield _Reference(request.node.name)
    if RECORD:
        with gzip.GzipFile(TAPE, "wb", mtime=0) as f:
            f.write(json.dumps(_tapes, sort_keys=True, separators=(",", ":")).encode())


def _decode_frame(frame: bytes) -> C.Msg:
    """decodeModesMessage on raw bytes (fresh ICAO cache), through the oracle's restatement
    (test_oracle.py::test_decode_bytes_matches_reference pins it to the reference)."""
    out = C.Msg()
    buf = (ctypes.c_uint8 * 14)(*(list(frame) + [0] * (14 - len(frame))))
    C.oracle_lib().oracle_decode_bytes(buf, 1, 0, ctypes.byref(out))
    return out


def _as_product(m) -> api.Message:
    p = api.Message()
    ctypes.memmove(ctypes.byref(p), ctypes.byref(m), ctypes.sizeof(api.Message))
    return p


def _run_both(reference, messages, times, check_crc=1):
    """Feed both trackers; compare aircraft state and SBS line after every message."""
    ref, got = reference.tracker(check_crc), api.Tracker(check_crc)
    tracked = 0
    for k, (m, t) in enumerate(zip(messages, times)):
        r = ref.update(m, t)
        g = got.update(_as_product(m), t)
        assert (r is None) == (g is None), f"message {k}: tracked by one side only"
        if r is None:
            continue
        tracked += 1
        assert g[0].as_tuple() == r[0].as_tuple(), f"message {k} (DF{m.msgtype} ME{m.metype}): aircraft differs"
        assert g[1] == r[1], f"message {k}: SBS line differs: {g[1]!r} != {r[1]!r}"
    assert [a.as_tuple() for a in got.aircraft()] == [a.as_tuple() for a in ref.aircraft()]
    assert got.reference() == ref.reference()
    for metric in (0, 1):
        assert got.json(metric) == ref.json(metric)
        for rows in (3, 15, 100):
            now = times[-1] + 4321 * (rows + metric)
            assert got.table(now, metric, rows) == ref.table(now, metric, rows)
    return ref, got, tracked


def test_nl_function_matches_reference(checker_libs, reference):
    """The zone-count table is generated from its defining formula: identical to the reference's
    literal table everywhere, including one ulp either side of every transition latitude."""
    nz = 15.0
    a = 1.0 - math.cos(math.pi / (2.0 * nz))
    lats = list(np.linspace(-90.5, 90.5, 20001))
    for nl in range(2, 60):
        t = round(math.degrees(math.acos(math.sqrt(a / (1.0 - math.cos(2.0 * math.pi / nl))))), 8)
        for d in (t, np.nextafter(t, 0), np.nextafter(t, 100), t - 1e-9, t + 1e-9):
            lats += [float(d), -float(d)]
    for lat in lats:
        assert api.cpr_nl(lat) == reference.cpr_nl(lat), lat


def test_tracker_on_decoded_traffic(checker_libs, reference):
    """Everything the decoder delivers from a mixed-traffic stream (identification, airborne and
    surface positions with random CPR fields, velocities, address/parity replies)."""
    data = synth.random_traffic(131072 * 12, 2600, 41, n_aircraft=25)
    for check_crc in (1, 0):
        msgs, _ = C.oracle_decode(data, check_crc=check_crc)
        times = [1_700_000_000_000 + 37 * k for k in range(len(msgs))]          # ~27 messages per second
        _, _, tracked = _run_both(reference, msgs, times, check_crc)
        assert tracked > 300


def _cpr_encode(lat, lon, odd):
    """Airborne CPR encoding of a position (17 bits each), the inverse of what the tracker decodes."""
    dlat = 360.0 / (60 - odd)
    yz = math.floor(131072 * ((lat % dlat) / dlat) + 0.5)
    rlat = dlat * (yz / 131072 + math.floor(lat / dlat))
    nl = api.cpr_nl(rlat)
    dlon = 360.0 / max(nl - odd, 1)
    xz = math.floor(131072 * ((lon % dlon) / dlon) + 0.5)
    return yz & 0x1FFFF, xz & 0x1FFFF


def _position_frame(icao, tc, odd, yz, xz, alt12=0x3A5):
    bits = (tc << 51) | (alt12 << 36) | (odd << 34) | (yz << 17) | xz
    return synth.make_frame(17, 5, icao.to_bytes(3, "big") + bits.to_bytes(7, "big"))


def test_tracker_decodes_real_positions(checker_libs, reference):
    """Aircraft flying real tracks: even/odd pairs decode to the encoded position (to CPR
    resolution), the reference position follows, surface frames decode against it — and every
    double equals the reference's."""
    rng = np.random.default_rng(5)
    fleet = [(0x4B1600 + i, 47.0 + rng.uniform(-3, 3), 8.0 + rng.uniform(-4, 4), rng.uniform(-0.002, 0.002),
              rng.uniform(-0.003, 0.003)) for i in range(8)]
    fleet += [(0xA00001, -33.9, 151.2, 0.001, 0.001), (0x7C0001, 69.7, 18.9, 0.0, 0.004), (0xE40001, -0.3, -78.5, 0.002, 0.0)]
    msgs, times = [], []
    t = 1_700_000_000_000
    for step in range(60):
        for icao, lat0, lon0, vlat, vlon in fleet:
            lat, lon = lat0 + vlat * step, lon0 + vlon * step
            odd = (step + icao) & 1
            yz, xz = _cpr_encode(lat, lon, odd)
            msgs.append(_decode_frame(_position_frame(icao, 11, odd, yz, xz)))
            times.append(t)
            t += int(rng.integers(20, 400))
            if step % 7 == 3:                                            # a surface frame from the same airframe
                sbits = (6 << 51) | (int(rng.integers(0, 128)) << 44) | (1 << 43) | (int(rng.integers(0, 128)) << 36) \
                        | (odd << 34) | ((yz * 4) & 0x1FFFF) << 17 | ((xz * 4) & 0x1FFFF)
                msgs.append(_decode_frame(synth.make_frame(17, 5, icao.to_bytes(3, "big") + sbits.to_bytes(7, "big"))))
                times.append(t)
                t += 50
        if step == 30:
            t += 11_000                                                   # a gap longer than the 10 s pairing window
    ref, got, tracked = _run_both(reference, msgs, times)
    assert tracked == len(msgs)
    # sanity of the test itself: the airborne fleet ends up where it was flown to
    by_addr = {a.addr: a for a in got.aircraft()}
    for icao, lat0, lon0, vlat, vlon in fleet:
        a = by_addr[icao]
        if a.altitude:                                                    # last frame was airborne
            assert abs(a.lat - (lat0 + vlat * 59)) < 0.02 and abs(a.lon - (lon0 + vlon * 59)) < 0.02
    assert got.reference()[2] > 100


def test_tracker_expiry_and_order(checker_libs, reference):
    msgs = [_decode_frame(synth.make_frame(17, 5, (0x400000 + i).to_bytes(3, "big") + bytes([0x20, 0x10, 0x82, 0x0C, 0x30, 0xC3, 0x0C])))
            for i in range(20)]
    ref, got = reference.tracker(), api.Tracker()
    t0 = 1_700_000_000_000
    for k, m in enumerate(msgs):
        ref.update(m, t0 + 1000 * k)
        got.update(_as_product(m), t0 + 1000 * k)
    assert [a.addr for a in got.aircraft()] == [a.addr for a in ref.aircraft()] == [0x400000 + i for i in reversed(range(20))]
    for now, ttl in ((t0 + 25_000, 60), (t0 + 25_000, 10), (t0 + 25_999, 9), (t0 + 40_000, 0)):
        assert got.expire(now, ttl) == ref.expire(now, ttl)
        assert [a.as_tuple() for a in got.aircraft()] == [a.as_tuple() for a in ref.aircraft()]
    assert got.aircraft() == []


def test_tracker_ignores_bad_crc_when_checking(checker_libs, reference):
    bad = _decode_frame(bytes.fromhex("8D4840D6202CC371C32CE0576099"))       # last byte off: CRC fails, not fixable to DF17? either way
    bad.crcok = 0
    assert api.Tracker(1).update(_as_product(bad), 1) is None and reference.tracker(1).update(bad, 1) is None
    assert api.Tracker(0).update(_as_product(bad), 1) is not None and reference.tracker(0).update(bad, 1) is not None


def test_stream_clock_starts_at_the_epoch(checker_libs, reference):
    """A file's stream clock (sample position / 2 MHz) starts at 0: fed to the tracker as is, the
    first airborne position of a new aircraft would be paired with the empty (time 0) slot of the
    other parity and decoded against zeros.  With MODES_STREAM_EPOCH_MS added — what the C host
    does — the first frame waits for its partner, exactly as under the reference's wall clock."""
    lat, lon, icao = 47.3, 8.5, 0x4B1601
    frames = []
    for step, odd in enumerate((0, 1, 0)):
        yz, xz = _cpr_encode(lat + 0.001 * step, lon, odd)
        frames.append(_decode_frame(_position_frame(icao, 11, odd, yz, xz)))
    stream_ms = [3, 450, 900]                                            # first seconds of a file
    # reference behaviour under its own (wall) clock: no position after one frame, a position after two
    ref, got = reference.tracker(), api.Tracker()
    for m, t in zip(frames, stream_ms):
        r = ref.update(m, 1_700_000_000_000 + t)
        g = got.update(_as_product(m), api.STREAM_EPOCH_MS + t)
        rt, gt = r[0].as_tuple(), g[0].as_tuple()
        assert (g[0].lat, g[0].lon) == (r[0].lat, r[0].lon)
        assert g[1] == r[1]                                               # SBS line
        if t == 3:
            assert (g[0].lat, g[0].lon) == (0.0, 0.0)
    assert abs(got.aircraft()[0].lat - lat) < 0.02 and abs(got.aircraft()[0].lon - lon) < 0.02
    # the hazard itself (documented in include/modes_b200.h): a clock starting at 0 pairs the first frame with nothing
    raw = api.Tracker()
    g = raw.update(_as_product(frames[0]), stream_ms[0])
    assert (g[0].lat, g[0].lon) != (0.0, 0.0)
