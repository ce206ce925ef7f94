"""Deterministic synthetic 2 MHz u8 I/Q streams with injected Mode S frames.

Utility for tests and bench.py (BASELINE.json configs 2-4: "synthetic IQ w/
injected DF17", low-SNR sweep).  All randomness comes from a counter-based
splitmix64 hash, so a (seed, parameters) pair produces the same bytes on every
machine and numpy version; nothing here depends on numpy's RNG streams.

Signal model (SURVEY.md §8(d) recipe): pulse-position modulation at one sample
per half-bit; preamble pulses at samples 0, 2, 7, 9 (dump1090.c:1570-1592);
data bit b is a pulse at sample 16+2b for a 1 and 17+2b for a 0
(dump1090.c:1669-1688); amplitude A on a carrier of random phase; additive
noise of standard deviation sigma LSB on I and Q; zero level 127
(dump1090.c:1462-1463); rounded and clipped to u8.  An optional fractional
delay leaks each pulse into the following sample, which is what the
reference's phase-corrected retry (dump1090.c:1498-1558) exists for.

The Mode S parity here is an independent bitwise polynomial division by the
generator 0x1FFF409; it is not shared with oracle/ or with the product.
"""
from __future__ import annotations

import numpy as np

GENERATOR = 0x1FFF409
_M64 = (1 << 64) - 1


def _mix64(x: np.ndarray) -> np.ndarray:
    """splitmix64 finaliser, elementwise on uint64."""
    x = x.astype(np.uint64, copy=True)
    with np.errstate(over="ignore"):
        x += np.uint64(0x9E3779B97F4A7C15)
        x ^= x >> np.uint64(30)
        x *= np.uint64(0xBF58476D1CE4E5B9)
        x ^= x >> np.uint64(27)
        x *= np.uint64(0x94D049BB133111EB)
        x ^= x >> np.uint64(31)
    return x


def _mix64_scalar(x: int) -> int:
    x = (x + 0x9E3779B97F4A7C15) & _M64
    x ^= x >> 30
    x = (x * 0xBF58476D1CE4E5B9) & _M64
    x ^= x >> 27
    x = (x * 0x94D049BB133111EB) & _M64
    x ^= x >> 31
    return x


class Counter:
    """Tiny deterministic scalar RNG (hash of a running counter)."""

    def __init__(self, seed: int):
        self.key = _mix64_scalar(seed & _M64)
        self.n = 0

    def u64(self) -> int:
        self.n += 1
        return _mix64_scalar(self.key ^ (self.n * 0xD1342543DE82EF95 & _M64))

    def below(self, n: int) -> int:
        return self.u64() % n

    def uniform(self) -> float:
        return (self.u64() >> 11) / float(1 << 53)


def noise(nvalues: int, sigma: float, seed: int, offset: int = 0) -> np.ndarray:
    """Approximately Gaussian noise (sum of four uniforms), float64, length nvalues."""
    idx = np.arange(offset, offset + nvalues, dtype=np.uint64)
    key = np.uint64(_mix64_scalar(seed & _M64))
    with np.errstate(over="ignore"):
        h = _mix64(idx * np.uint64(0x2545F4914F6CDD1D) ^ key)
    parts = [((h >> np.uint64(16 * k)) & np.uint64(0xFFFF)).astype(np.float64) for k in range(4)]
    s = (parts[0] + parts[1] + parts[2] + parts[3]) / 65536.0 - 2.0   # var = 4/12
    return s * (sigma * np.sqrt(3.0))


def modes_parity(data: bytes) -> int:
    """24-bit Mode S parity of the data bits (everything except the last 3 bytes)."""
    reg = 0
    for byte in data:
        for k in range(7, -1, -1):
            reg = (reg << 1) | ((byte >> k) & 1)
            if reg & (1 << 24):
                reg ^= GENERATOR
    # append 24 zero bits (multiply by x^24) and reduce
    for _ in range(24):
        reg <<= 1
        if reg & (1 << 24):
            reg ^= GENERATOR
    return reg & 0xFFFFFF


def make_frame(df: int, first_byte_low3: int, body: bytes, icao_for_ap: int | None = None) -> bytes:
    """Assemble a frame: 5-bit DF + 3 bits, then `body`, then 24 parity bits.

    DF 16..21 frames are 14 bytes (body = 10 bytes), others 7 bytes (body = 3).
    If icao_for_ap is given the parity is XORed with it (address/parity field,
    as in DF 0/4/5/16/20/21, dump1090.c:962-974).
    """
    nbody = 10 if 16 <= df <= 21 else 3
    assert len(body) == nbody
    data = bytes([((df & 31) << 3) | (first_byte_low3 & 7)]) + body
    p = modes_parity(data)
    if icao_for_ap is not None:
        p ^= icao_for_ap & 0xFFFFFF
    return data + bytes([(p >> 16) & 0xFF, (p >> 8) & 0xFF, p & 0xFF])


def flip_bits(frame: bytes, positions) -> bytes:
    b = bytearray(frame)
    for p in positions:
        b[p >> 3] ^= 0x80 >> (p & 7)
    return bytes(b)


def frame_envelope(frame: bytes, frac: float = 0.0) -> np.ndarray:
    """Amplitude envelope (0..1) of preamble + frame, one value per 0.5 us sample."""
    nbits = len(frame) * 8
    env = np.zeros(16 + 2 * nbits + 1, dtype=np.float64)
    for p in (0, 2, 7, 9):
        env[p] = 1.0
    for b in range(nbits):
        bit = (frame[b >> 3] >> (7 - (b & 7))) & 1
        env[16 + 2 * b + (0 if bit else 1)] = 1.0
    if frac > 0.0:
        shifted = np.zeros_like(env)
        shifted[1:] = env[:-1]
        env = (1.0 - frac) * env + frac * shifted
    return env


def _rate_ratio(sample_rate: int) -> tuple[int, int]:
    """sample_rate / 2 MHz as a reduced fraction (a, b): one 0.5 us half-bit slot is a / b samples."""
    from math import gcd
    g = gcd(int(sample_rate), 2_000_000)
    return int(sample_rate) // g, 2_000_000 // g


def _slot_edge(slot: int, frac: float, a: int, b: int) -> tuple[int, float]:
    """The start of half-bit slot `slot` (counted in 0.5 us from the stream start) delayed by frac slots,
    in samples at a / b samples per slot: (whole samples, fraction in [0, 1))."""
    whole, rem = divmod(a * slot, b)
    f = rem / b + (frac * a) / b
    carry = int(np.floor(f))
    return whole + carry, f - carry


def frame_envelope_at(frame: bytes, pos: int, frac: float, sample_rate: int) -> tuple[int, np.ndarray]:
    """Amplitude envelope (0..1) of preamble + frame arriving at 2 MHz position pos + frac, sampled at
    sample_rate: each 0.5 us pulse is a rectangle, and each sample is the pulse's overlap with its sample
    period, over the period.  Returns (index of the first sample, envelope from it).  At 2 MHz this is
    frame_envelope(frame, frac) at sample pos, bit for bit."""
    a, b = _rate_ratio(sample_rate)
    nbits = len(frame) * 8
    slots = [0, 2, 7, 9] + [16 + 2 * k + (0 if (frame[k >> 3] >> (7 - (k & 7))) & 1 else 1) for k in range(nbits)]
    first, _ = _slot_edge(pos, frac, a, b)
    last, _ = _slot_edge(pos + 16 + 2 * nbits + 1, frac, a, b)
    env = np.zeros(last - first + 2, dtype=np.float64)
    for p in sorted(slots):
        ks, fs = _slot_edge(pos + p, frac, a, b)
        ke, fe = _slot_edge(pos + p + 1, frac, a, b)
        ks -= first
        ke -= first
        if ks == ke:
            env[ks] += fe - fs
            continue
        env[ks] += 1.0 - fs
        env[ks + 1: ke] += 1.0
        env[ke] += fe
    return first, env


def synth_stream_at(nsamples: int, frames, sigma: float = 1.5, seed: int = 1, sample_rate: int = 2_000_000,
                    dtype: str = "uc8", scale: float = 1.0, tone=None, carrier_hz: float = 0.0, dc=None) -> np.ndarray:
    """synth_stream at any sample rate: frames are (pos, frame_bytes, amplitude_lsb, carrier_phase_rad,
    frac) with the arrival time pos + frac in 2 MHz samples (0.5 us), pulses per frame_envelope_at, and
    the same noise per sample as synth_stream.  At 2 MHz it equals synth_stream bit for bit.
    dtype="sc16": the same signal as signed little-endian 16-bit I/Q bytes (4 a sample), scale int16
    units to an 8-bit LSB (16 is SC16Q11's full scale, 256 SC16's), rounded and clamped to int16.
    tone=(offset_hz, amplitude_lsb): a continuous carrier at that offset from the channel centre is added
    (an out-of-band interferer where the offset is past 1 MHz); None, the default, adds nothing.
    carrier_hz: the frames are sent at that offset from the baseband's 0 Hz (a radio tuned carrier_hz below
    1090 MHz), their phase turning by 2 pi carrier_hz / sample_rate per sample of the stream; 0, the
    default, leaves them as they were.  A frame tuple may carry a sixth element, the frame's own carrier
    offset in Hz (its transmitter's offset from 1090 MHz), which adds to carrier_hz for that frame.
    dc=(i, q): a constant (a zero-IF radio's DC spike, in 8-bit LSB) added to every sample; None, the
    default, adds nothing."""
    i = noise(nsamples, sigma, seed * 2 + 11)
    q = noise(nsamples, sigma, seed * 2 + 12)
    if tone is not None:
        offset_hz, tone_amp = tone
        w = 2 * np.pi * (offset_hz / sample_rate) * np.arange(nsamples, dtype=np.float64)
        i += tone_amp * np.cos(w)
        q += tone_amp * np.sin(w)
    for fr in frames:
        pos, frame, amp, phase, frac = fr[:5]
        f_hz = carrier_hz + (fr[5] if len(fr) > 5 else 0.0)
        start, env = frame_envelope_at(frame, pos, frac, sample_rate)
        env = env * amp
        if sample_rate == 2_000_000:                       # synth_stream's envelope length
            env = env[: 16 + 2 * len(frame) * 8 + 1]
        end = min(nsamples, start + len(env))
        if start >= nsamples or end <= start:
            continue
        seg = env[: end - start]
        if f_hz:
            ph = phase + 2 * np.pi * (f_hz / sample_rate) * np.arange(start, end, dtype=np.float64)
            i[start:end] += seg * np.cos(ph)
            q[start:end] += seg * np.sin(ph)
        else:
            i[start:end] += seg * np.cos(phase)
            q[start:end] += seg * np.sin(phase)
    if dc is not None:
        i += dc[0]
        q += dc[1]
    if dtype == "sc16":
        out16 = np.empty(2 * nsamples, dtype="<i2")
        out16[0::2] = np.clip(np.rint(scale * i), -32768, 32767)
        out16[1::2] = np.clip(np.rint(scale * q), -32768, 32767)
        return out16.view(np.uint8)
    if dtype != "uc8":
        raise ValueError(f"dtype {dtype!r}: uc8 or sc16")
    out = np.empty(2 * nsamples, dtype=np.uint8)
    out[0::2] = np.clip(np.rint(127.0 + i), 0, 255).astype(np.uint8)
    out[1::2] = np.clip(np.rint(127.0 + q), 0, 255).astype(np.uint8)
    return out


def synth_stream(nsamples: int, frames, sigma: float = 1.5, seed: int = 1) -> np.ndarray:
    """Build a u8 interleaved I/Q stream of `nsamples` samples.

    frames: iterable of (pos, frame_bytes, amplitude_lsb, carrier_phase_rad, frac), optionally with a sixth
    element, the frame's carrier offset in Hz from the centre of the stream (its phase then turns by
    2 pi offset / 2 MHz per sample of the stream).  Overlapping frames add coherently in I/Q.  Returns
    uint8 array of 2*nsamples.
    """
    i = noise(nsamples, sigma, seed * 2 + 11)
    q = noise(nsamples, sigma, seed * 2 + 12)
    for fr in frames:
        pos, frame, amp, phase, frac = fr[:5]
        f_hz = fr[5] if len(fr) > 5 else 0.0
        env = frame_envelope(frame, frac) * amp
        end = min(nsamples, pos + len(env))
        if pos >= nsamples or end <= pos:
            continue
        seg = env[: end - pos]
        if f_hz:
            ph = phase + 2 * np.pi * (f_hz / 2_000_000) * np.arange(pos, end, dtype=np.float64)
            i[pos:end] += seg * np.cos(ph)
            q[pos:end] += seg * np.sin(ph)
        else:
            i[pos:end] += seg * np.cos(phase)
            q[pos:end] += seg * np.sin(phase)
    out = np.empty(2 * nsamples, dtype=np.uint8)
    out[0::2] = np.clip(np.rint(127.0 + i), 0, 255).astype(np.uint8)
    out[1::2] = np.clip(np.rint(127.0 + q), 0, 255).astype(np.uint8)
    return out


# ------------------------------------------------------------------ traffic mix

def _me_ident(rng: Counter) -> bytes:
    tc = 1 + rng.below(4)
    chars = [1 + rng.below(26) for _ in range(6)] + [48 + rng.below(10), 32]
    v = 0
    for c in chars:
        v = (v << 6) | (c & 63)
    return bytes([(tc << 3) | rng.below(8)]) + v.to_bytes(6, "big")


def _me_airborne(rng: Counter) -> bytes:
    tc = 9 + rng.below(10)
    alt12 = rng.below(4096)
    if rng.below(8):
        alt12 |= 0x10                                    # Q bit (msg[5] & 1), mostly set
    bits = (tc << 51) | (rng.below(8) << 48) | (alt12 << 36) | (rng.below(2) << 35) \
        | (rng.below(2) << 34) | (rng.below(1 << 17) << 17) | rng.below(1 << 17)
    return bits.to_bytes(7, "big")


def _me_velocity(rng: Counter) -> bytes:
    sub = 1 + rng.below(4)
    bits = (19 << 51) | (sub << 48) | (rng.below(1 << 48))
    return bits.to_bytes(7, "big")


def _me_surface(rng: Counter) -> bytes:
    tc = 5 + rng.below(4)
    bits = (tc << 51) | rng.below(1 << 51)
    return bits.to_bytes(7, "big")


def _me_other(rng: Counter) -> bytes:
    tc = [0, 20, 23, 28, 29, 31][rng.below(6)]
    bits = (tc << 51) | rng.below(1 << 51)
    return bits.to_bytes(7, "big")


def random_traffic(nsamples: int, nframes: int, seed: int, sigma: float = 1.5,
                   amp_range=(12.0, 110.0), max_flips: int = 3, frac_prob: float = 0.5,
                   n_aircraft: int = 12, return_truth: bool = False):
    """A stream with `nframes` frames of mixed downlink formats from a small fleet.

    Mix: DF17 (identification / airborne position / velocity / surface / other
    ME types), DF18, DF11 (some with a small interrogator id XORed into the
    parity, dump1090.c:1204-1209), and address/parity formats DF0/4/5/16/20/21
    (decodable only after the address was announced, dump1090.c:1183-1192).
    A share of frames carries 1..max_flips flipped bits (some in the DF field)
    and a share is sampled off-phase.  Frames are placed on a jittered grid so
    some straddle the reference's 131072-sample buffer boundaries.
    """
    rng = Counter(seed)
    fleet = [0x400000 + rng.below(0x3FFFFF) for _ in range(n_aircraft)]
    frames, truth = [], []
    slot = max(300, nsamples // max(1, nframes))
    for k in range(nframes):
        icao = fleet[rng.below(n_aircraft)]
        kind = rng.below(100)
        aa = icao.to_bytes(3, "big")
        if kind < 50:
            me = [_me_ident, _me_airborne, _me_airborne, _me_velocity, _me_surface, _me_other][rng.below(6)](rng)
            frame = make_frame(17, rng.below(8), aa + me)
        elif kind < 56:
            frame = make_frame(18, rng.below(8), aa + _me_airborne(rng))
        elif kind < 74:
            frame = make_frame(11, rng.below(8), aa)
            if rng.below(4) == 0:                       # interrogator id in the parity
                iid = 1 + rng.below(100)
                frame = frame[:4] + ((int.from_bytes(frame[4:], "big") ^ iid).to_bytes(3, "big"))
        else:
            df = [0, 4, 5, 16, 20, 21][rng.below(6)]
            nbody = 10 if df >= 16 else 3
            body = bytes(rng.below(256) for _ in range(nbody))
            frame = make_frame(df, rng.below(8), body, icao_for_ap=icao)
        nflip = 0
        r = rng.below(100)
        if r < 30 and max_flips >= 1:
            nflip = 1
        elif r < 45 and max_flips >= 2:
            nflip = 2
        elif r < 52 and max_flips >= 3:
            nflip = 3
        nbits = len(frame) * 8
        flips = sorted({rng.below(nbits) for _ in range(nflip)})
        sent = flip_bits(frame, flips)
        amp = amp_range[0] + (amp_range[1] - amp_range[0]) * rng.uniform()
        phase = 2 * np.pi * rng.uniform()
        frac = 0.15 + 0.7 * rng.uniform() if rng.uniform() < frac_prob else 0.0
        pos = k * slot + rng.below(max(1, slot - 260))
        if rng.below(16) == 0:                           # park one right at a buffer seam
            seam = 131072 * (1 + rng.below(max(1, nsamples // 131072))) - 238
            pos = max(0, min(nsamples - 260, seam - 230 + rng.below(240)))
        frames.append((pos, sent, amp, phase, frac))
        truth.append((pos, frame, flips))
    stream = synth_stream(nsamples, frames, sigma=sigma, seed=seed)
    return (stream, truth) if return_truth else stream


def df17_grid(nsamples: int, period: int, seed: int, sigma: float = 1.5, amp: float = 60.0,
              flips_cycle=(0, 1, 2, 3)) -> np.ndarray:
    """DF17 frames every `period` samples, flip count cycling through flips_cycle
    (BASELINE.json config 2: 'synthetic IQ w/ injected DF17')."""
    rng = Counter(seed)
    frames = []
    k = 0
    pos = 300
    while pos + 260 < nsamples:
        icao = 0x400000 + rng.below(0x3FFFFF)
        frame = make_frame(17, 5, icao.to_bytes(3, "big") + _me_airborne(rng))
        nflip = flips_cycle[k % len(flips_cycle)]
        flips = sorted({5 + rng.below(107) for _ in range(nflip)})
        frames.append((pos, flip_bits(frame, flips), amp, 2 * np.pi * rng.uniform(), 0.0))
        pos += period
        k += 1
    return synth_stream(nsamples, frames, sigma=sigma, seed=seed)


def _fleet_frame(frames: list, fleet, rng: Counter, k: int, n_aircraft: int, amp: float, period: int, carrier_of):
    """fleet_at's frame k (appended to frames, as its hex returned); carrier_of(address) -> Hz, when given, is
    each aircraft's own carrier offset, carried as the frame tuple's sixth element."""
    icao = fleet[rng.below(n_aircraft)]
    me = [_me_ident, _me_airborne, _me_airborne, _me_velocity][rng.below(4)](rng)
    frame = make_frame(17, 5, icao.to_bytes(3, "big") + me)
    fr = (200 + k * period + rng.below(100), frame, amp, 2 * np.pi * rng.uniform(), 0.5 * rng.uniform())
    frames.append(fr if carrier_of is None else fr + (float(carrier_of(icao)),))
    return frame.hex()


def fleet_at(snr_db: float, nframes: int, seed: int, n_aircraft: int = 20, amp: float = 20.0, period: int = 400,
             carrier_of=None):
    """DF17 extended squitters (identification, airborne position, velocity) of a fleet of n_aircraft,
    each sending many frames, in noise at snr_db (pulse power / noise power = amp^2 / (2 sigma^2)), one
    frame every ~period samples.  carrier_of(address) -> Hz gives each aircraft its own carrier offset;
    None, the default, sends every frame at 0 Hz.  Returns (stream, set of the frames' hex)."""
    sigma = amp / (np.sqrt(2.0) * 10 ** (snr_db / 20.0))
    rng = Counter(seed)
    fleet = [0x400000 + rng.below(0x3FFFFF) for _ in range(n_aircraft)]
    frames, truth = [], set()
    for k in range(nframes):
        truth.add(_fleet_frame(frames, fleet, rng, k, n_aircraft, amp, period, carrier_of))
    return synth_stream(200 + nframes * period + 400, frames, sigma=sigma, seed=seed), truth


def fleet_at_rate(snr_db: float, nframes: int, seed: int, sample_rate: int = 2_400_000, n_aircraft: int = 20,
                  amp: float = 20.0, period: int = 400, dtype: str = "uc8", scale: float = 1.0, tone=None,
                  carrier_hz: float = 0.0, dc=None, carrier_of=None):
    """fleet_at sampled at sample_rate (2.4 MS/s: what dump1090-fa and readsb record): the same frames,
    arrival times, amplitudes and carrier phases, over the same stretch of time, with the same noise per
    sample; dtype, scale, tone, carrier_hz and dc as synth_stream_at, carrier_of as fleet_at (each
    aircraft's offset adds to carrier_hz).  Returns (stream, set of the frames' hex)."""
    sigma = amp / (np.sqrt(2.0) * 10 ** (snr_db / 20.0))
    rng = Counter(seed)
    fleet = [0x400000 + rng.below(0x3FFFFF) for _ in range(n_aircraft)]
    frames, truth = [], set()
    for k in range(nframes):
        truth.add(_fleet_frame(frames, fleet, rng, k, n_aircraft, amp, period, carrier_of))
    a, b = _rate_ratio(sample_rate)
    n = -(-(200 + nframes * period + 400) * a // b)
    return synth_stream_at(n, frames, sigma=sigma, seed=seed, sample_rate=sample_rate, dtype=dtype, scale=scale,
                           tone=tone, carrier_hz=carrier_hz, dc=dc), truth


def tile_to(data: np.ndarray, nbytes: int) -> np.ndarray:
    """Tile a capture back-to-back to exactly nbytes (SURVEY §8(d) input 2)."""
    reps = -(-nbytes // data.size)
    return np.tile(data, reps)[:nbytes].copy()
