"""Accuracy of the carrier measurement (modes_set_carrier) on synthetic DF17 fleets of known per-aircraft
carrier offsets, on CPU.  Each aircraft of a fleet of 24 gets its own offset, its address hashed to one of 17
steps from -400 to +400 kHz, plus a common receiver offset; the stream is synthesised at the input rate (with the frames moved
by the input offset, as a radio tuned off 1090 MHz records them), brought to the 2 MHz bytes the decoder
decodes by the numpy restatements of the resampler, decimator and frequency shift, and decoded by the oracle.
Each delivered message gets the code of the numpy restatement (tests/carrier_model.py; the GPU computes the
same codes, tests/test_carrier.py), and its frequency is compared with its aircraft's true offset.  The
receiver estimate is api.carrier_summary's median over aircraft of their medians, compared with the common
offset plus the median of the measured aircraft's own offsets (the receiver estimate's true value).  Noise is
density-matched: sigma = 1.5 sqrt(rate / 2 MHz) LSB per input sample.
Usage: carrier_accuracy.py [N frames]  (default 3000); prints a markdown table."""
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
for p in (str(ROOT), str(ROOT / "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)
import numpy as np

import carrier_model as CM
import checker as C
import decimate_model as DM
import resample_model as RM
import shift_model as SM
from dump1090_b200 import api, synth

N_AIRCRAFT = 24
RECEIVER_HZ = 7300.0                                     # the common offset every frame carries
CASES = [(2_000_000, 0), (2_400_000, 0), (8_000_000, 0), (8_000_000, 2_000_000)]
AMPS = (8.0, 12.0, 20.0, 60.0)


def aircraft_hz(addr: int) -> float:
    """An aircraft's own offset: its address hashed to one of 17 steps from -400 to +400 kHz."""
    return -400_000.0 + 50_000.0 * ((addr * 2654435761) % 17)


def true_hz(addr: int) -> float:
    return RECEIVER_HZ + aircraft_hz(addr)


def receiver_truth_hz(summary: dict) -> float:
    """What the receiver estimate of carrier_summary should read for the aircraft it measured: the median over
    them of their true offsets."""
    return float(np.median([true_hz(a) for a in summary["per_aircraft"]]))


def two_mhz_bytes(rate: int, offset: int, amp: float, n_frames: int, seed: int) -> np.ndarray:
    """The 2 MHz bytes the decoder decodes for a fleet synthesised at `rate` with the input offset."""
    sigma = 1.5 * np.sqrt(rate / 2_000_000)
    snr_db = 20 * np.log10(amp / (np.sqrt(2.0) * sigma))
    x, _ = synth.fleet_at_rate(snr_db, n_frames, seed, sample_rate=rate, n_aircraft=N_AIRCRAFT, amp=amp,
                               period=400, carrier_hz=float(offset), carrier_of=true_hz)
    if rate == 2_000_000:
        return x
    if rate == 2_400_000:
        return RM.resample(x)
    m = rate // 2_000_000
    return SM.shift_decimate(x, m, offset) if offset else DM.decimate(x, m)


def measure(rate: int, offset: int, amp: float, n_frames: int = 3000, seed: int = 5) -> dict:
    """Per-message errors (Hz) of the oracle's decode of one fleet, and the receiver estimate's error."""
    y = two_mhz_bytes(rate, offset, amp, n_frames, seed)
    msgs, _ = C.oracle_decode(y)
    err, measured = [], []
    for m in msgs:
        code = CM.expected_code(y, m)
        assert code != 0
        addr = (int(m.aa1) << 16) | (int(m.aa2) << 8) | int(m.aa3)
        hz = CM.hz_of(code)
        err.append(hz - true_hz(addr))
        measured.append(_Msg(code, addr))
    s = api.carrier_summary(measured)
    e = np.abs(np.array(err)) if err else np.zeros(0)
    return dict(rate=rate, offset=offset, amp=amp, messages=len(err), aircraft=s["aircraft"],
                median_hz=float(np.median(e)) if e.size else None, p95_hz=float(np.percentile(e, 95)) if e.size else None,
                bias_hz=float(np.mean(err)) if err else None,
                receiver_err_hz=None if s["receiver_hz"] is None else s["receiver_hz"] - receiver_truth_hz(s))


class _Msg:
    """What carrier_summary reads of a message."""

    def __init__(self, code, addr):
        self.code, self.aa1, self.aa2, self.aa3 = code, addr >> 16, (addr >> 8) & 0xFF, addr & 0xFF

    def carrier_hz(self):
        return CM.hz_of(self.code)


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 3000
    C.build_oracle()
    print("| input | amp (LSB) | messages | aircraft | median abs error (Hz) | p95 (Hz) | mean (Hz) | receiver estimate error (Hz) |")
    print("|---|---|---|---|---|---|---|---|")
    for rate, offset in CASES:
        for amp in AMPS:
            r = measure(rate, offset, amp, n)
            what = f"{rate / 1e6:g} MS/s" + (f", offset {offset / 1e6:+g} MHz" if offset else "")
            if not r["messages"]:
                print(f"| {what} | {amp:g} | 0 | 0 | - | - | - | - |")
                continue
            print(f"| {what} | {amp:g} | {r['messages']} | {r['aircraft']} | {r['median_hz']:.0f} | {r['p95_hz']:.0f} | "
                  f"{r['bias_hz']:+.0f} | {r['receiver_err_hz']:+.0f} |")


if __name__ == "__main__":
    main()
