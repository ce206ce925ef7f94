"""CPU sweep behind the 2.4 MS/s resampler's filter (DESIGN §6): true and false DF17 frames the oracle
decodes from the 2.4 MS/s fleet after the integer 6:5 resampler, against the native 2 MHz fleet with
the same frames, arrival times and noise per sample, for each SNR and candidate filter; and the
round trip of the modes1.bin head (upsampled 6:5 with scipy, resampled back).

    python scripts/resample_quality.py [--frames 400] [--seeds 3]

Needs no GPU: the oracle (`make oracle`) and the numpy model of the resampler (tests/resample_model.py).
"""
from __future__ import annotations

import argparse
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
for p in (str(ROOT), str(ROOT / "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402

import checker  # noqa: E402
import resample_model as RM  # noqa: E402
from dump1090_b200 import synth  # noqa: E402

FILTERS = [(4, 1.0e6), (6, 0.9e6), (6, 1.0e6), (6, 1.1e6), (6, 1.2e6), (8, 1.0e6), (8, 1.1e6)]


def df17_counts(msgs, truth):
    got = [bytes(m.msg[:14]).hex() for m in msgs if m.msgtype == 17 and m.msgbits == 112]
    true = sum(1 for h in got if h in truth)
    return true, len(got) - true


def upsample_modes1() -> np.ndarray:
    from scipy.signal import resample_poly
    x = checker.modes1().astype(np.float64).reshape(-1, 2) - 127.0
    y = resample_poly(x, 6, 5, axis=0)
    return np.clip(np.rint(y + 127.0), 0, 255).astype(np.uint8).reshape(-1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=400)
    ap.add_argument("--seeds", type=int, default=3)
    args = ap.parse_args()
    checker.build_oracle()
    snrs = list(range(6, 19, 2))
    print("SNR dB | native 2 MHz true/false | " + " | ".join(f"T={t} {fc / 1e6:.1f} MHz true/false" for t, fc in FILTERS))
    tables = {f: RM.derive_taps(*f) for f in FILTERS}
    for snr in snrs:
        nat = [0, 0]
        res = {f: [0, 0] for f in FILTERS}
        for seed in range(args.seeds):
            s2, truth = synth.fleet_at(snr, args.frames, seed)
            t, f = df17_counts(checker.oracle_decode(s2)[0], truth)
            nat[0] += t; nat[1] += f
            s24, _ = synth.fleet_at_rate(snr, args.frames, seed)
            for flt in FILTERS:
                t, f = df17_counts(checker.oracle_decode(RM.resample(s24, tables[flt]))[0], truth)
                res[flt][0] += t; res[flt][1] += f
        print(f"{snr:6d} | {nat[0]:5d}/{nat[1]} | " + " | ".join(f"{res[f][0]:5d}/{res[f][1]}" for f in FILTERS), flush=True)
    print(f"frames sent per SNR: {args.frames * args.seeds}")
    up = upsample_modes1()
    m0, _ = checker.oracle_decode(checker.modes1())
    d0 = {bytes(m.msg[: m.msgbits // 8]).hex() for m in m0}
    print(f"modes1 head at 2 MHz: {len(m0)} messages, {len(d0)} distinct frames")
    for flt in FILTERS:
        m1, _ = checker.oracle_decode(RM.resample(up, tables[flt]))
        d1 = {bytes(m.msg[: m.msgbits // 8]).hex() for m in m1}
        print(f"  T={flt[0]} {flt[1] / 1e6:.1f} MHz round trip: {len(m1)} messages, {len(d1 & d0)} of the {len(d0)} frames, "
              f"{len(d1 - d0)} others")


if __name__ == "__main__":
    main()
