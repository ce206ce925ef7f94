"""CPU comparison behind the input offset (DESIGN §6): true and false DF17 frames the oracle decodes from the
same synthetic fleet at 8 and 10 MS/s, with a zero-IF radio's DC spike, received two ways:
  centred  the channel at 0 Hz, on top of the spike, decoded without an offset (tests/decimate_model.py);
  offset   the radio tuned 2 MHz below the channel (frames sent at carrier_hz = +2 MHz), decoded with
           input_offset = +2 MHz (tests/shift_model.py), which moves the spike to -2 MHz, out of the filter.
The spike is a constant (d, d) / sqrt(2) added to every sample, d at 0, -10 and -20 dB below the frames'
amplitude, or absent.  The fleet's noise is density-matched: snr_db - 10 log10(M) per input sample.

    python scripts/offset_quality.py [--frames 300] [--seeds 2] [--rates 8000000 10000000]

Needs no GPU: the oracle (`make oracle`) and the numpy models.
"""
from __future__ import annotations

import argparse
import sys
from concurrent.futures import ProcessPoolExecutor
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
for p in (str(ROOT), str(ROOT / "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402

import checker  # noqa: E402
import decimate_model as DM  # noqa: E402
import shift_model as SM  # noqa: E402
from dump1090_b200 import synth  # noqa: E402

SNRS = (8, 10, 12, 14, 18)
SPIKES = (None, 0, -10, -20)       # dB below the frame amplitude
AMP = 20.0                         # fleet_at's frame amplitude
OFFSET = 2_000_000


def count(msgs, truth):
    got = [bytes(x.msg[:14]).hex() for x in msgs if x.msgtype == 17 and x.msgbits == 112]
    true = sum(1 for h in got if h in truth)
    return true, len(got) - true


def run(job):
    hz, snr, spike, frames, seed = job
    m = DM.RATES[hz]
    dc = None if spike is None else (AMP * 10 ** (spike / 20) / np.sqrt(2),) * 2
    res = {}
    for case, carrier in (("centred", 0.0), ("offset", float(OFFSET))):
        x, truth = synth.fleet_at_rate(snr - 10 * np.log10(m), frames, seed, sample_rate=hz, carrier_hz=carrier, dc=dc)
        y = DM.decimate(x, m) if carrier == 0 else SM.shift_decimate(x, m, OFFSET)
        res[case] = count(checker.oracle_decode(y)[0], truth)
    return job, res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--seeds", type=int, default=2)
    ap.add_argument("--rates", type=int, nargs="+", default=[8_000_000, 10_000_000])
    args = ap.parse_args()
    checker.build_oracle()
    jobs = [(hz, snr, spike, args.frames, seed) for hz in args.rates for spike in SPIKES for snr in SNRS
            for seed in range(args.seeds)]
    tot = {}
    with ProcessPoolExecutor() as ex:
        for (hz, snr, spike, _, _), res in ex.map(run, jobs):
            for case, (t, f) in res.items():
                a = tot.setdefault((hz, spike, case, snr), [0, 0])
                a[0] += t
                a[1] += f
    n = args.frames * args.seeds
    print(f"true / false DF17 frames of {n} sent, per SNR (dB, density-matched), {args.seeds} seeds")
    print("| rate | DC spike | received | " + " | ".join(f"{s} dB" for s in SNRS) + " |")
    print("|---|---|---|" + "---|" * len(SNRS))
    for hz in args.rates:
        for spike in SPIKES:
            for case in ("centred", "offset"):
                cells = " | ".join(f"{tot[(hz, spike, case, s)][0]} / {tot[(hz, spike, case, s)][1]}" for s in SNRS)
                what = "none" if spike is None else f"{spike} dB"
                recv = "at 0 Hz" if case == "centred" else f"+{OFFSET / 1e6:g} MHz, shifted back"
                print(f"| {hz / 1e6:g} MS/s | {what} | {recv} | {cells} |")


if __name__ == "__main__":
    main()
