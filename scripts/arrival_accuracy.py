"""Accuracy of the arrival-time measurement (modes_set_arrival) on synthetic DF17 frames of known
arrival, on CPU: per amplitude, a stream of N frames (sigma = 1.5, fraction uniform in [0, 1)) is
decoded by the oracle, each delivered message gets the code of the numpy restatement
(tests/arrival_model.py; the GPU computes the same codes, tests/test_arrival.py), and its refined
arrival 6 * sample_pos + code - 8 is compared with the true 6 * (pos + frac) ticks, next to today's
6 * sample_pos.  Usage: arrival_accuracy.py [N] [rate]  (default 2500, 2000000).  A rate of 4000000 ...
10000000 synthesises the same frames at that rate with density-matched noise (sigma 1.5 sqrt(M)) and measures
the oracle's decode of the decimated bytes (tests/decimate_model.py), as the decoder decodes such a stream."""
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
import numpy as np

import checker as C
import decimate_model as DM
import test_arrival as T
from dump1090_b200 import synth


def at_rate(amp, seed, n, m):
    """_known_arrival_stream's frames and truth at 2 M MS/s, decimated to 2 MHz."""
    _, truth = T._known_arrival_stream(amp, seed=seed, n_frames=n)
    rng = synth.Counter(seed)
    frames = []
    for pos, frac, frame in truth:                         # the same carrier phases as the 2 MHz stream
        rng.below(0x3FFFFF)
        for _ in range(7):
            rng.below(256)
        rng.below(100)
        rng.uniform()
        frames.append((pos, frame, amp, 2 * np.pi * rng.uniform(), frac))
    x = synth.synth_stream_at(m * (300 + n * 420 + 500), frames, sigma=1.5 * np.sqrt(m), seed=seed,
                              sample_rate=2_000_000 * m)
    return DM.decimate(x, m), truth


def row(err):
    if not err.size:
        return "- | - | -"
    a = np.abs(err)
    return f"{np.median(a):.2f} | {np.percentile(a, 95):.2f} | {err.mean():+.2f}"


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 2500
    m = DM.RATES.get(int(sys.argv[2]), 1) if len(sys.argv) > 2 else 1
    C.build_oracle()
    print("| amp (LSB) | messages (of which retry) | median abs error | p95 | mean (bias) | 6*sample_pos: median | p95 | mean |")
    print("|---|---|---|---|---|---|---|---|")
    for amp in (6.0, 8.0, 12.0, 20.0, 60.0):
        if m == 1:
            data, truth = T._known_arrival_stream(amp, seed=int(amp) + 3, n_frames=n)
        else:
            data, truth = at_rate(amp, int(amp) + 3, n, m)
        msgs, _ = C.oracle_decode(data)
        fine, coarse, retry = T.arrival_errors(data, truth, msgs)
        print(f"| {amp:g} | {fine.size} ({retry}) | {row(fine)} | {row(coarse)} |")


if __name__ == "__main__":
    main()
