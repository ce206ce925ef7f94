"""Accuracy of the arrival-time measurement (modes_set_arrival) on synthetic DF17 frames of known
arrival, on CPU: per amplitude, a stream of N frames (sigma = 1.5, fraction uniform in [0, 1)) is
decoded by the oracle, each delivered message gets the code of the numpy restatement
(tests/arrival_model.py; the GPU computes the same codes, tests/test_arrival.py), and its refined
arrival 6 * sample_pos + code - 8 is compared with the true 6 * (pos + frac) ticks, next to today's
6 * sample_pos.  Usage: arrival_accuracy.py [N]  (default 2500)."""
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
import numpy as np

import checker as C
import test_arrival as T


def row(err):
    a = np.abs(err)
    return f"{np.median(a):.2f} | {np.percentile(a, 95):.2f} | {err.mean():+.2f}"


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 2500
    C.build_oracle()
    print("| amp (LSB) | messages (of which retry) | median abs error | p95 | mean (bias) | 6*sample_pos: median | p95 | mean |")
    print("|---|---|---|---|---|---|---|---|")
    for amp in (6.0, 8.0, 12.0, 20.0, 60.0):
        data, truth = T._known_arrival_stream(amp, seed=int(amp) + 3, n_frames=n)
        msgs, _ = C.oracle_decode(data)
        fine, coarse, retry = T.arrival_errors(data, truth, msgs)
        print(f"| {amp:g} | {fine.size} ({retry}) | {row(fine)} | {row(coarse)} |")


if __name__ == "__main__":
    main()
