"""Device time the arrival-time measurement adds to the 1 GiB bench workload (bench.py's default
stream, --no-fix), next to the signal-level pass alone and both switches together.

The stream stays resident in HBM; detect_device runs with no pass, signal only, arrival only and both,
in alternation, each step timed with CUDA events on the context's stream.  Prints the medians, what
each switch set adds to the no-pass time, the candidate count, how many attempts were measured and
the spread of their codes, and the card's name and power limit read in the same run."""
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
import numpy as np
import torch

import bench
from dump1090_b200 import api

WARMUP, STEPS = 5, 25
NBUF = (1 << 30) // api.BUFFER_BYTES
SETS = [("none", False, False), ("signal", True, False), ("arrival", False, True), ("both", True, True)]


def card():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def main():
    cap, src = bench.load_capture()
    data = np.ascontiguousarray(bench.shard_bytes(cap, 0, 1 << 30))
    d = torch.from_numpy(data).cuda()
    dec = api.Decoder(fix_errors=0)
    stream = torch.cuda.ExternalStream(dec.stream)
    times = {name: [] for name, _, _ in SETS}
    n_cand = 0
    for step in range(WARMUP + STEPS):
        for name, sig, arr in SETS:
            dec.set_signal(sig)
            dec.set_arrival(arr)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            dec.detect_device(d.data_ptr(), NBUF)
            b.record(stream)
            n_cand = dec.detect_wait()
            b.synchronize()
            if step >= WARMUP:
                times[name].append(a.elapsed_time(b))
    cands, _ = dec.detect_fetch(NBUF)                      # the last step ran with both switches on
    decoded = (cands["p"]["flags"] & api.EVAL_DECODED) != 0
    codes = cands["p"]["flags"][decoded] >> api.EVAL_ARRIVAL_SHIFT
    assert np.all((cands["p"]["flags"][~decoded] >> api.EVAL_ARRIVAL_SHIFT) == 0), "codes only for decoded attempts"
    med = {name: statistics.median(t) for name, t in times.items()}
    print(f"card: {card()}")
    print(f"stream: {src}, 1 GiB, --no-fix; {n_cand} candidates, {int(decoded.sum())} decoded attempts measured")
    print("codes (0 = not measured, else offset + 8):", np.bincount(codes, minlength=16).tolist())
    for name, _, _ in SETS:
        t = times[name]
        print(f"detect_device {name:8s}: median {med[name]:.4f} ms (min {min(t):.4f}, max {max(t):.4f}), "
              f"added {med[name] - med['none']:.4f} ms per GiB")
    k4 = med["signal"] - med["none"]
    if k4 > 0:
        print(f"both / signal alone (added time): {(med['both'] - med['none']) / k4:.2f}")


if __name__ == "__main__":
    main()
