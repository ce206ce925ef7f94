"""Device time the signal-level pass adds to the 1 GiB bench workload (bench.py's default stream,
--no-fix), and the end-to-end decode of the same GiB with the pass off and on.

The stream stays resident in HBM; detect_device runs with signal measurement off and on in
alternation, each step timed with CUDA events on the context's stream.  Prints the medians, their
difference, the candidate count and how many attempts the pass measured, and the card's name and
power limit read in the same run."""
import statistics
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
import numpy as np
import torch

import bench
from dump1090_b200 import api

WARMUP, STEPS, E2E_REPS = 5, 25, 5
NBUF = (1 << 30) // api.BUFFER_BYTES


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
    times = {False: [], True: []}
    n_cand = 0
    for step in range(WARMUP + STEPS):
        for on in (False, True):
            dec.set_signal(on)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            dec.detect_device(d.data_ptr(), NBUF)
            b.record(stream)
            n_cand = dec.detect_wait()
            b.synchronize()
            if step >= WARMUP:
                times[on].append(a.elapsed_time(b))
    cands, _ = dec.detect_fetch(NBUF)                      # the last step ran with the pass on
    decoded = (cands["p"]["flags"] & api.EVAL_DECODED) != 0
    measured = int(decoded.sum())
    assert np.all((cands["p"]["signal"] > 0) == decoded), "signal written exactly for the decoded attempts"
    off, on = statistics.median(times[False]), statistics.median(times[True])
    # end to end: the same GiB from pinned host memory through the streaming decode
    pin = api.PinnedBuffer(data.size)
    pin.array[:] = data
    dec.set_output_array(1 << 20)
    e2e = {False: [], True: []}
    for rep in range(E2E_REPS + 1):
        for flag in (False, True):
            dec.set_signal(flag)
            dec.reset(); dec.rearm_output()
            t0 = time.perf_counter()
            dec.process_ptr(pin.ptr, data.size)
            dec.finish()
            if rep:
                e2e[flag].append((time.perf_counter() - t0) * 1e3)
    print(f"card: {card()}")
    print(f"stream: {src}, 1 GiB, --no-fix; {n_cand} candidates, {measured} decoded attempts measured")
    print(f"detect_device, median of {STEPS}: signal off {off:.4f} ms, on {on:.4f} ms, added {on - off:.4f} ms per GiB")
    print(f"  off: min {min(times[False]):.4f} max {max(times[False]):.4f}; on: min {min(times[True]):.4f} max {max(times[True]):.4f}")
    print(f"streaming decode of the GiB from pinned memory, median of {E2E_REPS}: off {statistics.median(e2e[False]):.2f} ms, "
          f"on {statistics.median(e2e[True]):.2f} ms")
    pin.free()


if __name__ == "__main__":
    main()
