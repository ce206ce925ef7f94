"""Device time of the level pass over the 1 GiB bench workload (bench.py's default stream, --no-fix),
and the end-to-end decode of the same GiB with levels off and on.

The stream stays resident in HBM.  Three steps run in alternation, each timed with CUDA events on the
context's stream: detect_device alone (levels off), detect_device followed by levels_device over the
same buffers (levels on), and levels_device alone (the kernel by itself).  Prints medians and spreads,
the time added per GiB, the bandwidth the kernel reaches, and the card's name and power limit read in
the same run.  The streaming decode of the GiB from pinned host memory is timed with the switch off
and on in alternation."""
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


def spread(v):
    return f"median {statistics.median(v):.4f} ms (min {min(v):.4f}, max {max(v):.4f})"


def main():
    cap, src = bench.load_capture()
    data = np.ascontiguousarray(bench.shard_bytes(cap, 0, 1 << 30))
    d = torch.from_numpy(data).cuda()
    dec = api.Decoder(fix_errors=0)
    stream = torch.cuda.ExternalStream(dec.stream)
    times = {"off": [], "on": [], "kernel": []}
    for step in range(WARMUP + STEPS):
        for what in times:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            if what != "kernel":
                dec.detect_device(d.data_ptr(), NBUF)
            if what != "off":
                dec.levels_device(d.data_ptr(), NBUF)
            b.record(stream)
            if what != "kernel":
                dec.detect_wait()
            b.synchronize()
            if step >= WARMUP:
                times[what].append(a.elapsed_time(b))
    summary = api.level_summary(dec.levels_fetch())
    off, on, k = (statistics.median(times[w]) for w in ("off", "on", "kernel"))
    # end to end: the same GiB from pinned host memory through the streaming decode
    pin = api.PinnedBuffer(data.size)
    pin.array[:] = data
    dec.set_output_array(1 << 20)
    e2e = {False: [], True: []}
    for rep in range(E2E_REPS + 1):
        for flag in (False, True):
            dec.set_levels(flag)
            dec.reset(); dec.rearm_output()
            t0 = time.perf_counter()
            dec.process_ptr(pin.ptr, data.size)
            dec.finish()
            if rep:
                e2e[flag].append((time.perf_counter() - t0) * 1e3)
            assert dec.take_levels().size == (NBUF + 1 if flag else 0)
    print(f"card: {card()}")
    print(f"stream: {src}, 1 GiB ({NBUF} buffers), --no-fix; noise {summary['noise_dbfs']:.2f} dBFS, "
          f"peak {summary['peak_dbfs']:.2f} dBFS, {summary['clipped']} clipped samples")
    print(f"medians of {STEPS} steps after {WARMUP} warm-up steps:")
    print(f"  detect_device:                 {spread(times['off'])}")
    print(f"  detect_device + levels_device: {spread(times['on'])}")
    print(f"  levels_device alone:           {spread(times['kernel'])} = {(1 << 30) / k / 1e9:.2f} TB/s")
    print(f"  added per GiB: {on - off:.4f} ms")
    print(f"streaming decode of the GiB from pinned memory, median of {E2E_REPS}: levels off "
          f"{statistics.median(e2e[False]):.2f} ms (min {min(e2e[False]):.2f}, max {max(e2e[False]):.2f}), "
          f"on {statistics.median(e2e[True]):.2f} ms (min {min(e2e[True]):.2f}, max {max(e2e[True]):.2f})")
    pin.free()


if __name__ == "__main__":
    main()
