"""Device time of the recovery pass over the 1 GiB bench workload (bench.py's default stream, --no-fix),
and the end-to-end decode of the same GiB with recovery off and on.

The stream stays resident in HBM.  Two steps run in alternation, each timed with CUDA events on the
context's stream: detect_device alone (recovery off), and detect_device followed by recover_device over
its records (recovery on).  Prints medians and spreads, the time added per GiB, the record counts by
status, and the card's name and power limit read in the same run.  The streaming decode of the GiB from
pinned host memory is timed with the switch off and on in alternation.  Last, the kernel's register and
spill report from ptxas (compiled into a temporary directory)."""
import statistics
import subprocess
import sys
import tempfile
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
import numpy as np
import torch

import bench
from dump1090_b200 import api

WARMUP, STEPS, E2E_REPS = 5, 30, 7
NBUF = (1 << 30) // api.BUFFER_BYTES


def card():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def spread(v):
    return f"median {statistics.median(v):.4f} ms (min {min(v):.4f}, max {max(v):.4f})"


def ptxas_report():
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run(["/usr/local/cuda/bin/nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                            f"-I{ROOT / 'include'}", "-Xptxas", "-v", "-c", str(ROOT / "dump1090_b200/csrc/modes_recover.cu"),
                            "-o", str(Path(d) / "r.o")], capture_output=True, text=True)
    lines = (r.stdout + r.stderr).splitlines()
    return [ln.strip() for ln in lines if "Used" in ln or "spill" in ln]


def main():
    cap, src = bench.load_capture()
    data = np.ascontiguousarray(bench.shard_bytes(cap, 0, 1 << 30))
    d = torch.from_numpy(data).cuda()
    dec = api.Decoder(fix_errors=0)
    stream = torch.cuda.ExternalStream(dec.stream)
    times = {"off": [], "on": []}
    n_cand = 0
    for step in range(WARMUP + STEPS):
        for what in times:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            dec.detect_device(d.data_ptr(), NBUF)
            if what == "on":
                dec.recover_device()
            b.record(stream)
            n_cand = dec.detect_wait()
            b.synchronize()
            if step >= WARMUP:
                times[what].append(a.elapsed_time(b))
    rec = dec.recover_fetch()
    by_status = np.bincount(rec["status"], minlength=4)
    off, on = (statistics.median(times[w]) for w in ("off", "on"))
    # end to end: the same GiB from pinned host memory through the streaming decode
    pin = api.PinnedBuffer(data.size)
    pin.array[:] = data
    dec.set_output_array(1 << 22)
    e2e = {False: [], True: []}
    counts = {}
    for rep in range(E2E_REPS + 1):
        for flag in (False, True):
            dec.set_recovery(flag)
            dec.reset(); dec.rearm_output()
            t0 = time.perf_counter()
            dec.process_ptr(pin.ptr, data.size)
            dec.finish()
            if rep:
                e2e[flag].append((time.perf_counter() - t0) * 1e3)
            counts[flag] = (dec.output_count(), dec.recovery_stats())
    print(f"card: {card()}")
    print(f"stream: {src}, 1 GiB ({NBUF} buffers), --no-fix; {n_cand} candidate records: "
          f"{by_status[0]} ineligible, {by_status[1]} found, {by_status[2]} ambiguous, {by_status[3]} not found")
    print(f"medians of {STEPS} alternating steps after {WARMUP} warm-up steps:")
    print(f"  detect_device:                  {spread(times['off'])}")
    print(f"  detect_device + recover_device: {spread(times['on'])}")
    print(f"  added per GiB: {on - off:.4f} ms")
    print(f"streaming decode of the GiB from pinned memory, median of {E2E_REPS} alternations: recovery off "
          f"{statistics.median(e2e[False]):.2f} ms (min {min(e2e[False]):.2f}, max {max(e2e[False]):.2f}), "
          f"on {statistics.median(e2e[True]):.2f} ms (min {min(e2e[True]):.2f}, max {max(e2e[True]):.2f})")
    print(f"messages off {counts[False][0]}, on {counts[True][0]}; recovery statistics {counts[True][1]}")
    print("ptxas: " + "; ".join(ptxas_report()))
    pin.free()


if __name__ == "__main__":
    main()
