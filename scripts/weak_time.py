"""Device time of the weak-preamble passes over the 1 GiB bench workload (bench.py's default stream,
--no-fix), and the end-to-end decode of the same GiB with the switch off and on.

The stream stays resident in HBM.  Three steps run in alternation, each timed with CUDA events on the
context's stream: detect_device alone, detect_device + recover_device (recovery), and detect_device +
recover_device + weak_device (recovery at weak preambles too).  Prints medians and spreads, the time
each adds per GiB, the weak-position count, and the card's name and power limit read in the same run.
The streaming decode of the GiB from pinned host memory is timed with recovery on and the weak switch
off and on in alternation.  Then, in a run of its own, torch.profiler gives the device time of each
kernel of the weak passes (and of the recovery search over the candidates, for comparison).  Last, the
kernels' register and spill report from ptxas (compiled into a temporary directory)."""
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
    out = []
    with tempfile.TemporaryDirectory() as d:
        for src in ("modes_weak.cu", "modes_recover.cu"):
            r = subprocess.run(["/usr/local/cuda/bin/nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                                f"-I{ROOT / 'include'}", "-Xptxas", "-v", "-c", str(ROOT / "dump1090_b200/csrc" / src),
                                "-o", str(Path(d) / "r.o")], capture_output=True, text=True)
            out += [ln.strip() for ln in (r.stdout + r.stderr).splitlines()
                    if "Used" in ln or "spill" in ln or "Compiling entry" in ln]
    return out


KERNELS = ("weak_scan_kernel", "weak_order_kernel", "weak_gather_kernel", "recover_weak_kernel", "recover_kernel(")


def kernel_split(dec, d, steps=10):
    """Mean device time per launch of each kernel of the weak passes, from a profiled run of its own."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(2):
        dec.detect_device(d.data_ptr(), NBUF); dec.recover_device(); dec.weak_device(); dec.weak_fetch()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            dec.detect_device(d.data_ptr(), NBUF); dec.recover_device(); dec.weak_device(); dec.weak_fetch()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        for k in KERNELS:
            if k in ev.key and ev.count:
                t = getattr(ev, "device_time_total", None)
                if t is None:
                    t = ev.cuda_time_total
                out[k.rstrip("(")] = (t / ev.count / 1e3, ev.count)
    return out


def main():
    cap, src = bench.load_capture()
    data = np.ascontiguousarray(bench.shard_bytes(cap, 0, 1 << 30))
    d = torch.from_numpy(data).cuda()
    dec = api.Decoder(fix_errors=0)
    stream = torch.cuda.ExternalStream(dec.stream)
    times = {"detect": [], "recover": [], "weak": []}
    n_cand = 0
    for step in range(WARMUP + STEPS):
        for what in times:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            dec.detect_device(d.data_ptr(), NBUF)
            if what != "detect":
                dec.recover_device()
            if what == "weak":
                dec.weak_device()
            b.record(stream)
            n_cand = dec.detect_wait()
            b.synchronize()
            if step >= WARMUP:
                times[what].append(a.elapsed_time(b))
    n_weak, _, wrec = dec.weak_fetch()
    by_status = np.bincount(wrec["status"], minlength=4)
    base, rec_on, weak_on = (statistics.median(times[w]) for w in ("detect", "recover", "weak"))
    # end to end: the same GiB from pinned host memory through the streaming decode
    pin = api.PinnedBuffer(data.size)
    pin.array[:] = data
    dec.set_output_array(1 << 22)
    e2e = {False: [], True: []}
    counts = {}
    dec.set_recovery(True)
    for rep in range(E2E_REPS + 1):
        for flag in (False, True):
            dec.set_weak_preambles(flag)
            dec.reset(); dec.rearm_output()
            t0 = time.perf_counter()
            dec.process_ptr(pin.ptr, data.size)
            dec.finish()
            if rep:
                e2e[flag].append((time.perf_counter() - t0) * 1e3)
            counts[flag] = (dec.output_count(), dec.recovery_stats(), dec.weak_recovery_stats())
    print(f"card: {card()}")
    print(f"stream: {src}, 1 GiB ({NBUF} buffers), --no-fix; {n_cand} candidate records; {n_weak} weak positions: "
          f"{by_status[1]} found, {by_status[2]} ambiguous, {by_status[3]} not found")
    print(f"medians of {STEPS} alternating steps after {WARMUP} warm-up steps:")
    print(f"  detect_device:                                {spread(times['detect'])}")
    print(f"  detect_device + recover_device:               {spread(times['recover'])}")
    print(f"  detect_device + recover_device + weak_device: {spread(times['weak'])}")
    print(f"  recovery adds {rec_on - base:.4f} ms per GiB, weak preambles {weak_on - rec_on:.4f} ms more")
    print(f"streaming decode of the GiB from pinned memory with recovery, median of {E2E_REPS} alternations: weak off "
          f"{statistics.median(e2e[False]):.2f} ms (min {min(e2e[False]):.2f}, max {max(e2e[False]):.2f}), "
          f"on {statistics.median(e2e[True]):.2f} ms (min {min(e2e[True]):.2f}, max {max(e2e[True]):.2f})")
    print(f"messages off {counts[False][0]}, on {counts[True][0]}; recovery statistics {counts[True][1]}; "
          f"weak statistics {counts[True][2]}")
    split = kernel_split(dec, d)
    print("device time per launch (torch.profiler, 10 steps, a run of its own): " +
          ", ".join(f"{k} {ms:.4f} ms" for k, (ms, _) in split.items()))
    print("ptxas: " + "; ".join(ptxas_report()))
    pin.free()


if __name__ == "__main__":
    main()
