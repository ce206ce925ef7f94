"""Device time of the 2.4 MS/s input resampler (K9, modes_resample.cu), its DRAM floor, and the end-to-end
streaming decode of a 2.4 MS/s capture against the 2 MHz GiB it resamples to.

    python scripts/resample_time.py [--steps 20] [--reps 3] [--rate 2400000] [--format uc8] [--gib 1]

--rate 4000000 ... 10000000 times the integer decimator (K11) instead, on a capture of random_traffic-style
frames at that rate (tests/test_input_decimation.traffic_at); --format sc16 feeds it 16-bit input, whose
kernel time comes from torch.profiler over a streaming decode of the capture (the stage-level entry takes
UC8 only).  --gib: GiB of 2 MHz output (the input is M or 2 M times as large).

- Kernel: modes_resample_device over 1 GiB of 2 MHz output (4096 reference buffers) from the 1.2 GiB of
  2.4 MS/s input it reads, timed with CUDA events; median, min and max over the steps.
- Floor: the bytes it reads and writes over the rate of a device-to-device copy (read + write) of the
  same input, measured in the same run.
- End to end: modes_process + modes_finish of the 1.2 GiB capture from pinned memory at 2.4 MS/s, and of
  the 2 MHz GiB it resamples to (made by the same kernel) at 2 MHz, alternated; wall time per run.
The card's name and power limit are read in the same run.  The capture is random_traffic-style
frames at 2.4 MS/s (tests/test_input_rate.traffic24), tiled.
"""
import argparse
import statistics
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

NBUF = (1 << 30) // 262144
B = 131072


def query(fields: str) -> str:
    q = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={fields}", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def spread(v) -> str:
    return f"median {statistics.median(v):.4f} ms (min {min(v):.4f}, max {max(v):.4f})"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--rate", type=int, default=2_400_000)
    ap.add_argument("--format", default="uc8", choices=["uc8", "sc16"])
    ap.add_argument("--gib", type=float, default=1.0)
    args = ap.parse_args()
    if args.rate != 2_400_000:
        return decimation(args)
    import numpy as np
    import torch

    import resample_model as RM
    from dump1090_b200 import api, synth
    from test_input_rate import traffic24

    card = query("name,power.limit")
    n_out = NBUF * B
    n_in = -(-6 * n_out // 5) + 8
    seed = traffic24(2_000_000, 2000, 9)
    cap = synth.tile_to(seed, 2 * n_in)
    d_in = torch.from_numpy(cap).cuda()
    d_out = torch.empty(2 * n_out, dtype=torch.uint8, device="cuda")
    dec = api.Decoder()
    stream = torch.cuda.Stream()                          # the kernel and the events on one stream
    torch.cuda.set_stream(stream)
    dec.set_stream(stream.cuda_stream)
    times = []
    for k in range(args.steps + 3):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        dec.resample_device(d_in.data_ptr(), d_in.numel(), 0, 0, NBUF, d_out.data_ptr(), want_carry=False)
        b.record()
        b.synchronize()
        if k >= 3:
            times.append(a.elapsed_time(b))
    lo, hi = RM.input_span(-238, n_out + 238)
    read_bytes, write_bytes = 2 * (hi - max(lo, 0)), 2 * n_out + 476
    dst = torch.empty_like(d_in)
    rates = []
    for k in range(6):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        dst.copy_(d_in)
        b.record()
        b.synchronize()
        if k:
            rates.append(2 * d_in.numel() / (a.elapsed_time(b) * 1e-3) / 1e12)
    del dst
    copy_tbs = statistics.median(rates)
    floor_ms = (read_bytes + write_bytes) / (copy_tbs * 1e12) * 1e3
    kern = statistics.median(times)
    # spot check against the model: the first and the last buffer
    torch.cuda.synchronize()
    got = d_out[: 2 * B].cpu().numpy()
    assert np.array_equal(got, RM.resample_range(cap[: 2 * (6 * B // 5 + 8)], 0, B)), "kernel output differs from the model"

    # end to end, alternated: 2.4 MS/s capture vs the 2 MHz GiB it resamples to
    h24 = api.PinnedBuffer(cap.size)
    h24.array[:] = cap
    y = d_out.cpu().numpy()
    h20 = api.PinnedBuffer(y.size)
    h20.array[:] = y
    del d_in, d_out
    torch.cuda.empty_cache()
    e2e = {"2.4 MS/s": [], "2 MHz": []}
    decs = {"2.4 MS/s": api.Decoder(input_rate=2_400_000), "2 MHz": api.Decoder()}
    counts = {}
    for name, dd in decs.items():
        dd.set_output_array(1 << 21)
    for rep in range(args.reps + 1):
        for name, dd in decs.items():
            buf = h24 if name == "2.4 MS/s" else h20
            dd.reset()
            dd.rearm_output()
            t0 = time.perf_counter()
            dd.process_ptr(buf.ptr, buf.nbytes)
            dd.finish()
            t = time.perf_counter() - t0
            counts[name] = dd.output_count()
            if rep:
                e2e[name].append(t * 1e3)
    print(f"card: {card}")
    print(f"K9 resample, {NBUF} buffers (1 GiB of 2 MHz output) from {cap.size / 2**30:.3f} GiB of 2.4 MS/s input: "
          f"{spread(times)}; {2 * n_out / 2**30 / (kern * 1e-3):.1f} GiB/s of output, {kern:.4f} ms per GiB of output")
    print(f"DRAM floor: {read_bytes / 1e9:.4f} GB read + {write_bytes / 1e9:.4f} GB written over a device-to-device "
          f"copy at {copy_tbs:.2f} TB/s (read + write) -> {floor_ms:.4f} ms; kernel {kern / floor_ms:.2f}x the floor")
    for name, v in e2e.items():
        nbytes = h24.nbytes if name == "2.4 MS/s" else h20.nbytes
        med = statistics.median(v)
        print(f"end to end {name}: {spread(v)} for {nbytes / 2**30:.3f} GiB from pinned memory "
              f"({nbytes / 1e9 / (med * 1e-3):.2f} GB/s of input); {counts[name]} messages")


def decimation(args) -> None:
    import numpy as np
    import torch

    import decimate_model as DM
    import input_format_model as IF
    from dump1090_b200 import api, synth
    from test_input_decimation import traffic_at

    m = DM.RATES[args.rate]
    sc16 = args.format == "sc16"
    bps = 4 if sc16 else 2
    card = query("name,power.limit")
    nbuf = int(args.gib * NBUF)
    n_out = nbuf * B
    n_in = m * n_out + 8
    # the UC8 capture; a 16-bit one holds the same samples (input_format_model.to_sc16 at shift 8), so both
    # decimate to the same 2 MHz bytes
    seed = traffic_at(m, "uc8", 2_000_000 * m, 9)
    cap = synth.tile_to(seed, 2 * n_in)
    label = f"{args.rate / 1e6:g} MS/s {args.format.upper()}"
    e, taps = DM.extent(DM.taps(m), m), DM.taps(m).size
    read_bytes, write_bytes = bps * (m * (n_out + 240) + e), 2 * n_out + 480
    d_in = torch.from_numpy(cap).cuda()
    d_out = torch.empty(2 * n_out, dtype=torch.uint8, device="cuda")
    dec = api.Decoder()
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    dec.set_stream(stream.cuda_stream)
    times = []
    for k in range(args.steps + 3):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        dec.resample_device_at(args.rate, d_in.data_ptr(), d_in.numel(), 0, 0, nbuf, d_out.data_ptr(), want_carry=False)
        b.record()
        b.synchronize()
        if k >= 3:
            times.append(a.elapsed_time(b))
    torch.cuda.synchronize()
    got = d_out[: 2 * B].cpu().numpy()
    assert np.array_equal(got, DM.decimate_range(cap[: 2 * (m * B + 8)], m, 0, B)), "kernel output differs from the model"
    y = d_out.cpu().numpy()
    dec.close()
    del d_out
    if sc16:
        del d_in
        cap = synth.tile_to(IF.to_sc16(seed, 8), 4 * n_in)
        d_in = torch.from_numpy(cap).cuda()
    dst = torch.empty_like(d_in)
    rates = []
    for k in range(6):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        dst.copy_(d_in)
        b.record()
        b.synchronize()
        if k:
            rates.append(2 * d_in.numel() / (a.elapsed_time(b) * 1e-3) / 1e12)
    del dst, d_in
    torch.cuda.empty_cache()
    copy_tbs = statistics.median(rates)
    floor_ms = (read_bytes + write_bytes) / (copy_tbs * 1e12) * 1e3

    hm = api.PinnedBuffer(cap.size)
    hm.array[:] = cap
    h20 = api.PinnedBuffer(y.size)
    h20.array[:] = y
    decs = {label: api.Decoder(input_rate=args.rate, input_format=args.format), "2 MHz": api.Decoder()}
    torch.cuda.set_stream(torch.cuda.default_stream())
    if sc16:
        # the kernel's device time from the profiler, over one streaming decode of the capture
        from torch.profiler import ProfilerActivity, profile
        times = []
        dd = decs[label]
        for k in range(min(args.steps, 5) + 1):
            dd.reset()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                dd.process_ptr(hm.ptr, hm.nbytes)
                dd.finish()
                torch.cuda.synchronize()
            us = sum(ev.device_time_total for ev in prof.key_averages() if "decimate_kernel" in ev.key)
            if k:
                times.append(us / 1e3 * nbuf / (nbuf + 1))          # without the EOF buffer's share
    kern = statistics.median(times)
    e2e = {label: [], "2 MHz": []}
    counts = {}
    for dd in decs.values():
        dd.set_output_array(1 << 21)
    for rep in range(args.reps + 1):
        for name, dd in decs.items():
            buf = hm if name == label else h20
            dd.reset()
            dd.rearm_output()
            t0 = time.perf_counter()
            dd.process_ptr(buf.ptr, buf.nbytes)
            dd.finish()
            t = time.perf_counter() - t0
            counts[name] = dd.output_count()
            if rep:
                e2e[name].append(t * 1e3)
    print(f"card: {card}")
    print(f"K11 decimate by {m} (T = {taps}), {nbuf} buffers ({2 * n_out / 2**30:.2f} GiB of 2 MHz output) from "
          f"{cap.size / 2**30:.3f} GiB of {label} input: {spread(times)}; {kern / (2 * n_out / 2**30):.4f} ms per GiB of output")
    print(f"DRAM floor: {read_bytes / 1e9:.4f} GB read + {write_bytes / 1e9:.4f} GB written over a device-to-device "
          f"copy at {copy_tbs:.2f} TB/s (read + write) -> {floor_ms:.4f} ms; kernel {kern / floor_ms:.2f}x the floor")
    for name, v in e2e.items():
        nbytes = hm.nbytes if name == label else h20.nbytes
        med = statistics.median(v)
        print(f"end to end {name}: {spread(v)} for {nbytes / 2**30:.3f} GiB from pinned memory "
              f"({nbytes / 1e9 / (med * 1e-3):.2f} GB/s of input); {counts[name]} messages")


if __name__ == "__main__":
    main()
