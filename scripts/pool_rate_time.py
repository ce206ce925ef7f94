"""The receiver pool with 2.4 MS/s receivers (modes_pool_set_input_rate): wall clock per step, receivers
held in real time, receiver 0's parity, and the device time of the pool's resampling launch against its
DRAM floor.

    python scripts/pool_rate_time.py [--receivers 256] [--steps 30] [--warmup 5] [--reps 2]

- Step: as `bench.py --workload receivers`: every step takes one MODES_BUFFER_BYTES buffer from each of R
  receivers in one pinned block (receiver r reads buffers r + k), submit(k+1) then collect(k), messages
  into one output array; --no-fix.  Three mixes: all 2 MHz, all 2.4 MS/s, and half / half (even
  receivers at 2.4 MS/s), alternated over --reps repetitions.
- Real time: a step brings 131072 input samples of each receiver, 65.536 ms of a 2 MHz receiver's time
  and 54.613 ms of a 2.4 MS/s receiver's; receivers in real time = R x (real time per step) / (wall
  clock per step), with the mix's mean real time per step.
- Parity: receiver 0's messages and statistics against the oracle's decode (no EOF buffer) of its
  first modes_pool_buffers(0) buffers, resampled when it is at 2.4 MS/s.
- Kernel: one more all-2.4 MS/s run, under torch.profiler; the resampling launch's (and the history step's)
  device time per GiB of 2 MHz output, against the bytes they read and write over a device-to-device
  copy rate measured in the same run.
The card's name and power limit are read in the same run.  The capture is random_traffic-style frames
at 2.4 MS/s (tests/test_input_rate.traffic24), tiled.  The all-2 MHz run reads the same frames resampled
to 2 MHz (the model's bytes, tiled), so that both runs resolve about as many messages; in the half / half
run every receiver reads the 2.4 MS/s bytes, and the 2 MHz receivers decode next to nothing from them.
"""
import argparse
import ctypes
import statistics
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

B = 131072
MIXES = ("2 MHz", "2.4 MS/s", "half / half")


def query(fields: str) -> str:
    q = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={fields}", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def rates_of(mix: str, n_rx: int):
    if mix == "2 MHz":
        return [2_000_000] * n_rx
    if mix == "2.4 MS/s":
        return [2_400_000] * n_rx
    return [2_000_000 if r % 2 else 2_400_000 for r in range(n_rx)]


def run(mix, pinned, n_rx, steps, warm, profile=False):
    """One timed run; returns (seconds per step, receiver 0's raw lines, its stats, its buffers, kernel times)."""
    import numpy as np
    import torch
    from dump1090_b200 import api

    BUF = api.BUFFER_BYTES
    ids = np.arange(n_rx, dtype=np.uint32)
    total = steps + warm
    live, raw0 = {}, []
    msg_size = ctypes.sizeof(api.Message)
    kernels = {}
    with api.ReceiverPool(n_rx, fix_errors=0) as pool:
        for r, hz in enumerate(rates_of(mix, n_rx)):
            pool.set_input_rate(r, hz)
        out, out_rx = pool.set_output_array(n_rx * 400 + 4096)

        def submit(k):
            live[k] = (ctypes.c_void_p * n_rx)(*[pinned.ptr + (r + k) * BUF for r in range(n_rx)])
            pool.submit_ptrs(ids, live[k])

        def collect(k):
            pool.rearm_output()
            pool.collect(None)
            del live[k]
            n = pool.output_count()
            assert n <= len(out), "message array too small"
            m0 = int(np.searchsorted(out_rx[:n], 1))
            raw0.append(ctypes.string_at(out, m0 * msg_size))

        submit(0)
        for k in range(1, warm + 1):
            submit(k)
            collect(k - 1)
        torch.cuda.synchronize()
        prof = None
        if profile:
            prof = torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA])
            prof.__enter__()
        t0 = time.perf_counter()
        for k in range(warm + 1, total + 1):
            if k < total:
                submit(k)
            collect(k - 1)
        dt = time.perf_counter() - t0
        if prof is not None:
            torch.cuda.synchronize()
            prof.__exit__(None, None, None)
            for ev in prof.events():
                for key in ("resample_pool_kernel", "history_pool_kernel"):
                    if key in ev.name:
                        kernels.setdefault(key, []).append(ev.device_time_total * 1e-3)   # ms
        lines = []
        for blob in raw0:
            arr = (api.Message * (len(blob) // msg_size)).from_buffer_copy(blob)
            lines.extend(m.raw_line() for m in arr)
        return dt / steps, lines, list(pool.stats(0).values()), pool.buffers(0), kernels


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--receivers", type=int, default=256)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    import numpy as np
    import torch

    import checker
    import pool_rate_model as PM
    import resample_model as RM
    from dump1090_b200 import api, synth
    from test_input_rate import traffic24

    torch.cuda.set_device(0)
    card = query("name,power.limit")
    n_rx, steps, warm = args.receivers, args.steps, args.warmup
    BUF = api.BUFFER_BYTES
    total = steps + warm
    seed = traffic24(2_000_000, 2000, 9)
    pinned = {"2.4 MS/s": api.PinnedBuffer((n_rx + total) * BUF), "2 MHz": api.PinnedBuffer((n_rx + total) * BUF)}
    pinned["2.4 MS/s"].array[:] = synth.tile_to(seed, (n_rx + total) * BUF)
    pinned["2 MHz"].array[:] = synth.tile_to(RM.resample(seed), (n_rx + total) * BUF)
    pinned["half / half"] = pinned["2.4 MS/s"]

    per_step = {m: [] for m in MIXES}
    parity = {}
    for rep in range(args.reps):
        for mix in MIXES:
            dt, lines, stats0, k0, _ = run(mix, pinned[mix], n_rx, steps, warm)
            per_step[mix].append(dt)
            if rep == 0:
                x0 = pinned[mix].array[: total * BUF]
                y0 = RM.resample_range(x0, 0, k0 * B) if rates_of(mix, n_rx)[0] == 2_400_000 else x0[: k0 * BUF]
                exp, exp_stats = checker.oracle_decode(y0, fix=0, drop_eof=1, cap=4_000_000)
                parity[mix] = (lines == [m.hexline() for m in exp] and stats0 == exp_stats, len(lines), k0)

    # the kernels' device time in a run of its own (tracing slows the host)
    kernels = run("2.4 MS/s", pinned["2.4 MS/s"], n_rx, steps, warm, profile=True)[4]

    # the device-to-device copy rate (read + write), measured now
    src = torch.empty(1 << 30, dtype=torch.uint8, device="cuda")
    dst = torch.empty_like(src)
    rates = []
    for k in range(6):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        dst.copy_(src)
        b.record()
        b.synchronize()
        if k:
            rates.append(2 * src.numel() / (a.elapsed_time(b) * 1e-3) / 1e12)
    del src, dst
    copy_tbs = statistics.median(rates)

    print(f"card: {card}")
    print(f"R = {n_rx} receivers, {steps} timed steps after {warm}, {args.reps} alternated repetitions, --no-fix")
    for mix in MIXES:
        rr = rates_of(mix, n_rx)
        real_ms = statistics.mean(1e3 * B / hz for hz in rr)
        med = statistics.median(per_step[mix])
        ok, n_msgs, k0 = parity[mix]
        print(f"{mix:>12}: {1e3 * med:.3f} ms per step (runs: {', '.join(f'{1e3 * v:.3f}' for v in per_step[mix])}); "
              f"{real_ms:.3f} ms of real time per step -> {int(n_rx * real_ms / (1e3 * med))} receivers in real time; "
              f"receiver 0: {k0} buffers, {n_msgs} messages, parity {'ok' if ok else 'FAILED'}")
    rs = kernels.get("resample_pool_kernel", [])
    hs = kernels.get("history_pool_kernel", [])
    if rs:
        # the all-2.4 MS/s receivers run in lock step: a launch has a job for every receiver (the calls in
        # which none completes a buffer launch no resampling)
        jobs = n_rx
        lo, hi = RM.input_span(-238, B + 238)
        out_bytes = jobs * (2 * B)
        rd, wr = jobs * 2 * (hi - lo), jobs * (2 * B + 476)
        kern = statistics.median(rs)
        floor = (rd + wr) / (copy_tbs * 1e12) * 1e3
        per_gib = kern * (2 ** 30 / out_bytes)
        print(f"resample_pool_kernel: median {kern:.4f} ms per launch ({len(rs)} launches, min {min(rs):.4f}, max {max(rs):.4f}); "
              f"{per_gib:.3f} ms per GiB of 2 MHz output; floor {(rd + wr) / 1e9:.4f} GB over a device-to-device copy at "
              f"{copy_tbs:.2f} TB/s = {floor:.4f} ms -> {kern / floor:.2f}x the floor")
    if hs:
        # the bytes a history step reads and writes, averaged over 60 calls of the pool's schedule
        kept = [call0 + BUF - keep for _, call0, _, _, keep in PM.receiver_calls(60)]
        hist_bytes = n_rx * 2 * statistics.mean(kept)
        kern = statistics.median(hs)
        print(f"history_pool_kernel: median {kern:.4f} ms per launch ({len(hs)} launches); "
              f"{hist_bytes / 1e9:.4f} GB read + written -> floor {hist_bytes / (copy_tbs * 1e12) * 1e3:.4f} ms")
    if not rs:
        print("resample_pool_kernel: no device time recorded by the profiler")


if __name__ == "__main__":
    main()
