"""The receiver pool with 16-bit receivers (modes_pool_set_input_format): wall clock per step, receivers
held in real time, receiver 0's parity, the upload's share of a step, and the device time of the pool's
conversion launch against its floor.

    python scripts/pool_format_time.py [--receivers 256] [--steps 30] [--warmup 5] [--reps 2]

- Step: as `bench.py --workload receivers`: every step takes one buffer (131072 samples) from each of R
  receivers in one pinned block (receiver r reads buffers r + k), submit(k+1) then collect(k), messages
  into one output array; --no-fix.  Four configurations, alternated over --reps repetitions: all UC8 at
  2 MHz, all SC16 at 2 MHz, all UC8 at 2.4 MS/s, all SC16 at 2.4 MS/s.
- The SC16 captures are the UC8 captures written as int16 (at SC16's default shift, random low bits) so
  that they convert back to the UC8 bytes: both formats resolve the same messages, and the difference
  between them is the upload of twice the bytes and the conversion.
- Real time: a step brings 131072 samples of each receiver, 65.536 ms of a 2 MHz receiver's time and
  54.613 ms of a 2.4 MS/s receiver's; receivers in real time = R x (real time per step) / (wall clock per
  step).
- Upload: the host-to-device rate from pinned memory, measured in the same run, and what one step's
  buffers take at that rate (64 MiB of UC8 or 128 MiB of SC16 at R = 256).
- Parity: receiver 0's messages and statistics against the oracle's decode (no EOF buffer) of its first
  modes_pool_buffers(0) buffers, resampled when it is at 2.4 MS/s.
- Kernel: one more all-SC16 2 MHz run under torch.profiler; convert_pool_kernel's device time per GiB of
  UC8 output, against a floor of 3 bytes moved (4 read, 2 written per sample) per output byte at the
  device-to-device copy rate measured in the same run.
The card's name and power limit are read in the same run.  The capture is random_traffic-style frames at
2.4 MS/s (tests/test_input_rate.traffic24) and the same frames resampled to 2 MHz, tiled.
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
CONFIGS = (("uc8", 2_000_000), ("sc16", 2_000_000), ("uc8", 2_400_000), ("sc16", 2_400_000))


def query(fields: str) -> str:
    q = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={fields}", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def name(cfg) -> str:
    return f"{cfg[0].upper()} at {'2 MHz' if cfg[1] == 2_000_000 else '2.4 MS/s'}"


def run(cfg, pinned, n_rx, steps, warm, profile=False):
    """One timed run; returns (seconds per step, receiver 0's raw lines, its stats, its buffers, kernel times)."""
    import numpy as np
    import torch
    from dump1090_b200 import api

    fmt, hz = cfg
    size = api.BUFFER_BYTES * (1 if fmt == "uc8" else 2)
    ids = np.arange(n_rx, dtype=np.uint32)
    total = steps + warm
    live, raw0 = {}, []
    msg_size = ctypes.sizeof(api.Message)
    kernels = []
    with api.ReceiverPool(n_rx, fix_errors=0, input_rate=hz, input_format=fmt) as pool:
        out, out_rx = pool.set_output_array(n_rx * 400 + 4096)

        def submit(k):
            live[k] = (ctypes.c_void_p * n_rx)(*[pinned.ptr + (r + k) * size for r in range(n_rx)])
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
            kernels = [ev.device_time_total * 1e-3 for ev in prof.events() if "convert_pool_kernel" in ev.name]   # ms
        lines = []
        for blob in raw0:
            arr = (api.Message * (len(blob) // msg_size)).from_buffer_copy(blob)
            lines.extend(m.raw_line() for m in arr)
        return dt / steps, lines, list(pool.stats(0).values()), pool.buffers(0), kernels


def rate_tbs(fn, nbytes, reps=6):
    """Median bytes per second (TB/s) of fn() over CUDA events, the first call left out."""
    import torch

    rates = []
    for k in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        if k:
            rates.append(nbytes / (a.elapsed_time(b) * 1e-3) / 1e12)
    return statistics.median(rates)


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
    import input_format_model as M
    import resample_model as RM
    from dump1090_b200 import api, synth
    from test_input_rate import traffic24

    torch.cuda.set_device(0)
    card = query("name,power.limit")
    n_rx, steps, warm = args.receivers, args.steps, args.warmup
    BUF = api.BUFFER_BYTES
    total = steps + warm
    seed = traffic24(2_000_000, 2000, 9)
    uc8 = {2_400_000: synth.tile_to(seed, (n_rx + total) * BUF), 2_000_000: synth.tile_to(RM.resample(seed), (n_rx + total) * BUF)}
    pinned = {}
    for fmt, hz in CONFIGS:
        x = uc8[hz]
        if fmt == "sc16":
            v = M.to_sc16(x, 8).view("<i2").astype(np.int32) + np.random.default_rng(hz).integers(0, 256, x.size, dtype=np.int32)
            x = v.astype("<i2").view(np.uint8)
            assert np.array_equal(M.convert(x[: 4 * B], 8), uc8[hz][: 2 * B])
        pinned[fmt, hz] = api.PinnedBuffer(x.size)
        pinned[fmt, hz].array[:] = x

    per_step = {c: [] for c in CONFIGS}
    parity = {}
    for rep in range(args.reps):
        for cfg in CONFIGS:
            dt, lines, stats0, k0, _ = run(cfg, pinned[cfg], n_rx, steps, warm)
            per_step[cfg].append(dt)
            if rep == 0:
                x0 = uc8[cfg[1]][: total * BUF]
                y0 = RM.resample_range(x0, 0, k0 * B) if cfg[1] == 2_400_000 else x0[: k0 * BUF]
                exp, exp_stats = checker.oracle_decode(y0, fix=0, drop_eof=1, cap=4_000_000)
                parity[cfg] = (lines == [m.hexline() for m in exp] and stats0 == exp_stats, len(lines), k0)

    # the conversion's device time in a run of its own (tracing slows the host)
    kern = run(("sc16", 2_000_000), pinned["sc16", 2_000_000], n_rx, steps, warm, profile=True)[4]

    # the device-to-device copy rate (read + write) and the host-to-device rate from pinned memory, now
    src = torch.empty(1 << 30, dtype=torch.uint8, device="cuda")
    dst = torch.empty_like(src)
    copy_tbs = rate_tbs(lambda: dst.copy_(src), 2 * src.numel())
    del src, dst
    h = torch.empty(n_rx * 2 * BUF, dtype=torch.uint8).pin_memory()
    d = torch.empty(h.numel(), dtype=torch.uint8, device="cuda")
    h2d_tbs = rate_tbs(lambda: d.copy_(h, non_blocking=True), h.numel())
    del h, d

    print(f"card: {card}")
    print(f"R = {n_rx} receivers, {steps} timed steps after {warm}, {args.reps} alternated repetitions, --no-fix")
    print(f"host-to-device from pinned memory: {h2d_tbs * 1e3:.1f} GB/s; device-to-device copy: {copy_tbs:.2f} TB/s")
    for cfg in CONFIGS:
        real_ms = 1e3 * B / cfg[1]
        med = statistics.median(per_step[cfg])
        ok, n_msgs, k0 = parity[cfg]
        up_ms = n_rx * BUF * (1 if cfg[0] == "uc8" else 2) / (h2d_tbs * 1e12) * 1e3
        print(f"{name(cfg):>15}: {1e3 * med:.3f} ms per step (runs: {', '.join(f'{1e3 * v:.3f}' for v in per_step[cfg])}); "
              f"upload {up_ms:.3f} ms of it at the measured rate; {real_ms:.3f} ms of real time per step -> "
              f"{int(n_rx * real_ms / (1e3 * med))} receivers in real time; "
              f"receiver 0: {k0} buffers, {n_msgs} messages, parity {'ok' if ok else 'FAILED'}")
    if kern:
        out_bytes = n_rx * BUF                                    # every receiver converts one buffer per launch
        k = statistics.median(kern)
        floor = 3 * out_bytes / (copy_tbs * 1e12) * 1e3
        print(f"convert_pool_kernel: median {k:.4f} ms per launch ({len(kern)} launches, min {min(kern):.4f}, max {max(kern):.4f}); "
              f"{k * 2 ** 30 / out_bytes:.3f} ms per GiB of UC8 output; floor {3 * out_bytes / 1e9:.4f} GB over a "
              f"device-to-device copy at {copy_tbs:.2f} TB/s = {floor:.4f} ms -> {k / floor:.2f}x the floor")
    else:
        print("convert_pool_kernel: no device time recorded by the profiler")


if __name__ == "__main__":
    main()
