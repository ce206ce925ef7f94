"""Receiver-pool steps fed from GPU memory (modes_pool_submit_device) against the two ways to feed the same
bytes from the host: R receivers, one buffer of each per step, two batches in flight (submit(k + 1), then
collect(k)), timed per step:
  (a) a_device:  CUDA tensors read in place (the rows of one 2-D tensor per step, ReceiverPool.submit);
  (b) b_copy:    the same rows copied to pinned host memory with .copy_() (what a user with I/Q in GPU memory did
                 before), then the host-fed pool;
  (c) c_pinned:  the rows already in pinned host memory, host-fed.
Cases: UC8 and SC16 receivers at 2 MHz and 2.4 MS/s, on dense traffic (about 190 frames per 2 MHz buffer) and
sparse traffic (4).  The three variants alternate, --reps times, each on a fresh pool, and must deliver the
same messages (digest of the shared output array and its receiver ids).  Also: the gather launch's device
time per launch (torch.profiler, a run of its own) against a device-to-device copy of the same bytes (CUDA
events), and the host time of modes_pool_submit_device's pointer checks at R receivers (a call refused at its
last receiver, after R - 1 checks).  Prints one JSON object, and with --out also writes it to that file.

    python scripts/pool_device_time.py [--receivers 256] [--steps 40] [--warmup 4] [--reps 3] [--out FILE]
"""
import argparse
import ctypes
import hashlib
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from dump1090_b200 import api, synth  # noqa: E402

BUF = api.BUFFER_BYTES
B = api.BUFFER_SAMPLES
CYCLE = 8                                  # distinct steps; receiver r reads block rows r + k % CYCLE
UNIQUE = 16                                # distinct buffers of traffic, tiled over the block
FRAMES = {"dense": 190, "sparse": 4}       # frames per 2 MHz buffer


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (x.strip() for x in q.stdout.splitlines()[0].split(","))
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def block(fmt: str, rate: int, traffic: str, rows: int) -> np.ndarray:
    """rows buffers of the case's bytes, one per row (UC8 traffic; SC16 as (x - 127) * 256, which converts back
    to x at SC16's default shift)."""
    n = UNIQUE * B
    if rate == 2_000_000:
        x = synth.random_traffic(n, FRAMES[traffic] * UNIQUE, seed=5)
    else:
        x, _ = synth.fleet_at_rate(20, FRAMES[traffic] * UNIQUE * 5 // 6, 5, sample_rate=rate,
                                   period=max(400, n * 5 // 6 // (FRAMES[traffic] * UNIQUE)))
    x = synth.tile_to(np.ascontiguousarray(x[: 2 * n]), rows * BUF).reshape(rows, BUF)
    if fmt == "uc8":
        return x
    return ((x.astype(np.int16) - 127) * 256).astype("<i2").view(np.uint8).reshape(rows, 2 * BUF)


def run(pool, ids, submit, steps: int, warm: int) -> tuple:
    """(seconds per step, messages, digest) of warm + steps steps, the first warm untimed."""
    import torch
    out, out_rx = pool._out, pool._out_rx
    h = hashlib.sha256()
    msgs = 0

    def collect():
        nonlocal msgs
        pool.rearm_output()
        pool.collect(None)
        n = pool.output_count()
        assert n <= len(out), "message array too small"
        h.update(ctypes.string_at(out, n * ctypes.sizeof(api.Message)))
        h.update(out_rx[:n].tobytes())
        msgs += n

    total = warm + steps
    submit(0)
    for k in range(1, warm + 1):
        submit(k)
        collect()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for k in range(warm + 1, total + 1):
        if k < total:
            submit(k)
        collect()
    return (time.perf_counter() - t0) / steps, msgs, h.hexdigest()[:16]


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--receivers", type=int, default=256)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cases", default="uc8:2000000:dense,uc8:2000000:sparse,sc16:2000000:dense,sc16:2000000:sparse,"
                                       "uc8:2400000:dense,uc8:2400000:sparse,sc16:2400000:dense,sc16:2400000:sparse")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.set_device(0)
    n_rx = args.receivers
    ids = np.arange(n_rx, dtype=np.uint32)
    res = dict(card=card(), receivers=n_rx, steps=args.steps, warmup=args.warmup, reps=args.reps, cases={})
    for case in args.cases.split(","):
        fmt, rate, traffic = case.split(":")
        rate = int(rate)
        x = block(fmt, rate, traffic, n_rx + CYCLE)
        row = x.shape[1]
        dev = torch.from_numpy(x).cuda()
        host = torch.from_numpy(x).pin_memory()
        stage = [torch.empty((n_rx, row), dtype=torch.uint8).pin_memory() for _ in range(2)]
        rows = lambda a, k: [a.data_ptr() + (r + k % CYCLE) * row for r in range(n_rx)]   # noqa: E731
        host_ptrs = [(ctypes.c_void_p * n_rx)(*rows(host, k)) for k in range(CYCLE)]
        stage_ptrs = [(ctypes.c_void_p * n_rx)(*[s.data_ptr() + r * row for r in range(n_rx)]) for s in stage]
        torch.cuda.synchronize()

        def make():
            pool = api.ReceiverPool(n_rx, max_batch=n_rx, input_rate=rate, input_format=fmt)
            pool.set_output_array(n_rx * 600 + 4096)
            return pool

        def variant(name, pool):
            if name == "a_device":
                return lambda k: pool.submit(ids, dev[k % CYCLE: k % CYCLE + n_rx])

            if name == "b_copy":
                def sub(k):
                    stage[k & 1].copy_(dev[k % CYCLE: k % CYCLE + n_rx])
                    pool.submit_ptrs(ids, stage_ptrs[k & 1])
                return sub
            return lambda k: pool.submit_ptrs(ids, host_ptrs[k % CYCLE])

        names = ("a_device", "b_copy", "c_pinned")
        times = {k: [] for k in names}
        outs = {}
        for rep in range(args.reps + 1):                               # rep 0 warms every path
            for name in names:
                with make() as pool:
                    dt, n_msgs, dig = run(pool, ids, variant(name, pool), args.steps, args.warmup)
                if rep:
                    times[name].append(dt * 1e3)
                outs.setdefault((n_msgs, dig), []).append(name)
        assert len(outs) == 1, (case, outs)
        (n_msgs, dig), = outs
        buffer_s = B / rate                                            # input time one buffer covers
        c = dict(format=fmt, rate=rate, traffic=traffic, messages_per_run=n_msgs, digest=dig, parity=True,
                 ms_per_step={k: dict(median=statistics.median(t), min=min(t), max=max(t), runs=t) for k, t in times.items()},
                 receivers_real_time={k: n_rx * buffer_s * 1e3 / statistics.median(t) for k, t in times.items()})
        if rate == 2_000_000:
            # the gather launch's device time per launch, in a profiled run of (a)
            with make() as pool:
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    run(pool, ids, variant("a_device", pool), args.steps, 1)
                    torch.cuda.synchronize()
            g = [e for e in prof.key_averages() if "gather_pool_kernel" in e.key]
            c["gather_us_per_launch"] = g[0].self_device_time_total / g[0].count if g else None
            c["gather_launches"] = g[0].count if g else 0
            # a device-to-device copy of the bytes the gather moves (UC8: every buffer; SC16: the carries only)
            nbytes = n_rx * BUF if fmt == "uc8" else n_rx * api.CARRY_BYTES * 2
            a, b = torch.empty(nbytes, dtype=torch.uint8, device="cuda"), torch.empty(nbytes, dtype=torch.uint8, device="cuda")
            for _ in range(5):
                b.copy_(a)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(100):
                b.copy_(a)
            e1.record()
            torch.cuda.synchronize()
            c["d2d_copy_floor_us"] = e0.elapsed_time(e1) * 1e3 / 100
            c["gather_bytes_moved"] = nbytes
        if fmt == "uc8" and rate == 2_000_000:
            # modes_pool_submit_device's checks at n_rx receivers: a call refused at the last one's alignment
            with make() as pool:
                ptrs = rows(dev, 0)
                ptrs[-1] += 4
                arr = (ctypes.c_void_p * n_rx)(*ptrs)
                L = api.lib()
                for _ in range(10):
                    L.modes_pool_submit_device(pool._h, api._ptr(ids), arr, n_rx)
                t0 = time.perf_counter()
                for _ in range(200):
                    assert L.modes_pool_submit_device(pool._h, api._ptr(ids), arr, n_rx) == -1
                c["pointer_checks_us"] = (time.perf_counter() - t0) / 200 * 1e6
                assert b"not 16-byte aligned" in L.modes_pool_last_error(pool._h)
                view = dev[:n_rx]
                t0 = time.perf_counter()
                for _ in range(200):
                    pool._device_buffers(ids, view)
                c["python_tensor_checks_us"] = (time.perf_counter() - t0) / 200 * 1e6
        res["cases"][case] = c
        del dev, host, stage
        torch.cuda.empty_cache()
        print(json.dumps({case: c}), file=sys.stderr, flush=True)
    out = json.dumps(res)
    print(out)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(out + "\n")


if __name__ == "__main__":
    main()
