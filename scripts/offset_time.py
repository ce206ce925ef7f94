"""Device time of the shifted decimator (K12, modes_set_input_offset) against the unshifted one (K11) and the
device-to-device copy floor, and the end-to-end streaming decode with and without an offset.

    python scripts/offset_time.py [--steps 20] [--gib 0.5] [--e2e-gib 0.25]

- UC8, every M: modes_resample_device_shift over --gib GiB of 2 MHz output at offset 0 (K11's kernel), at
  the rate's largest offset and at an odd one, alternated step by step, timed with CUDA events; median, min
  and max.  The floor is the bytes the kernel reads and writes over the rate of a device-to-device copy of
  the same input, measured in the same run.
- End to end, SC16 and UC8 at M = 2 and 5: modes_process + modes_finish of --e2e-gib GiB of 2 MHz output's
  capture from pinned memory, at offset 0 and at the largest offset, each capture's frames sent at the offset
  it is decoded with; wall time of the last three of four runs, and the decimator's device time from
  torch.profiler over one more (for SC16 the only way to time it: the stage-level entry takes UC8 only).
The card's name and power limit are read in the same run.  The captures are random_traffic-style frames
with a DC spike (tests/test_input_offset.traffic_off), tiled.
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
    ap.add_argument("--gib", type=float, default=0.5)
    ap.add_argument("--e2e-gib", type=float, default=0.25)
    args = ap.parse_args()
    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile

    import decimate_model as DM
    import input_format_model as IF
    import shift_model as SM
    from dump1090_b200 import api, synth
    from test_input_offset import traffic_off

    print(f"card: {query('name,power.limit')}")
    dec = api.Decoder()
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    dec.set_stream(stream.cuda_stream)
    for hz, m in DM.RATES.items():
        nbuf = int(args.gib * (1 << 30) // (2 * B))
        n_out = nbuf * B
        seed = traffic_off(m, "uc8", 1e6, 2_000_000 * m, 9)
        cap = synth.tile_to(seed, 2 * (m * n_out + 8))
        d_in = torch.from_numpy(cap).cuda()
        d_out = torch.empty(2 * n_out, dtype=torch.uint8, device="cuda")
        mx = SM.max_offset(hz)
        cases = {"offset 0 (K11)": 0, f"offset {mx}": mx, "offset 765433": 765_433, "offset -313373": -313_373}
        times = {c: [] for c in cases}
        for k in range(args.steps + 2):
            for c, o in cases.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                dec.resample_device_shift(hz, o, d_in.data_ptr(), d_in.numel(), 0, 0, nbuf, d_out.data_ptr(),
                                          want_carry=False)
                b.record()
                b.synchronize()
                if k >= 2:
                    times[c].append(a.elapsed_time(b))
                if k == 0:
                    got = d_out[: 2 * B].cpu().numpy()
                    assert np.array_equal(got, SM.shift_decimate_range(cap[: 2 * (m * B + 8)], m, o, 0, B)), (hz, o)
        dst = torch.empty_like(d_in)
        rates = []
        for k in range(6):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            dst.copy_(d_in)
            b.record()
            b.synchronize()
            if k:
                rates.append(2 * d_in.numel() / (a.elapsed_time(b) * 1e-3))
        floor = (2 * m * n_out + 2 * n_out) / statistics.median(rates) * 1e3
        gib = 2 * n_out / (1 << 30)
        base = statistics.median(times["offset 0 (K11)"])
        print(f"{hz / 1e6:g} MS/s UC8: floor {floor / gib:.3f} ms/GiB out")
        for c, v in times.items():
            med = statistics.median(v)
            print(f"  {c:>18}: {med / gib:.3f} ms/GiB out, {med / base:.3f}x K11, {med / floor:.3f}x floor  [{spread(v)}]")
        del d_in, d_out, dst
        torch.cuda.empty_cache()
    dec.close()
    torch.cuda.set_stream(torch.cuda.default_stream())

    for m, fmt in ((2, "sc16"), (5, "sc16"), (2, "uc8"), (5, "uc8")):
        hz = 2_000_000 * m
        mx = SM.max_offset(hz)
        bps = 4 if fmt == "sc16" else 2
        nbytes = int(args.e2e_gib * (1 << 30)) * m * bps // 2
        res = {}
        for o in (0, mx):
            # the same traffic sent at the offset the decoder is told, so both decode the same frames
            seed = traffic_off(m, "uc8", float(o), 2_000_000 * m, 9)
            cap = synth.tile_to(IF.to_sc16(seed, 8) if fmt == "sc16" else seed, nbytes)
            hm = api.PinnedBuffer(cap.size)
            hm.array[:] = cap
            d = api.Decoder(input_rate=hz, input_format=fmt, input_offset=o)
            wall = []
            for k in range(4):
                d.reset()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                d.process_ptr(hm.ptr, hm.nbytes)
                d.finish()
                wall.append((time.perf_counter() - t0) * 1e3)
                n = len(d.take_messages())
            d.reset()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                d.process_ptr(hm.ptr, hm.nbytes)
                d.finish()
                torch.cuda.synchronize()
            d.take_messages()
            us = sum(ev.device_time_total for ev in prof.key_averages() if "decimate_kernel" in ev.key)
            res[o] = (us / 1e3, wall[1:], n)
            d.close()
            hm.free()
        gib_out = nbytes / bps / m * 2 / (1 << 30)
        print(f"{hz / 1e6:g} MS/s {fmt.upper()} end to end, {nbytes / (1 << 30):.2f} GiB of input from pinned memory:")
        for o, (kern, wall, n) in res.items():
            print(f"  offset {o:>8}: decimator {kern / gib_out:.3f} ms/GiB out (profiler), decode {spread(wall)}, "
                  f"{nbytes / (1 << 30) / (statistics.median(wall) / 1e3):.1f} GiB/s of input, {n} messages")


if __name__ == "__main__":
    main()
