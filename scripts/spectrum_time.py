"""Time of the input spectrum pass (K13, modes_set_spectrum) on the GPU: the kernel's device time per GiB of
2 MHz output at 2 MHz UC8, 2.4 MS/s UC8 and 10 MS/s SC16, against the device-copy floor of the input span it
reads, and the end-to-end decode with and without the switch.  Kernel times come from torch.profiler (CUDA
activity, kernels named spectrum_kernel); the floor is the time to read the input bytes once at the HBM
traffic a device-to-device copy reaches in the same run (twice the bytes it copies: each is read and
written).  Prints one JSON object, and with --out also writes it to that file.

    python scripts/spectrum_time.py [--buffers 256] [--reps 5] [--out FILE]
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path


ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from dump1090_b200 import api, synth  # noqa: E402

CASES = [(2_000_000, "uc8"), (2_400_000, "uc8"), (10_000_000, "sc16")]


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (x.strip() for x in q.stdout.splitlines()[0].split(","))
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def stream(rate, fmt, n_buffers):
    """n_buffers 2 MHz buffers of traffic at the rate and format (a synthetic capture tiled)."""
    x, _ = synth.fleet_at_rate(20, 300, 7, sample_rate=rate, dtype="uc8" if fmt == "uc8" else "sc16",
                               scale=256.0 if fmt == "sc16" else 1.0)
    bps = 2 if fmt == "uc8" else 4
    n_in = api.BUFFER_BYTES // 2 * n_buffers * rate // 2_000_000
    return synth.tile_to(x, n_in * bps)


def copy_rate(nbytes) -> float:
    """Bytes per second of a device-to-device copy of nbytes (read + write counted once: the bytes copied)."""
    import torch
    a = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    b = torch.empty_like(a)
    for _ in range(3):
        b.copy_(a)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(20):
        b.copy_(a)
    e1.record()
    torch.cuda.synchronize()
    return nbytes * 20 / (e0.elapsed_time(e1) / 1e3)


def kernel_time(dec, x) -> tuple:
    """(seconds of spectrum_kernel, launches) in one decode of x."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        dec.decode(x)
    ev = [e for e in prof.events() if "spectrum_kernel" in e.name]
    return sum(e.device_time for e in ev) / 1e6, len(ev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--buffers", type=int, default=256)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    import torch
    torch.cuda.init()
    res = dict(card=card(), buffers=a.buffers, cases=[])
    out_gib = a.buffers * api.BUFFER_BYTES / 2 ** 30
    for rate, fmt in CASES:
        x = stream(rate, fmt, a.buffers)
        floor_rate = copy_rate(x.size)
        with api.Decoder(spectrum=True, input_rate=rate, input_format=fmt) as on, \
                api.Decoder(input_rate=rate, input_format=fmt) as off:
            on.decode(x), off.decode(x)                                      # warm-up: every shape, every buffer
            on.take_spectra()
            kt, launches = kernel_time(on, x)
            assert on.take_spectra().size == a.buffers + 1 and launches >= 1
            wall = {"on": [], "off": []}
            for _ in range(a.reps):
                for name, d in (("off", off), ("on", on)):
                    t0 = time.perf_counter()
                    d.decode(x)
                    wall[name].append(time.perf_counter() - t0)
                on.take_spectra()
        case = dict(rate=rate, format=fmt, input_bytes=int(x.size), kernel_ms_per_gib_out=kt * 1e3 / out_gib,
                    floor_ms_per_gib_out=x.size / (2 * floor_rate) * 1e3 / out_gib, copy_gbps=floor_rate / 1e9,
                    decode_ms_off=min(wall["off"]) * 1e3, decode_ms_on=min(wall["on"]) * 1e3)
        case["kernel_over_floor"] = case["kernel_ms_per_gib_out"] / case["floor_ms_per_gib_out"]
        res["cases"].append(case)
    txt = json.dumps(res, indent=1)
    print(txt)
    if a.out:
        Path(a.out).write_text(txt)


if __name__ == "__main__":
    main()
