"""Wall clock of a stream decoded from GPU memory (modes_process_device) against the two ways to decode it
from the host: per GiB of 2 MHz output, (a) decode(cuda_tensor), (b) decode(cuda_tensor.cpu()) with the
device-to-host copy timed too (what a user with I/Q in GPU memory did before), and (c) decode(pinned host
array).  Cases: 2 MHz UC8 dense (modes1.bin tiled, the bench's capture) and sparse (mostly noise), 2.4 MS/s
UC8, and 10 MS/s SC16 with a 3 MHz input offset.  The stream is one period of the case's capture, fed
again and again in calls of --call-mib; the three variants alternate, --reps times, and must give the same
messages (digest of the delivered records) and statistics.  A run of its own under torch.profiler gives
the device time of the device-to-device copies (a) adds per GiB.  Prints one JSON object, and with --out
also writes it to that file.

    python scripts/device_input_time.py [--gib 1] [--reps 3] [--call-mib 64] [--out FILE]
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

PERIOD = 512 << 20                 # bytes of input held once on the device and once in pinned memory
OUT_CAP = 2_000_000                # delivered messages kept for the digest


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (x.strip() for x in q.stdout.splitlines()[0].split(","))
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def capture(case: str):
    """(rate, format, offset, one period of the stream)."""
    if case == "2mhz_dense":
        p = ROOT / "oracle" / "_ref" / "modes1.bin"
        x = np.fromfile(p, dtype=np.uint8) if p.exists() else synth.random_traffic(356868, 560, seed=1)
        return 2_000_000, "uc8", 0, synth.tile_to(x, PERIOD)
    if case == "2mhz_sparse":
        return 2_000_000, "uc8", 0, synth.tile_to(synth.random_traffic(4_000_000, 40, seed=2), PERIOD)
    if case == "2.4msps":
        x, _ = synth.fleet_at_rate(20, 300, 7, sample_rate=2_400_000)
        return 2_400_000, "uc8", 0, synth.tile_to(x, PERIOD)
    x, _ = synth.fleet_at_rate(20, 300, 7, sample_rate=10_000_000, dtype="sc16", scale=256.0, carrier_hz=3e6)
    return 10_000_000, "sc16", 3_000_000, synth.tile_to(x, PERIOD)


def stream_bytes(rate: int, fmt: str, gib: float) -> int:
    """Input bytes that make gib GiB of 2 MHz UC8 output, in whole input samples."""
    bps = 2 if fmt == "uc8" else 4
    return int(gib * (1 << 30)) // 2 * rate // 2_000_000 * bps


def run(dec, feed, total: int, call: int) -> tuple:
    """(seconds, messages, digest, stats) of one stream of `total` bytes fed by feed(offset, n)."""
    dec.reset()
    dec.rearm_output()
    t0 = time.perf_counter()
    off = 0
    while off < total:
        n = min(call, total - off, PERIOD - off % PERIOD)
        feed(off % PERIOD, n)
        off += n
    dec.finish()
    dt = time.perf_counter() - t0
    n = dec.output_count()
    k = min(n, len(dec._out))
    digest = hashlib.sha256(ctypes.string_at(ctypes.addressof(dec._out), k * ctypes.sizeof(api.Message))).hexdigest()[:16]
    return dt, n, digest, dec.stats()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=1.0, help="GiB of 2 MHz output per stream")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--call-mib", type=int, default=64)
    ap.add_argument("--cases", default="2mhz_dense,2mhz_sparse,2.4msps,10msps_sc16_offset")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    call = args.call_mib << 20
    res = dict(card=card(), gib=args.gib, call_bytes=call, reps=args.reps, cases={})
    for case in args.cases.split(","):
        rate, fmt, offset, x = capture(case)
        total = stream_bytes(rate, fmt, args.gib)
        d = torch.from_numpy(x).cuda()
        pinned = api.PinnedBuffer(PERIOD)
        pinned.array[:] = x
        dec = api.Decoder(input_rate=rate, input_format=fmt, input_offset=offset)
        dec.set_output_array(OUT_CAP)
        torch.cuda.synchronize()
        variants = {
            "a_device": lambda o, n: dec.process(d[o: o + n]),
            "b_copy_to_host": lambda o, n: dec.process(d[o: o + n].cpu().numpy()),
            "c_pinned_host": lambda o, n: dec.process_ptr(pinned.ptr + o, n),
        }
        for v in variants.values():                                    # warm every path once
            run(dec, v, min(total, 4 * call), call)
        times = {k: [] for k in variants}
        outs = {}
        for _ in range(args.reps):
            for k, v in variants.items():
                dt, n, dig, st = run(dec, v, total, call)
                times[k].append(dt / args.gib)
                outs.setdefault((n, dig, tuple(st.values())), []).append(k)
        assert len(outs) == 1, (case, outs)
        (n_msgs, dig, _), = outs
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run(dec, variants["a_device"], total, call)
            torch.cuda.synchronize()
        dtod = sum(e.self_device_time_total for e in prof.key_averages() if "DtoD" in e.key)     # microseconds
        all_dev = sum(e.self_device_time_total for e in prof.key_averages())
        res["cases"][case] = dict(
            rate=rate, format=fmt, offset=offset, input_bytes=total, messages=n_msgs, digest=dig, parity=True,
            seconds_per_gib={k: dict(median=statistics.median(t), min=min(t), max=max(t), runs=t) for k, t in times.items()},
            profiled_dtod_ms_per_gib=dtod / 1e3 / args.gib, profiled_device_ms_per_gib=all_dev / 1e3 / args.gib)
        dec.close()
        pinned.free()
        del d
        torch.cuda.empty_cache()
        print(json.dumps({case: res["cases"][case]}), file=sys.stderr, flush=True)
    out = json.dumps(res)
    print(out)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(out + "\n")


if __name__ == "__main__":
    main()
