"""Device time the carrier measurement (modes_set_carrier) adds to the 1 GiB bench workload (bench.py's default
stream, --no-fix), next to the signal pass alone (K4), the arrival pass alone (K8) and their combinations,
and the device-to-host bytes it adds.

The stream stays resident in HBM; detect_device runs with each switch set in alternation, each step timed with
CUDA events on the context's stream.  Prints the medians, what each set adds to the no-pass time, the candidate
count (each candidate's carrier record is 16 bytes copied to the host beside its 56-byte record), and the card's
name and power limit read in the same run.  --out FILE also writes the result as JSON."""
import json
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
import numpy as np
import torch

import bench
from dump1090_b200 import api

WARMUP, STEPS = 5, 25
NBUF = (1 << 30) // api.BUFFER_BYTES
SETS = [("none", False, False, False), ("signal", True, False, False), ("arrival", False, True, False),
        ("signal+arrival", True, True, False), ("carrier", False, False, True), ("signal+carrier", True, False, True),
        ("arrival+carrier", False, True, True), ("all", True, True, True)]


def card():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def main():
    out = sys.argv[sys.argv.index("--out") + 1] if "--out" in sys.argv else None
    cap, src = bench.load_capture()
    data = np.ascontiguousarray(bench.shard_bytes(cap, 0, 1 << 30))
    d = torch.from_numpy(data).cuda()
    dec = api.Decoder(fix_errors=0)
    stream = torch.cuda.ExternalStream(dec.stream)
    times = {name: [] for name, *_ in SETS}
    n_cand = 0
    for step in range(WARMUP + STEPS):
        for name, sig, arr, car in SETS:
            dec.set_signal(sig)
            dec.set_arrival(arr)
            dec.set_carrier(car)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            dec.detect_device(d.data_ptr(), NBUF)
            b.record(stream)
            n_cand = dec.detect_wait()
            b.synchronize()
            if step >= WARMUP:
                times[name].append(a.elapsed_time(b))
    med = {name: statistics.median(t) for name, t in times.items()}
    res = dict(card=card(), stream=src, candidates=int(n_cand), carrier_bytes_per_gib=16 * int(n_cand),
               record_bytes_per_gib=56 * int(n_cand), median_ms=med,
               added_ms={k: v - med["none"] for k, v in med.items()})
    print(f"card: {res['card']}")
    print(f"stream: {src}, 1 GiB, --no-fix; {n_cand} candidates: the carrier adds {16 * n_cand / 1e6:.2f} MB of "
          f"device-to-host copies per GiB beside {56 * n_cand / 1e6:.2f} MB of candidate records")
    for name, *_ in SETS:
        t = times[name]
        print(f"detect_device {name:16s}: median {med[name]:.4f} ms (min {min(t):.4f}, max {max(t):.4f}), "
              f"added {med[name] - med['none']:.4f} ms per GiB")
    k4 = med["signal"] - med["none"]
    k8_on_k4 = med["signal+arrival"] - med["signal"]
    res["carrier_on_signal_ms"] = med["signal+carrier"] - med["signal"]
    res["arrival_on_signal_ms"] = k8_on_k4
    print(f"K4 alone {k4:.4f} ms; K8 on top of K4 {k8_on_k4:.4f} ms; carrier on top of K4 {res['carrier_on_signal_ms']:.4f} ms; "
          f"carrier on top of K4+K8 {med['all'] - med['signal+arrival']:.4f} ms per GiB")
    if out:
        Path(out).parent.mkdir(parents=True, exist_ok=True)
        Path(out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
