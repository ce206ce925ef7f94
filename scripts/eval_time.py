"""Device time of the scan (K1) and frame-evaluation (K2) kernels over the 1 GiB bench workload, for one or
more builds of the library in alternation, and the floors of both kernels.

    python scripts/eval_time.py [--workload tiled_nofix|df17_aggressive] [NAME=path/to/libmodes_b200.so ...]

Without builds the tree's own library is timed.  Each build runs in a worker process of its own (a
process loads one library); the workers hold the same GiB in HBM and take turns, one step each, so
that every build sees the same card state.  Per build: scan and frame-evaluation times from the
context's CUDA events (kernel_times_ms), median, min and max over the timed steps, and whether its
candidate records are identical to the first build's.

The DRAM floor: the distinct 32-byte sectors of all candidate windows (the 121 words the kernel reads
per candidate, samples -1 .. 240 rounded out to whole words) and the 56-byte records it writes, over
the rate of a device-to-device copy (read + write) measured in the same run.  The scan's read floor: one
read-only pass over the same GiB (a sum of it as int64), timed in the same run.  The card's name, power
limit and median SM clock under the timed steps are read in the same run."""
import argparse
import hashlib
import json
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

WARMUP, STEPS = 5, 30
NBUF = (1 << 30) // 262144
HALO_SAMPLES = 240                       # kHaloSamples: positions below it have windows in the carry block


def worker(lib_path: str, workload: str) -> None:
    import numpy as np
    import torch

    import bench
    from dump1090_b200 import api
    api.LIB_PATH = Path(lib_path).resolve()
    cap, _ = bench.workload_source(workload)
    d = torch.from_numpy(np.ascontiguousarray(bench.shard_bytes(cap, 0, 1 << 30))).cuda()
    dec = api.Decoder(profile=1, **bench.WORKLOADS[workload]["cfg"])

    def reply(obj):
        sys.stdout.write(json.dumps(obj) + "\n")
        sys.stdout.flush()

    reply({"ready": True})
    for line in sys.stdin:
        cmd = line.strip()
        if cmd == "step":
            dec.detect_device(d.data_ptr(), NBUF)
            n = dec.detect_wait()
            t = dec.kernel_times_ms()
            reply({"scan": t[0], "eval": t[1], "n": n})
        elif cmd == "records":
            cands, _ = dec.detect_fetch(NBUF)
            cands = cands[np.argsort(cands["t"], kind="stable")]   # (the scan appends candidates in no fixed order)
            reply({"digest": hashlib.sha256(cands.tobytes()).hexdigest(), "n": int(cands.size)})
        elif cmd == "floor":
            cands, _ = dec.detect_fetch(NBUF)
            v = cands["t"].astype(np.int64) + 2                  # the kernel's candidate position
            body = v[v > HALO_SAMPLES]
            start = 4 * ((body - 1 - HALO_SAMPLES) >> 1)         # first byte of the 121-word window
            first, last = start // 32, (start + 483) // 32
            sectors = first[:, None] + np.arange(17)[None, :]
            sectors = np.unique(sectors[sectors <= last[:, None]])
            # device-to-device copy of the GiB: bytes read + bytes written over its time
            dst = torch.empty_like(d)
            rates = []
            for k in range(6):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                dst.copy_(d)
                b.record()
                b.synchronize()
                if k:
                    rates.append(2 * d.numel() / (a.elapsed_time(b) * 1e-3) / 1e12)
            del dst
            # read-only pass over the GiB (K1's floor: it reads every byte once and writes almost nothing)
            words = d.view(torch.int64)
            reads = []
            for k in range(11):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                words.sum()
                b.record()
                b.synchronize()
                if k:
                    reads.append(a.elapsed_time(b))
            reply({"cands": int(v.size), "in_carry": int(v.size - body.size), "window_bytes": int(sectors.size) * 32,
                   "record_bytes": int(v.size) * 56, "copy_tbs": statistics.median(rates),
                   "read_ms": reads, "read_bytes": d.numel()})
        elif cmd == "quit":
            break


class Worker:
    def __init__(self, name: str, lib_path: str, workload: str):
        self.name = name
        self.p = subprocess.Popen([sys.executable, __file__, "--worker", lib_path, "--workload", workload],
                                  stdin=subprocess.PIPE, stdout=subprocess.PIPE, text=True, cwd=str(ROOT))
        self.read()

    def ask(self, cmd: str) -> dict:
        self.p.stdin.write(cmd + "\n")
        self.p.stdin.flush()
        return self.read()

    def read(self) -> dict:
        line = self.p.stdout.readline()
        if not line:
            raise RuntimeError(f"worker {self.name} ended (exit code {self.p.wait()})")
        return json.loads(line)

    def close(self):
        try:
            self.p.stdin.write("quit\n")
            self.p.stdin.close()
        finally:
            self.p.wait()


def query(fields: str) -> str:
    q = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={fields}", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def spread(v) -> str:
    return f"median {statistics.median(v):.4f} ms (min {min(v):.4f}, max {max(v):.4f})"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="tiled_nofix", choices=["tiled_nofix", "df17_aggressive"])
    ap.add_argument("--worker")
    ap.add_argument("builds", nargs="*", help="NAME=path of a libmodes_b200.so (default: the tree's)")
    args = ap.parse_args()
    if args.worker:
        worker(args.worker, args.workload)
        return
    import bench
    builds = [b.split("=", 1) for b in args.builds] or [["tree", str(ROOT / "dump1090_b200" / "libmodes_b200.so")]]
    workers = [Worker(name, path, args.workload) for name, path in builds]
    try:
        times = {w.name: {"scan": [], "eval": []} for w in workers}
        counts = {}
        sampler = bench.ClockSampler(0)
        for step in range(WARMUP + STEPS):
            if step == WARMUP:
                sampler.start()
            for w in workers:
                r = w.ask("step")
                counts[w.name] = r["n"]
                if step >= WARMUP:
                    times[w.name]["scan"].append(r["scan"])
                    times[w.name]["eval"].append(r["eval"])
        clocks = sampler.stop()
        clock_after = query("clocks.sm")                    # (the sampler may catch nothing in so short a run)
        digests = {w.name: w.ask("records")["digest"] for w in workers}
        fl = workers[0].ask("floor")
    finally:
        for w in workers:
            w.close()
    print(f"card: {query('name,power.limit')}; SM clock under the timed steps: median {clocks['sm_mhz']} MHz "
          f"({clocks['samples']} samples, throttle reasons {clocks['reasons'] or 'none'}), "
          f"{clock_after} right after them")
    print(f"workload: {args.workload}, 1 GiB ({NBUF} buffers); {STEPS} steps after {WARMUP} warm-up steps, builds alternating")
    ref = digests[workers[0].name]
    for w in workers:
        t = times[w.name]
        print(f"  {w.name:>12}: eval {spread(t['eval'])}; scan {spread(t['scan'])}; {counts[w.name]} candidates; "
              f"records {'identical' if digests[w.name] == ref else 'DIFFER'}")
    floor_ms = fl["window_bytes"] / (fl["copy_tbs"] * 1e12) * 1e3
    rec_ms = fl["record_bytes"] / (fl["copy_tbs"] * 1e12) * 1e3
    print(f"DRAM floor of eval: {fl['cands']} candidates ({fl['in_carry']} with windows in the carry block, not counted), "
          f"distinct window sectors {fl['window_bytes'] / 1e9:.4f} GB + records {fl['record_bytes'] / 1e9:.4f} GB; "
          f"device-to-device copy {fl['copy_tbs']:.2f} TB/s (read + write) -> windows {floor_ms:.4f} ms, "
          f"with records {floor_ms + rec_ms:.4f} ms")
    read_ms = statistics.median(fl["read_ms"])
    print(f"read floor of scan: one read-only pass over the GiB (sum as int64) {spread(fl['read_ms'])}, "
          f"{fl['read_bytes'] / (read_ms * 1e-3) / 1e12:.2f} TB/s")
    for w in workers:
        print(f"  {w.name:>12}: scan median {statistics.median(times[w.name]['scan']) / read_ms:.2f}x the read floor")


if __name__ == "__main__":
    main()
