"""Many finite captures at once through the receiver pool (api.decode_captures: every capture one pool receiver,
fed one buffer per call with two batches in flight, then finished with its tail by modes_pool_finish) against
the same captures decoded one after another through one Decoder (Decoder.decode, which resets between them).

K seeded synthetic captures of uneven lengths (each --min to --max whole buffers plus a random tail) at the
chosen rate and format, dense traffic.  The two ways alternate, --reps times; every capture's messages must be
the same both ways (byte for byte).  Prints one JSON object with the wall clock of every repetition, the
medians and their ratio, the parity, and the card's name and power limit read in the same run; with --out also
writes it to that file.

    python scripts/pool_finish_time.py [--captures 256] [--min 2] [--max 20] [--reps 3] [--rate 2000000]
                                       [--format uc8] [--out FILE]
"""
import argparse
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
UNIQUE = 24                                # distinct buffers of traffic the captures are cut from


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power = (x.strip() for x in q.stdout.splitlines()[0].split(","))
    return dict(name=name, power_limit=power)


def captures(k: int, lo: int, hi: int, rate: int, fmt: str, seed: int) -> list:
    """k captures of lo..hi whole buffers plus a tail of 0 .. one buffer - 1 bytes, each cut from its own offset
    of a tiled stretch of traffic (SC16 as (x - 127) * 256, which converts back to x at SC16's default shift)."""
    n = UNIQUE * B
    if rate == 2_000_000:
        x = synth.random_traffic(n, 190 * UNIQUE, seed=seed)
    else:
        x = synth.fleet_at_rate(20, 150 * UNIQUE, seed, sample_rate=rate, period=700)[0]
    x = np.ascontiguousarray(x[: 2 * n])
    if fmt != "uc8":
        x = ((x.astype(np.int16) - 127) * 256).astype("<i2").view(np.uint8)
    full = BUF * (1 if fmt == "uc8" else 2)
    rng = np.random.default_rng(seed)
    base = synth.tile_to(x, (hi + 2) * full + x.size)
    out = []
    for _ in range(k):
        size = int(rng.integers(lo, hi + 1)) * full + int(rng.integers(0, full))
        at = int(rng.integers(0, x.size // 4)) * 4
        out.append(np.ascontiguousarray(base[at: at + size]))
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--captures", type=int, default=256)
    ap.add_argument("--min", type=int, default=2)
    ap.add_argument("--max", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--rate", type=int, default=2_000_000)
    ap.add_argument("--format", default="uc8")
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--out")
    a = ap.parse_args()
    caps = captures(a.captures, a.min, a.max, a.rate, a.format, a.seed)
    settings = dict(input_rate=a.rate, input_format=a.format)
    dec = api.Decoder(**settings)
    dec.decode(caps[0])                                       # warm-up: contexts, buffers, the pool's too
    api.decode_captures(caps[:2], **settings)
    pool_s, seq_s, parity = [], [], True
    for _ in range(a.reps):
        t0 = time.perf_counter()
        got = api.decode_captures(caps, **settings)
        pool_s.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        want = [dec.decode(c) for c in caps]
        seq_s.append(time.perf_counter() - t0)
        parity &= len(got) == len(want) and all(
            len(g) == len(w) and all(bytes(x) == bytes(y) for x, y in zip(g, w)) for g, w in zip(got, want))
    dec.close()
    total = sum(c.size for c in caps)
    res = dict(card=card(), captures=a.captures, buffers=f"{a.min}-{a.max} + tail", rate=a.rate, format=a.format,
               input_mib=round(total / 2 ** 20, 1), messages=sum(len(g) for g in got),
               pool_s=[round(t, 4) for t in pool_s], sequential_s=[round(t, 4) for t in seq_s],
               pool_median_s=round(statistics.median(pool_s), 4), sequential_median_s=round(statistics.median(seq_s), 4),
               speedup=round(statistics.median(seq_s) / statistics.median(pool_s), 2), parity=parity)
    print(json.dumps(res))
    if a.out:
        Path(a.out).write_text(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
