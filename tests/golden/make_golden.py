"""Generate tests/golden/*.json.gz from the UNMODIFIED reference (oracle/_ref/libref.so).

Run where `make oracle` built oracle/_ref:   python tests/golden/make_golden.py

For every (input, flags) case the reference's delivered messages are stored as
the --raw lines plus the struct modesMessage fields the reference assigns for
that DF (checker.defined_fields), and the eight statistics counters.  The one
stored input is the head of modes1.bin (checker.modes1()); synthetic
streams are regenerated from (generator, arguments, seed) by
dump1090_b200.synth, whose output is deterministic, and their sha256 is
recorded so drift is detected.
"""
import gzip
import hashlib
import json
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE.parent.parent))

import checker as C  # noqa: E402
from dump1090_b200 import synth  # noqa: E402

FLAGS = [dict(), dict(aggressive=1), dict(fix=0), dict(check_crc=0), dict(check_crc=0, aggressive=1),
         dict(drop_eof=1), dict(fix=0, drop_eof=1), dict(check_crc=0, drop_eof=1)]

INPUTS = {
    "modes1": ("modes1", {}),
    "traffic_s1": ("random_traffic", dict(nsamples=300000, nframes=400, seed=1)),
    "traffic_s2": ("random_traffic", dict(nsamples=300000, nframes=400, seed=2)),
    "traffic_lowsnr": ("random_traffic", dict(nsamples=280000, nframes=350, seed=9, sigma=4.0, amp_range=(6.0, 30.0))),
    "traffic_loud": ("random_traffic", dict(nsamples=150000, nframes=250, seed=4, amp_range=(100.0, 200.0))),
    "grid": ("df17_grid", dict(nsamples=280000, period=700, seed=5)),
    "exact_buffers": ("random_traffic", dict(nsamples=262144, nframes=300, seed=6)),
    "tiny": ("random_traffic", dict(nsamples=1000, nframes=2, seed=8)),
}


def make_input(kind, args):
    if kind == "modes1":
        return C.modes1()
    if kind == "empty":
        import numpy as np
        return np.zeros(0, dtype=np.uint8)
    return getattr(synth, kind)(**args)


def flag_id(kw):
    return "-".join(f"{k}{v}" for k, v in sorted(kw.items())) or "default"


def main():
    C.build_oracle()
    for name, (kind, args) in INPUTS.items():
        data = make_input(kind, args)
        doc = {"generator": kind, "args": args, "nbytes": int(data.size),
               "sha256": hashlib.sha256(data.tobytes()).hexdigest(), "cases": {}}
        for kw in FLAGS:
            msgs, stats = C.ref_decode(data, **kw)
            doc["cases"][flag_id(kw)] = {"flags": kw, "stats": stats,
                                         "messages": [C.msg_fields(m) for m in msgs]}
        out = HERE / f"{name}.json.gz"
        with gzip.GzipFile(out, "wb", mtime=0) as f:
            f.write(json.dumps(doc, sort_keys=True, separators=(",", ":")).encode())
        print(out.name, {k: len(v["messages"]) for k, v in doc["cases"].items()})


if __name__ == "__main__":
    main()
