"""What the soft-decision recovery adds, computed on CPU: a fleet sweep (synth.fleet_at: DF17 squitters
of a fleet of 20 aircraft that each send many frames, in noise at -3..+18 dB), decoded with --aggressive
through the host resolve over the oracle's candidate records, with recovery records from the numpy
restatement (tests/recover_model.py).  The GPU computes the same records (tests/test_recover.py).

    python scripts/recover_gain.py [frames_per_point]      -> one JSON line per SNR point

Per point: the reference's true frames, the extra true frames recovered, false recoveries (recovered
frames that were never sent) and the recovery statistics."""
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

import recover_model as R
from dump1090_b200 import synth


def main():
    nframes = int(sys.argv[1]) if len(sys.argv) > 1 else 5000
    for snr in list(range(-3, 7, 3)) + [7, 8, 9, 10, 11, 12, 14, 16, 18]:
        data, truth = synth.fleet_at(float(snr), nframes, 1000 + snr)
        msgs, _, rstats, _, _ = R.cpu_decode(data, dict(aggressive=1))
        ref = {m.hex() for m in msgs if not m.recovered} & truth
        rec = [m.hex() for m in msgs if m.recovered]
        extra = set(rec) & truth - ref
        print(json.dumps({"snr_db": snr, "frames": nframes, "reference_true": len(ref), "recovered": len(rec),
                          "recovered_true_extra": len(extra), "false_recoveries": sum(h not in truth for h in rec),
                          "gain": round(len(extra) / len(ref), 4) if ref else None, "stats": rstats}), flush=True)


if __name__ == "__main__":
    main()
