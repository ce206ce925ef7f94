"""CPU sweep behind the integer decimator's filters (DESIGN §6): true and false DF17 frames the oracle decodes
from the fleet at 2 M MS/s (M = 2..5) after decimation by M, for each SNR and candidate filter, against the
native 2 MHz fleet with the same frames and arrival times.  Three cases per SNR:
  dm     density-matched noise: the fleet at snr_db - 10 log10(M), so each sample's noise grows with the
         bandwidth (the physically fair comparison);
  same   the same noise per sample as the 2 MHz fleet (the convention of the 2.4 MS/s sweep);
  tone   dm plus a continuous carrier at +2.5 MHz (at 4 MS/s it wraps to -1.5 MHz), as strong as the frames:
         an out-of-band interferer that aliases into the 2 MHz band after decimation.
Then the round trip of modes1 repeated M times per sample.

    python scripts/decimate_quality.py [--frames 300] [--seeds 2] [--m 2 3 4 5]

Needs no GPU: the oracle (`make oracle`) and the numpy model of the decimator (tests/decimate_model.py).
"""
from __future__ import annotations

import argparse
import sys
from concurrent.futures import ProcessPoolExecutor
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
for p in (str(ROOT), str(ROOT / "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402

import checker  # noqa: E402
import decimate_model as DM  # noqa: E402
from dump1090_b200 import synth  # noqa: E402

SNRS = list(range(6, 19, 2))
CUTOFFS = (0.8e6, 1.0e6, 1.2e6)
TONE_HZ = 2.5e6
AMP = 20.0                        # fleet_at's frame amplitude; the tone is as strong


def filters(m: int):
    yield "box", 0, None
    for e in range(1, m + 1):
        for fc in CUTOFFS:
            yield f"E={e} {fc / 1e6:.1f}", e, fc


def df17_counts(msgs, truth):
    got = [bytes(m.msg[:14]).hex() for m in msgs if m.msgtype == 17 and m.msgbits == 112]
    true = sum(1 for h in got if h in truth)
    return true, len(got) - true


def sweep(m: int, frames: int, seeds: int):
    """{case: {filter name: {snr: [true, false]}}} for one M, and the filters' T."""
    rate = 2_000_000 * m
    flt = list(filters(m))
    tables = {name: DM.derive_taps(m, e, fc) for name, e, fc in flt}
    res = {c: {name: {s: [0, 0] for s in SNRS} for name, _, _ in flt} for c in ("dm", "same", "tone")}
    for snr in SNRS:
        for seed in range(seeds):
            dm_snr = snr - 10 * np.log10(m)
            streams = {
                "dm": synth.fleet_at_rate(dm_snr, frames, seed, sample_rate=rate),
                "same": synth.fleet_at_rate(snr, frames, seed, sample_rate=rate),
                "tone": synth.fleet_at_rate(dm_snr, frames, seed, sample_rate=rate, tone=(TONE_HZ, AMP)),
            }
            for case, (x, truth) in streams.items():
                for name, _, _ in flt:
                    t, f = df17_counts(checker.oracle_decode(DM.decimate(x, m, tables[name]))[0], truth)
                    res[case][name][snr][0] += t
                    res[case][name][snr][1] += f
    return m, {name: tables[name].size for name, _, _ in flt}, res


def native(frames: int, seeds: int):
    out = {}
    for snr in SNRS:
        t = f = 0
        for seed in range(seeds):
            s2, truth = synth.fleet_at(snr, frames, seed)
            a, b = df17_counts(checker.oracle_decode(s2)[0], truth)
            t += a
            f += b
        out[snr] = (t, f)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--seeds", type=int, default=2)
    ap.add_argument("--m", type=int, nargs="+", default=[2, 3, 4, 5])
    args = ap.parse_args()
    checker.build_oracle()
    nat = native(args.frames, args.seeds)
    print(f"frames sent per SNR: {args.frames * args.seeds}")
    print("native 2 MHz true/false: " + ", ".join(f"{s} dB {t}/{f}" for s, (t, f) in nat.items()))
    with ProcessPoolExecutor(len(args.m)) as ex:
        runs = list(ex.map(sweep, args.m, [args.frames] * len(args.m), [args.seeds] * len(args.m)))
    m1 = checker.modes1()
    d0 = {bytes(m.msg[: m.msgbits // 8]).hex() for m in checker.oracle_decode(m1)[0]}
    for m, t_of, res in runs:
        print(f"\n## M = {m} ({2 * m} MS/s): true/false DF17 frames per SNR (dB {SNRS[0]}..{SNRS[-1]}), total true")
        totals = {}
        for case in ("dm", "same", "tone"):
            print(f"  {case}:")
            for name, per in res[case].items():
                tot = sum(v[0] for v in per.values())
                false = sum(v[1] for v in per.values())
                totals[(case, name)] = (tot, false)
                print(f"    {name:>10} T={t_of[name]:2d} | " + " ".join(f"{v[0]:4d}/{v[1]}" for v in per.values())
                      + f" | {tot} true, {false} false")
        # the rule: the shortest filter within 2 % of the best true count in dm and tone, no false frame anywhere
        best = {c: max(totals[(c, n)][0] for n in t_of) for c in ("dm", "tone")}
        ok = [n for n in t_of
              if all(totals[(c, n)][0] >= 0.98 * best[c] for c in ("dm", "tone"))
              and all(totals[(c, n)][1] == 0 for c in ("dm", "same", "tone"))]
        if ok:
            pick = min(ok, key=lambda n: (t_of[n], n != "box"))
        else:   # no filter is near the best in both cases: the one whose worse share of the two bests is highest
            clean = [n for n in t_of if all(totals[(c, n)][1] == 0 for c in ("dm", "same", "tone"))]
            pick = max(clean, key=lambda n: min(totals[(c, n)][0] / best[c] for c in ("dm", "tone")))
        print(f"  best true: dm {best['dm']}, tone {best['tone']}; within 2 % of both with no false frame: {ok}; "
              f"chosen: {pick}")
        for name in ("box", pick):
            e = (t_of[name] - m) // 2
            fc = None if name == "box" else float(name.split()[1]) * 1e6
            h = DM.derive_taps(m, e, fc)
            y = DM.decimate(DM.upsample(m1, m), m, h)
            d1 = {bytes(x.msg[: x.msgbits // 8]).hex() for x in checker.oracle_decode(y)[0]}
            print(f"  modes1 round trip with {name}: {'byte for byte' if np.array_equal(y, m1) else 'not byte for byte'}, "
                  f"{len(d1 & d0)} of the {len(d0)} frames, {len(d1 - d0)} others; taps {h.tolist()}")


if __name__ == "__main__":
    main()
