"""Device time of the 16-bit input kernels (K10 convert_kernel at 2 MHz; K9 with its int16 loader at
2.4 MS/s; modes_resample.cu), their DRAM floors, and the end-to-end streaming decode of an SC16 capture
against the UC8 stream it converts to.

    python scripts/input_format_time.py [--steps 20] [--reps 3]

- Kernels: one launch over 1 GiB of 2 MHz output (4096 reference buffers and the carry block) through
  the device harness (tests/device_shim/input_device.cu, `make dshim`), timed with CUDA events around
  each launch; median, min and max over the steps.
- Floors: the bytes each launch reads and writes (K10: 4 read + 2 written per output sample; K9: 4.8 + 2)
  over the rate of a device-to-device copy (read + write) measured in the same run.
- End to end: modes_process + modes_finish of a 2 GiB SC16 capture at 2 MHz (1 GiB of 2 MHz output) from
  pinned memory, and of the UC8 GiB it converts to, alternated; wall time per run.
The card's name and power limit are read in the same run.
"""
import argparse
import ctypes
import statistics
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

NBUF = (1 << 30) // 262144
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
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import numpy as np

    import input_format_model as M
    from dump1090_b200 import api, synth

    subprocess.run(["make", "-s", "-C", str(ROOT), "dshim"], check=True)
    lib = ctypes.CDLL(str(ROOT / "tests" / "_build" / "libinput_device.so"))
    lib.input_error.restype = ctypes.c_char_p
    lib.input_time.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_uint64, ctypes.c_int, ctypes.c_void_p,
                               ctypes.POINTER(ctypes.c_uint64)]
    lib.input_copy_time.argtypes = [ctypes.c_uint64, ctypes.c_int, ctypes.c_void_p]

    card = query("name,power.limit")
    n_out = NBUF * B
    copy_bytes = 4 * n_out
    ms = np.zeros(args.steps, np.float32)
    if lib.input_copy_time(copy_bytes, args.steps, ms.ctypes.data):
        raise RuntimeError(lib.input_error().decode())
    copy_tbs = statistics.median(2 * copy_bytes / (t * 1e-3) / 1e12 for t in ms)
    kern = {}
    for name, rate24 in (("K10 convert (2 MHz)", 0), ("K9 int16 (2.4 MS/s)", 1)):
        fb = ctypes.c_uint64()
        ms = np.zeros(args.steps, np.float32)
        if lib.input_time(rate24, 8, n_out, args.steps, ms.ctypes.data, ctypes.byref(fb)):
            raise RuntimeError(lib.input_error().decode())
        kern[name] = ([float(t) for t in ms], fb.value)

    # end to end, alternated: a 2 MHz SC16 capture vs the UC8 GiB it converts to
    seed = M.to_sc16(synth.random_traffic(1_000_000, 1000, 9), 8)      # random_traffic written as SC16
    cap = synth.tile_to(seed, 4 * n_out)
    h16 = api.PinnedBuffer(cap.size)
    h16.array[:] = cap
    y = M.convert(cap, 8)
    h8 = api.PinnedBuffer(y.size)
    h8.array[:] = y
    del cap, y
    e2e = {"SC16": [], "UC8": []}
    decs = {"SC16": api.Decoder(input_format="sc16"), "UC8": api.Decoder()}
    counts = {}
    for dd in decs.values():
        dd.set_output_array(1 << 21)
    for rep in range(args.reps + 1):
        for name, dd in decs.items():
            buf = h16 if name == "SC16" else h8
            dd.reset()
            dd.rearm_output()
            t0 = time.perf_counter()
            dd.process_ptr(buf.ptr, buf.nbytes)
            dd.finish()
            t = time.perf_counter() - t0
            counts[name] = dd.output_count()
            if rep:
                e2e[name].append(t * 1e3)
    assert counts["SC16"] == counts["UC8"], counts

    print(f"card: {card}")
    print(f"device-to-device copy of {copy_bytes / 2**30:.1f} GiB: {copy_tbs:.2f} TB/s (read + write)")
    for name, (v, fb) in kern.items():
        med = statistics.median(v)
        floor_ms = fb / (copy_tbs * 1e12) * 1e3
        print(f"{name}, {NBUF} buffers (1 GiB of 2 MHz output): {spread(v)}; {med:.4f} ms per GiB of output; "
              f"floor {fb / 1e9:.4f} GB ({fb / n_out:.2f} B per output sample) -> {floor_ms:.4f} ms; "
              f"{med / floor_ms:.2f}x the floor")
    for name, v in e2e.items():
        nbytes = h16.nbytes if name == "SC16" else h8.nbytes
        med = statistics.median(v)
        print(f"end to end {name}: {spread(v)} for {nbytes / 2**30:.3f} GiB from pinned memory "
              f"({nbytes / 1e9 / (med * 1e-3):.2f} GB/s of input, {n_out / (med * 1e-3) / 1e9:.3f} G output samples/s); "
              f"{counts[name]} messages")


if __name__ == "__main__":
    main()
