"""Write the SASS of the two hot loops to profiles/ (from the object files of the current build):
the scan kernel's row-pair loop and the frame-evaluation kernel's two per-bit block loops."""
import re, subprocess, sys
from collections import Counter
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
tag = sys.argv[1] if len(sys.argv) > 1 else "r2"


def sass(obj, fun=None):
    cmd = ["cuobjdump", "-sass"] + (["-fun", fun] if fun else []) + [str(ROOT / "build" / obj)]
    txt = subprocess.run(cmd, capture_output=True, text=True, check=True).stdout
    ins = []
    for l in txt.splitlines():
        m = re.match(r"\s+/\*([0-9a-f]{4})\*/\s+(.*?);", l)
        if m:
            ins.append((int(m.group(1), 16), m.group(2).strip(), re.sub(r"\s+/\* 0x[0-9a-f]+ \*/$", "", l)))
    return ins


def loops(ins):
    out = []
    for a, t, _ in ins:
        m = re.search(r"BRA(?:\.U)?\s+(?:!?U?P\d,\s*)?(0x[0-9a-f]+)", t)
        if m and int(m.group(1), 16) < a:
            out.append((int(m.group(1), 16), a, (a - int(m.group(1), 16)) // 16 + 1))
    return out


def histogram(ins, lo, hi):
    c = Counter()
    for a, t, _ in ins:
        if lo <= a <= hi:
            p = t.split()
            c[(p[1] if p[0].startswith("@") else p[0])] += 1
    return ", ".join(f"{k} {v}" for k, v in c.most_common(14))


k1 = sass("modes_scan2.o")
(ROOT / "profiles").mkdir(exist_ok=True)
lo, hi, n = next(x for x in loops(k1) if x[2] > 500)
head = (f"# scan_kernel, the row-pair loop: {n} SASS instructions in the loop body (the slow path of the first/last tile\n"
        f"# included; 64 positions per lane and trip on the fast path).  sm_90a, nvcc 12.9.\n# opcodes: {histogram(k1, lo, hi)}\n")
(ROOT / "profiles" / f"{tag}_sass_k1_row_loop.txt").write_text(head + "\n".join(l for a, _, l in k1 if lo <= a <= hi) + "\n")

# the default frame-evaluation kernel: eval_fused_kernel<4, 12>, the 28-pair block of the walk
k2 = [x for x in [None]]
txt = subprocess.run(["cuobjdump", "-sass", str(ROOT / "build" / "modes_eval_fused.o")], capture_output=True, text=True, check=True).stdout
ins, on = [], False
for l in txt.splitlines():
    if "Function :" in l:
        on = "ILi4ELi12E" in l
        continue
    m = re.match(r"\s+/\*([0-9a-f]{4})\*/\s+(.*?);", l)
    if on and m:
        ins.append((int(m.group(1), 16), m.group(2).strip(), re.sub(r"\s+/\* 0x[0-9a-f]+ \*/$", "", l)))
lo, hi, n = next(x for x in loops(ins) if 500 < x[2] < 1000)
head = (f"# eval_fused_kernel<4, 12> (the default frame evaluation), one block of the walk = 28 sample pairs, both attempts\n"
        f"# (dump1090.c:1667-1690 and :1498-1558): {n} instructions = {n / 28:.1f} per bit.  sm_90a, nvcc 12.9.\n"
        f"# opcodes: {histogram(ins, lo, hi)}\n")
(ROOT / "profiles" / f"{tag}_sass_k2_walk_block.txt").write_text(head + "\n".join(l for a, _, l in ins if lo <= a <= hi) + "\n")
print("written", tag)
