#!/usr/bin/env python
"""Writes the SASS of ONE octave of the headline kernel (cuobjdump -sass of the built library) with its opcode histogram - the evidence
for the FFMA / FMUL / FADD / LDS counts DESIGN.md quotes.   python tools/sass_excerpt.py octave.txt
At 8 octaves (the headline) the domain-warp kernel runs a fully unrolled octave loop: a straight-line body of 8 octaves, which has no
back-branch; its instructions per octave are the body's count / 8. Other octave counts run the rolled loop, reported on the line after."""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = os.path.join(ROOT, "3dworld_b200", "lib3dworld_b200.so")
sass = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout.split("\n")
keep, on = [], False
for ln in sass:
    if "Function : " in ln:
        on = "noise_grid2_kernelILb1ELb1ELi0E" in ln
    if on:
        keep.append(ln)
ins = [(int(m.group(1), 16), m.group(2)) for ln in keep for m in [re.match(r"\s+/\*([0-9a-f]{4,5})\*/\s+(.*?);", ln)] if m]


def op(t):
    return re.sub(r"^@!?U?P\d\s+", "", t).split()[0].split(".")[0]


def octaves(body):
    """octaves (for a pair of cells) in a piece of code: 8 floors (FRND) each; 0 if it is not octave code"""
    h = collections.Counter(op(t) for _, t in body)
    fp = h["FFMA"] + h["FMUL"] + h["FADD"]
    return h["FRND"] // 8 if h["FRND"] and h["FRND"] % 8 == 0 and h["LDS"] and fp > 80 * (h["FRND"] // 8) else 0


# rolled octave loops: a back-branch around exactly one octave
loops = []
for a, t in ins:
    m = re.search(r"BRA.*?(0x[0-9a-f]+)", t)
    if m and int(m.group(1), 16) < a:
        body = [(x, u) for x, u in ins if int(m.group(1), 16) <= x <= a]
        if octaves(body) == 1:
            loops.append(body)
# unrolled octave bodies: straight-line runs (no control-flow instruction, no branch target inside) of several octaves
targets = {int(m.group(1), 16) for _, t in ins for m in [re.search(r"(?:BRA|BSSY \w+,|CALL\.\S+)\s.*?(0x[0-9a-f]+)", t)] if m}
runs, cur = [], []
for a, t in ins:
    if a in targets and cur:
        runs.append(cur)
        cur = []
    if op(t) in ("BRA", "BSSY", "BSYNC", "CALL", "RET", "EXIT", "BREAK", "WARPSYNC"):
        if cur:
            runs.append(cur)
        cur = []
        continue
    cur.append((a, t))
runs.append(cur)
unrolled = [r for r in runs if octaves(r) > 1]

body, n = (unrolled[0], octaves(unrolled[0])) if unrolled else (loops[0], 1)
hist = collections.Counter(op(t) for _, t in body)
per = lambda c: ("%d" % (c // n)) if c % n == 0 else ("%.2f" % (c / n))  # noqa: E731
kind = ("the unrolled %d-octave body, 0x%04x .. 0x%04x, %d instructions / %d" % (n, body[0][0], body[-1][0], len(body), n)) if unrolled else \
       ("loop 0x%04x .. 0x%04x" % (body[0][0], body[-1][0]))
out = ["SASS excerpt (cuobjdump -sass 3dworld_b200/lib3dworld_b200.so, sm_90a) of noise_grid2_kernel<simplex, warp, shape 0>: ONE fBm octave of gen_noise2",
       "for a pair of cells at the headline's 8 octaves (%d such bodies in the kernel; the domain warp's five fBm calls run it in turn): %s = %s instructions per octave:"
       % (len(unrolled) if unrolled else len(loops), kind, per(len(body))),
       "  " + ", ".join("%s %s" % (k, per(v)) for k, v in hist.most_common()),
       "Rolled octave loop (other octave counts): %s" % ("%d instructions, %s" % (len(loops[0]), ", ".join("%s %d" % kv for kv in collections.Counter(op(t) for _, t in loops[0]).most_common()))
                                                          if loops else "none"),
       "FMA-pipe instructions per octave and warp: FMUL + FADD + FFMA = %s; FMUL / FADD are the reference's unfused multiplies / adds, FFMA only the"
       % per(hist["FMUL"] + hist["FADD"] + hist["FFMA"]),
       "exact products of csrc/tw_noise2.cuh (table addressing, mod 289, power-of-two octave weights); LDS = hash / gradient table look-ups; FRND = floor().", ""]
out += ["        /*%04x*/  %s ;" % (x, t) for x, t in body[:len(body) // n]]
if n > 1:
    out.append("        ... (%d more octaves)" % (n - 1))
open(sys.argv[1] if len(sys.argv) > 1 and not sys.argv[1].startswith("-") else "/dev/stdout", "w").write("\n".join(out) + "\n")
