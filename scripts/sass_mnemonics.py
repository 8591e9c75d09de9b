#!/usr/bin/env python
"""Per-kernel SASS instruction mnemonics of the built library (no GPU needed): evidence that the sm_90a code uses
TMA bulk copies, mbarriers, cluster barriers and programmatic dependent launch.
   python scripts/sass_mnemonics.py"""
import collections, os, re, subprocess, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = os.path.join(ROOT, "rootba_b200", "librootba_b200.so")
sass = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
names = subprocess.run(["c++filt"], input="\n".join(re.findall(r"Function : (\S+)", sass)), capture_output=True, text=True).stdout.split("\n")
INTEREST = re.compile(r"^(UBLKCP|SYNCS|UCGABAR|ACQBULK|SHFL|[DF]FMA|LDG|STG|LDS|STS|ATOMG|REDG|REDUX|MEMBAR|ERRBAR|CCTL|BAR|HMMA|UTC|MUFU)")
print("SASS evidence (cuobjdump -sass rootba_b200/librootba_b200.so, sm_90a) -- instruction mnemonics per kernel")
print("UBLKCP = cp.async.bulk (TMA 1-D bulk copy); SYNCS.* = mbarrier arrive.expect_tx / try_wait; UCGABAR_* = barrier.cluster;")
print("ACQBULK = griddepcontrol.wait (programmatic dependent launch); SHFL = warp shuffles; no HMMA / UTC*MMA by design (DESIGN.md section 4).")
print()
blocks = re.split(r"Function : \S+", sass)[1:]
for name, body in zip(names, blocks):
    cnt = collections.Counter()
    total = 0
    for m in re.finditer(r"/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", body):
        op = m.group(1)
        total += 1
        if INTEREST.match(op):
            key = op if op.startswith(("SYNCS", "UCGABAR", "LDG", "STG", "LDS", "STS")) else op.split(".")[0]
            if key.startswith(("LDG", "STG", "LDS", "STS")):
                parts = key.split(".")
                key = ".".join(p for p in parts if p in ("LDG", "STG", "LDS", "STS", "E", "64", "128", "U"))
            cnt[key] += 1
    short = re.sub(r"\(.*", "", name)
    print(f"{short:90s} total={total:6d}  " + " ".join(f"{k}={v}" for k, v in sorted(cnt.items())))
