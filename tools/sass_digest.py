#!/usr/bin/env python
"""Instruction-mix digest of one kernel's SASS (cuobjdump -sass of the in-tree library), for profiles/.

    python tools/sass_digest.py lane_scan_kernel [lib.so] > profiles/r2_lane_scan_sass.txt

Prints, per instantiation of the kernel: total SASS instructions, the count per mnemonic class, and the presence of the
data-movement mnemonics Hopper's SASS uses (LDGSTS = cp.async, UBLKCP / UTMALDG = TMA bulk copies, SYNCS = mbarrier).
"""
import collections
import re
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
kernel = sys.argv[1] if len(sys.argv) > 1 else "lane_scan_kernel"
lib = sys.argv[2] if len(sys.argv) > 2 else str(ROOT / "ai_crypto_trader_b200" / "libb200bt.so")
txt = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
fn, counts, order = None, {}, []
for line in txt.splitlines():
    m = re.match(r"\s*Function : (\S+)", line)
    if m:
        fn = m.group(1) if kernel in m.group(1) else None
        if fn:
            counts[fn] = collections.Counter()
            order.append(fn)
        continue
    if fn:
        m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
        if m:
            counts[fn][m.group(1).split(".")[0]] += 1
print(f"# SASS digest of `{kernel}` in {Path(lib).name} (cuobjdump -sass, sm_90a)")
for fn in order:
    c = counts[fn]
    tot = sum(c.values())
    demangled = subprocess.run(["c++filt", fn], capture_output=True, text=True).stdout.strip()
    print(f"\n## {demangled}\ntotal {tot} SASS instructions")
    groups = {"shared loads (LDS)": ("LDS",), "shared stores (STS)": ("STS",), "cp.async (LDGSTS)": ("LDGSTS", "LDGDEPBAR", "DEPBAR"),
              "TMA / bulk copy (UBLKCP, UTMALDG)": ("UBLKCP", "UTMALDG", "UTMASTG"), "mbarrier (SYNCS)": ("SYNCS",),
              "global loads (LDG)": ("LDG",), "global stores (STG)": ("STG",), "atomics (ATOMG, RED)": ("ATOMG", "RED", "ATOM"),
              "fp32 min/max (FMNMX)": ("FMNMX", "FMNMX3"), "fp32 compare (FSETP, FSET)": ("FSETP", "FSET"), "fp32 mul/add (FMUL, FADD, FFMA)": ("FMUL", "FADD", "FFMA"),
              "fp64 (DADD, DMUL, DFMA, DSETP)": ("DADD", "DMUL", "DFMA", "DSETP", "MUFU"),
              "select (SEL, FSEL)": ("SEL", "FSEL"), "logic / predicates (LOP3, PLOP3)": ("LOP3", "PLOP3", "ULOP3"), "integer (IADD3, IMAD, LEA, ISETP)": ("IADD3", "IMAD", "LEA", "ISETP", "IADD", "UIADD3", "UIMAD", "ULEA", "UISETP", "SHF", "USHF"),
              "votes / shuffles (VOTE, SHFL)": ("VOTE", "VOTEU", "SHFL"), "barriers (BAR)": ("BAR",), "convergence (BSSY, BSYNC, WARPSYNC)": ("BSSY", "BSYNC", "WARPSYNC"),
              "branches (BRA, EXIT)": ("BRA", "EXIT", "CALL", "RET", "BRX")}
    seen = set()
    for name, keys in groups.items():
        n = sum(c[k] for k in keys)
        seen.update(keys)
        print(f"  {name:42s} {n:5d}")
    rest = {k: v for k, v in c.items() if k not in seen}
    print("  other: " + ", ".join(f"{k} {v}" for k, v in sorted(rest.items(), key=lambda kv: -kv[1])[:14]))
