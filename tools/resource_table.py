#!/usr/bin/env python
"""tools/resource_table.py -- static facts about every kernel in the built library, read from the cubin with cuobjdump (no
GPU needed): registers, shared memory, local-memory stack and spills (`--dump-resource-usage`), plus the count of the SASS
mnemonics that prove a mechanism (UBLKCP = cp.async.bulk, SYNCS = mbarrier, ATOMG/RED = global atomics, MEMBAR.SYS = system
fence, LDG.*.SYS / STG.*.SYS = system-scope acquire/release used by the peer-memory flags).
    python tools/resource_table.py > profiles/kernel_resources.md
"""
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "openmm_b200", "libb200md.so")


def demangle(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.split("\n")
    return dict(zip(names, out))


def short(sig):
    """name<template args> without the parameter list"""
    sig = re.sub(r"^void ", "", sig)
    depth = 0
    for k, ch in enumerate(sig):
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif ch == "(" and depth == 0:
            return sig[:k]
    return sig


def main():
    res = subprocess.run(["cuobjdump", "--dump-resource-usage", LIB], capture_output=True, text=True).stdout
    rows = {}
    cur = None
    for line in res.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            cur = m.group(1)
            continue
        if cur and "REG:" in line:
            kv = dict(re.findall(r"(\w+):(\d+)", line))
            rows[cur] = kv
            cur = None
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
    counts = {}
    cur = None
    pats = {"UBLKCP": r"\bUBLKCP", "SYNCS": r"\bSYNCS", "ATOM/RED": r"\b(ATOMG?|REDG?)\b", "MEMBAR.SYS": r"MEMBAR\.\w+\.SYS", "LD.SYS": r"\bLDG?\.[\w.]*SYS", "ST.SYS": r"\bSTG?\.[\w.]*SYS",
            "SHFL": r"\bSHFL", "MUFU": r"\bMUFU", "DFMA": r"\bDFMA", "FFMA": r"\bFFMA"}
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            counts[cur] = {k: 0 for k in pats}
            continue
        if cur:
            for k, p in pats.items():
                if re.search(p, line):
                    counts[cur][k] += 1
    names = demangle(sorted(rows))
    print("# Static kernel resources of openmm_b200/libb200md.so (sm_90a cubin, cuobjdump; no GPU involved)\n")
    print("`python tools/resource_table.py`.  REG = registers per thread, SHARED = static shared memory (bytes), STACK = local-memory frame (bytes; 0 = no spills, no")
    print("local arrays), then counts of SASS instructions: UBLKCP = `cp.async.bulk` (TMA engine), SYNCS = mbarrier, ATOM/RED = global atomics, MEMBAR.SYS = system")
    print("fence, LD.SYS / ST.SYS = system-scope acquire loads / release stores of the peer-memory flags, DFMA / FFMA = double / single FMAs.\n")
    keys = list(pats)
    print("| kernel | REG | SHARED | STACK | " + " | ".join(keys) + " |")
    print("|---|---|---|---|" + "---|"*len(keys))
    for mangled in sorted(rows, key=lambda k: names[k]):
        r = rows[mangled]
        c = counts.get(mangled, {k: 0 for k in keys})
        sig = names[mangled]
        label = short(sig)
        print("| `%s` | %s | %s | %s | " % (label, r.get("REG", "?"), r.get("SHARED", "?"), r.get("STACK", "?")) + " | ".join(str(c[k]) for k in keys) + " |")
    print("""
Notes.
* `k_pair<false, M>` (forces only; M = 0 no cutoff, 2 reaction field, 4 PME) is capped at 64 registers by `__launch_bounds__(256, 4)`: four CTAs per SM hide the
  latency of the shuffle-bound inner loop (four versus three resident CTAs was measured in round 1; the close-pair path would otherwise take 80).  The price is
  the 16..32-byte frame above (`-Xptxas -v`: 132 B of spill stores / 244 B of spill loads, static, for `<false, 4>`); the energy instantiations run at 2 CTAs/SM
  and do not spill.  SHARED includes the 1 KiB the driver reserves per CTA on sm_90.
* `k_grid_push_tma`, `k_pos_push`, `k_force_push_tma` are the only kernels with UBLKCP / SYNCS: bulk copies into PEER memory through the TMA engine, completion
  on an mbarrier (DESIGN.md section 5).  There is no tcgen05 anywhere: nothing on this path is GEMM-shaped (DESIGN.md section 4).
* System-scope traffic (MEMBAR.SYS, LD.SYS, ST.SYS) appears exactly in the kernels that talk to other GPUs; with one rank those branches are not taken.
* DFMA in `k_pair<*, 4>` is the close-pair path (pairs under 0.36 nm, evaluated in double); in `k_pme_spread` / `k_pme_gather` it is the
  double B-spline weights and sums (DESIGN.md section 4 says why they are there).""")


if __name__ == "__main__":
    sys.exit(main())
