#!/usr/bin/env python
"""profiles/sass_evidence_r1.md from `cuobjdump -sass ezrt_b200/libezrt_b200.so`: instruction mix per kernel."""
import re
import subprocess
import sys

COLS = [("FADD2", r"\bFADD2\b"), ("FMUL2", r"\bFMUL2\b"), ("LDG.E.*.256", r"\bLDG\.[A-Z0-9.]*256"), ("LDG.NA (no L1 allocate)", r"\bLDG\.E\.NA"),
        ("LDG.E.128", r"\bLDG\.E[A-Z.]*\.128"), ("FMNMX3", r"\bFMNMX3\b"), ("FMNMX", r"\bFMNMX\b"), ("FFMA", r"\bFFMA\b"), ("DFMA/DMUL/DADD", r"\bD(FMA|MUL|ADD)\b"),
        ("VOTE", r"\bVOTEU?\b"), ("SHFL", r"\bSHFL\b"), ("LDL/STL", r"\b(LDL|STL)\b"), ("LDS/STS", r"\b(LDS|STS)\b"), ("MUFU", r"\bMUFU\b"),
        ("HMMA/UTCMMA (tensor)", r"\b(HMMA|UTC[A-Z]*MMA|IMMA|QMMA)\b")]


def main():
    so = sys.argv[1] if len(sys.argv) > 1 else "ezrt_b200/libezrt_b200.so"
    out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    kernels, cur = [], None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = [m.group(1), []]
            kernels.append(cur)
        elif cur is not None and re.match(r"\s+/\*[0-9a-f]{4}\*/", line):
            cur[1].append(line)
    demangled = subprocess.run(["c++filt"] + [k[0] for k in kernels], capture_output=True, text=True).stdout.splitlines()
    print("# SASS evidence, round 1 (`python tools/sass_evidence.py`: cuobjdump -sass %s, sm_90a) -- instruction counts per kernel\n" % so)
    print("| kernel | instructions | " + " | ".join(c for c, _ in COLS) + " |")
    print("|---|---|" + "---|" * len(COLS))
    for (name, ins), dm in zip(kernels, demangled):
        short = re.sub(r"\(.*", "", dm.replace("(anonymous namespace)::", "")).replace("void ", "")
        counts = [sum(1 for l in ins if re.search(rx, l)) for _, rx in COLS]
        print("| `%s` | %d | %s |" % (short, len(ins), " | ".join(str(c) for c in counts)))
    print("\nFADD2/FMUL2 = packed fp32x2 slab arithmetic (same bits as two scalar IEEE operations); LDG.E.ENL2.256 = 256-bit read-only loads of node "
          "and triangle records (LDG.NA: triangle records of large scenes bypass L1 allocation); FFMA appears only where `EZ_FMA` spells it "
          "(dot/cross products; the Cephes polynomials are mul+add: compiled with -fmad=false); D* = the fp64 luminance of calculateHdrCache "
          "(the reference's double literals); no tensor-core instructions by design (no dense contraction on this path).")


if __name__ == "__main__":
    main()
