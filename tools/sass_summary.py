#!/usr/bin/env python
"""Per-kernel SASS mnemonic counts of libselfrec_b200.so (cuobjdump -sass): the evidence that the tensor-core
kernels really are wgmma + TMA (HGMMA / WARPGROUP / UTMALDG / SYNCS) and that the HBM-bound ones use 128-bit accesses.

    python tools/sass_summary.py [out.txt]          (default: stdout)
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "selfrec_b200", "libselfrec_b200.so")
WATCH = ["HGMMA", "WARPGROUP", "UTMALDG", "UBLKCP", "SYNCS", "LDG.E.128", "LDG.E.64", "STG.E.128", "RED.E",
         "REDG", "ATOMG", "LDS.128", "FFMA", "FMNMX3", "FMNMX", "SHFL", "MUFU.EX2", "BAR.SYNC", "CCTL"]


def main():
    out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    kernels = collections.OrderedDict()
    cur = None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip() or m.group(1)
            name = re.sub(r"\(.*", "", name).replace("void ", "").replace("srb::", "")
            cur = kernels.setdefault(name, collections.Counter())
            continue
        if cur is None:
            continue
        m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
        if m:
            op = m.group(1)
            cur["_total"] += 1
            for w in WATCH:
                if op == w or op.startswith(w + ".") or (w.count(".") and op.startswith(w)):
                    cur[w] += 1
    lines = ["# SASS mnemonic counts per kernel: cuobjdump -sass selfrec_b200/libselfrec_b200.so (sm_90a)",
             "# columns: instructions | " + " ".join(WATCH), ""]
    for name, c in kernels.items():
        hits = " ".join(f"{w}={c[w]}" for w in WATCH if c[w])
        lines.append(f"{name:<60s} {c['_total']:6d} | {hits}")
    tc = [n for n, c in kernels.items() if c["HGMMA"]]
    lines += ["", f"kernels issuing wgmma (HGMMA): {len(tc)}: " + ", ".join(tc)]
    text = "\n".join(lines) + "\n"
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            f.write(text)
    else:
        sys.stdout.write(text)


if __name__ == "__main__":
    main()
