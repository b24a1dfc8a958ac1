#!/usr/bin/env python
"""Static SASS opcode histograms of the hot kernels of libi3d_b200.so (cuobjdump -sass), written to profiles/<tag>_sass.txt.
Usage: python profiles/sass_hist.py <tag> [kernel-substring ...]
What to look for: FP64 (DFMA/DMUL/DADD) vs FP32 mix and F2F conversions in k_eg_rows; ACQBULK / PREEXIT = griddepcontrol.wait /
launch_dependents (programmatic dependent launch) at the head of every kernel of the GN iteration; no tensor-pipe (HMMA/UTCMMA) and no
bulk-copy (UBLKCP/UTMALDG) opcodes: the path has no dense contraction, and bulk-async staging was measured slower twice (DESIGN.md §4)."""
import collections
import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "..", "intrinsic3d_b200", "libi3d_b200.so")
DEFAULT = ["k_eg_rowsILi0", "k_eg_rowsILi1", "k_eg_apply", "k_eg_accum", "k_select_obsILi5", "k_op_partial", "k_cg_updateILb0", "k_cg_dir4", "k_xchg_pull", "k_reg_build"]


def main():
    tag = sys.argv[1]
    pats = sys.argv[2:] or DEFAULT
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
    res = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True).stdout
    usage = {}
    cur = None
    for line in res.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            cur = m.group(1)
        elif cur and "REG:" in line:
            usage[cur] = line.strip()
            cur = None
    hist = collections.defaultdict(collections.Counter)
    cur = None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            continue
        if cur:
            m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)", line)
            if m:
                hist[cur][m.group(1)] += 1
    out = os.path.join(HERE, f"{tag}_sass.txt")
    with open(out, "w") as f:
        f.write("# static SASS opcode counts (cuobjdump -sass intrinsic3d_b200/libi3d_b200.so, sm_90a), top 24 per kernel\n")
        tot_special = collections.Counter()
        for fn, h in hist.items():
            for op in ("ACQBULK", "PREEXIT", "UBLKCP", "UTMALDG", "UTCMMA", "HMMA", "TLD4", "SYNCS"):
                if h.get(op):
                    tot_special[op] += h[op]
        f.write("# whole library, special opcodes: " + ", ".join(f"{k}={v}" for k, v in sorted(tot_special.items())) + "\n")
        for p in pats:
            for fn, h in hist.items():
                if p in fn:
                    f.write(f"\n## {fn}\n#  {usage.get(fn, '')}\n#  total {sum(h.values())} instructions\n")
                    for op, c in h.most_common(24):
                        f.write(f"{op:14s} {c}\n")
    print("wrote", out)


if __name__ == "__main__":
    main()
