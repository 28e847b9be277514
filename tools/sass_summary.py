#!/usr/bin/env python
"""Per-kernel SASS mnemonic counts of libtensorlink_b200.so (cuobjdump -sass): which kernels carry wgmma
(HGMMA), TMA tensor loads (UTMALDG), bulk copies (UBLKCP, UBLKPF = L2 prefetch), mma.sync (HMMA), mbarrier waits
(SYNCS), grid-dependency control (ACQBULK / PREEXIT).

    python tools/sass_summary.py
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "tensorlink_b200", "csrc", "libtensorlink_b200.so")
KEYS = ["HGMMA", "UTMALDG", "UTMASTG", "UBLKCP", "UBLKPF", "HMMA", "SYNCS", "ACQBULK", "PREEXIT", "FFMA", "LDS", "LDG", "STG", "ATOM", "RED", "MEMBAR"]


def main():
    out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    counts, cur = collections.OrderedDict(), None
    for ln in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", ln)
        if m:
            cur = m.group(1)
            counts[cur] = collections.Counter()
            continue
        if cur is None:
            continue
        m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", ln)
        if m:
            op = m.group(1).split(".")[0]
            counts[cur][op] += 1
            counts[cur]["_total"] += 1
    demangled = subprocess.run(["c++filt"], input="\n".join(counts), capture_output=True, text=True).stdout.splitlines()
    print(f"# SASS mnemonic counts per kernel, {os.path.relpath(LIB, ROOT)} (sm_90a), `python tools/sass_summary.py`")
    print("# columns: " + " ".join(KEYS) + " | total instructions")
    rows = []
    for (mangled, c), name in zip(counts.items(), demangled):
        short = re.sub(r"\(.*", "", name)
        rows.append((short, c))
    rows.sort(key=lambda r: r[0])
    w = max(len(r[0]) for r in rows)
    print(f"{'kernel':{w}s} " + " ".join(f"{k:>7s}" for k in KEYS) + "   total")
    for short, c in rows:
        print(f"{short:{w}s} " + " ".join(f"{c.get(k, 0):7d}" for k in KEYS) + f" {c['_total']:7d}")


if __name__ == "__main__":
    sys.exit(main())
