"""Per-kernel counts of the SASS mnemonics that show which hardware path a kernel uses (wgmma = HGMMA, mma.sync =
HMMA, TMA = UTMALDG / UBLKCP, mbarrier = SYNCS, cp.async = LDGSTS, FP64 adds = DADD ...).
Runs `cuobjdump -sass` on the in-tree libwts.so (no GPU needed).

    python tools/sass_summary.py
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "whisper-timestamped_b200", "whisper_timestamped", "libwts.so")
WATCH = ["HGMMA", "WARPGROUP", "UTMALDG", "UTMAPF", "UBLKCP", "SYNCS", "LDGSTS", "HMMA", "DADD", "DSETP", "FFMA",
         "SHFL", "LDS", "STS", "LDG", "STG", "ATOM", "RED", "BAR", "STL", "LDL"]


def main():
    out = subprocess.run(["cuobjdump", "-sass", SO], capture_output=True, text=True, check=True).stdout
    kern, counts, total = None, collections.OrderedDict(), collections.Counter()
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            kern = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip().split("(")[0]
            counts[kern] = collections.Counter()
            continue
        m = re.search(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_]*)", line)
        if m and kern:
            op = m.group(1)
            counts[kern][op] += 1
            total[kern] += 1
    print(f"# cuobjdump -sass {os.path.relpath(SO, ROOT)} (sm_90a): static instruction counts per kernel")
    print("# kernel | total | " + " ".join(WATCH))
    for k, c in counts.items():
        print(f"{k} | {total[k]} | " + " ".join(f"{w}={c[w]}" for w in WATCH if c[w]))


if __name__ == "__main__":
    main()
