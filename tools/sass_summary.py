#!/usr/bin/env python
"""Per-kernel SASS mnemonic counts of the built library: the committed evidence that the tensor-core kernels are
Hopper-native (HGMMA = wgmma.mma_async, UTMALDG = TMA loads, WARPGROUP = wgmma fences / waits) and which kernels run on
the legacy warp-level path (HMMA = mma.sync).  Usage: python tools/sass_summary.py > sass.txt"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "betty_b200", "csrc", "libbetty_b200.so")
WATCH = ["HGMMA", "WARPGROUP", "UTMALDG", "UTMASTG", "UTMAPF", "HMMA", "LDSM",
         "SYNCS", "FFMA", "LDG", "STG", "LDS", "STS", "ATOM", "RED", "ELECT"]


def main():
    sass = subprocess.run(["cuobjdump", "-sass", SO], stdout=subprocess.PIPE, check=True).stdout.decode()
    ver = subprocess.run(["nvcc", "--version"], stdout=subprocess.PIPE).stdout.decode().strip().splitlines()[-1]
    counts = collections.OrderedDict()
    cur = None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = subprocess.run(["c++filt", m.group(1)], stdout=subprocess.PIPE).stdout.decode().strip()
            cur = counts.setdefault(name, collections.Counter())
            continue
        if cur is None:
            continue
        m = re.search(r"/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d\s+)?([A-Z0-9_]+)", line)
        if m:
            cur["_total"] += 1
            op = m.group(1)
            for w in WATCH:
                if op.startswith(w):
                    cur[w] += 1
                    break
    print(f"# cuobjdump -sass betty_b200/csrc/libbetty_b200.so  ({ver}; -gencode arch=compute_90a,code=sm_90a)")
    print("# HGMMA = wgmma.mma_async, WARPGROUP = wgmma.fence / wait_group, UTMALDG = cp.async.bulk.tensor (TMA), "
          "HMMA = mma.sync (legacy warp-level path), LDSM = ldmatrix")
    tc = [(k, c) for k, c in counts.items() if c["HGMMA"] or c["UTMALDG"]]
    hm = [(k, c) for k, c in counts.items() if c["HMMA"] and not c["HGMMA"]]
    rest = [(k, c) for k, c in counts.items() if not (c["HGMMA"] or c["UTMALDG"] or c["HMMA"])]

    def short(k):
        k = k.replace("(anonymous namespace)::", "").replace("void ", "")
        k = re.sub(r"\((?:const |__grid_constant__ )?[A-Za-z_:].*$", "", k)
        return k if len(k) <= 110 else k[:107] + "..."

    def table(rows, cols):
        print("| kernel | instr | " + " | ".join(cols) + " |")
        print("|---|---|" + "---|" * len(cols))
        for k, c in sorted(rows, key=lambda kc: kc[0]):
            print(f"| `{short(k)}` | {c['_total']} | " + " | ".join(str(c[w]) for w in cols) + " |")

    print(f"\n## wgmma / TMA kernels ({len(tc)})\n")
    table(tc, ["HGMMA", "WARPGROUP", "UTMALDG", "UTMASTG", "SYNCS", "ELECT", "HMMA"])
    print(f"\n## warp-level tensor-core kernels, mma.sync ({len(hm)})\n")
    table(hm, ["HMMA", "LDSM", "LDG", "STG", "LDS", "STS", "FFMA"])
    print(f"\n## SIMT kernels ({len(rest)})\n")
    table(rest, ["FFMA", "LDG", "STG", "LDS", "STS", "ATOM", "RED"])
    tot = collections.Counter()
    for c in counts.values():
        tot.update(c)
    print("\n## totals\n")
    print(", ".join(f"{w} {tot[w]}" for w in WATCH if tot[w]))


if __name__ == "__main__":
    sys.exit(main())
