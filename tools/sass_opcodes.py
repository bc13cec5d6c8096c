#!/usr/bin/env python
"""Per-kernel SASS opcode census of libb200attn.so (cuobjdump -sass): the evidence that the hot ops run on
wgmma / TMA (HGMMA, UTMALDG, UTMASTG, USETMAXREG) and that the product build has no legacy mma.sync
(HMMA.16816) path.

    python tools/sass_opcodes.py > sass_opcodes.txt
"""
import collections
import re
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
LIB = ROOT / "mini-sglang_b200" / "libb200attn.so"
WATCH = ["HGMMA", "WARPGROUP", "UTMALDG", "UTMASTG", "UTMAPF", "HMMA", "LDGSTS", "SYNCS", "MUFU.EX2",
         "USETMAXREG", "ACQBULK", "LDG", "STG", "LDS", "STS", "RED", "ATOM", "BAR", "FFMA", "SHFL"]


def main():
    txt = subprocess.run(["cuobjdump", "-sass", str(LIB)], check=True, capture_output=True, text=True).stdout
    fn, per = None, collections.OrderedDict()
    for line in txt.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn = m.group(1)
            per[fn] = collections.Counter()
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Za-z0-9_.]+)", line)
        if fn and m:
            per[fn][m.group(1)] += 1
    demangled = subprocess.run(["c++filt"], input="\n".join(per), capture_output=True, text=True).stdout.splitlines()
    total = collections.Counter()
    print(f"# {LIB.name}: SASS opcode census per kernel (cuobjdump -sass), sm_90a")
    for (fn, cnt), name in zip(per.items(), demangled):
        short = re.sub(r"\(.*", "", name)
        n = sum(cnt.values())
        groups = collections.Counter()
        for op, c in cnt.items():
            for w in WATCH:
                if op == w or op.startswith(w + ".") or (w in ("UTMALDG", "UTMASTG") and op.startswith(w)):
                    key = op if w in ("UTMALDG", "UTMASTG", "HGMMA", "HMMA") else w
                    groups[key] += c
                    break
        total.update(groups)
        keys = [k for k in groups if not k.startswith(("LDG", "STG", "LDS", "STS", "BAR", "FFMA", "SHFL", "RED", "ATOM", "SYNCS"))]
        print(f"\n{short}\n  instructions: {n}")
        print("  " + ", ".join(f"{k}: {groups[k]}" for k in sorted(keys)) if keys else "  (no tensor / TMA opcodes)")
        print("  " + ", ".join(f"{k}: {groups[k]}" for k in sorted(groups) if k not in keys))
    print("\n# totals over the library")
    print(", ".join(f"{k}: {v}" for k, v in sorted(total.items())))
    print(f"# legacy mma.sync (HMMA.16816*) instructions in the product library: {sum(v for k, v in total.items() if k.startswith('HMMA'))}")


if __name__ == "__main__":
    sys.exit(main())
