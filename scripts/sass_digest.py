"""Opcode digest of the shipped library: per kernel, how many wgmma / TMA / mbarrier SASS instructions it holds
(cuobjdump -sass), plus the proof of absence of the legacy mma.sync tensor-core path (HMMA / IMMA).  Written to
profiles/<tag>_sass_digest.txt; runs on the build host (no GPU needed).

  python scripts/sass_digest.py [tag]
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "omg_b200", "lib", "libomg_b200.so")
WATCH = ("HGMMA", "WARPGROUP", "UTMALDG", "UTMASTG", "UTMAPF", "UTMACCTL", "SYNCS", "USETMAXREG", "HMMA", "IMMA",
         "MUFU.EX2", "LDGSTS", "BAR.SYNC", "ERRBAR")


def main():
    tag = sys.argv[1] if len(sys.argv) > 1 else "r02"
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    per = collections.OrderedDict()
    cur = None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip() or m.group(1)
            cur = re.sub(r"\(.*", "", cur)
            per[cur] = collections.Counter()
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,6}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
        if m and cur:
            op = m.group(1)
            per[cur]["_total"] += 1
            for w in WATCH:
                if op.startswith(w):
                    per[cur][w] += 1
    out = [f"# SASS opcode digest of {os.path.relpath(LIB, ROOT)} (cuobjdump -sass, sm_90a)", ""]
    tot = collections.Counter()
    for fn, c in per.items():
        tot.update(c)
        cols = "  ".join(f"{k}={v}" for k, v in sorted(c.items()) if k != "_total")
        out.append(f"{fn}\n    instructions={c['_total']}  {cols}")
    out += ["", "TOTAL  " + "  ".join(f"{k}={v}" for k, v in sorted(tot.items()) if k != "_total"),
            f"legacy tensor-core opcodes: HMMA={tot['HMMA']} IMMA={tot['IMMA']}"]
    path = os.path.join(ROOT, "profiles", f"{tag}_sass_digest.txt")
    open(path, "w").write("\n".join(out) + "\n")
    print("\n".join(out[-2:]))
    print("written", path)


if __name__ == "__main__":
    main()
