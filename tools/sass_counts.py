"""Per-kernel SASS instruction counts that show the Hopper paths: HGMMA (wgmma.mma_async), WARPSYNC / WARPGROUP (warpgroup
fences), UTMALDG / UTMASTG / UTMAPF (TMA load / store / prefetch), UBLKCP (cp.async.bulk 1-D), SYNCS (mbarrier), plus the classic
pipes for contrast (HMMA / FFMA / SHFL).  Usage: python tools/sass_counts.py [lib.so] > sass_counts.txt"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "voiceprintrecognition-paddlepaddle_b200", "lib", "libppv_b200.so")
OPS = ["HGMMA", "WARPGROUP", "UTMALDG", "UTMASTG", "UTMAPF", "UBLKCP", "SYNCS", "HMMA", "FFMA", "SHFL", "LDS", "STS"]


def main():
    out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    demangle = {}
    counts = collections.OrderedDict()
    cur = None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            counts[cur] = collections.Counter()
            continue
        if cur is None:
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)", line)
        if m:
            op = m.group(1)
            for o in OPS:
                if op.startswith(o):
                    counts[cur][o] += 1
            counts[cur]["_total"] += 1
    names = list(counts)
    try:
        dm = subprocess.run(["cu++filt"] + names, capture_output=True, text=True).stdout.splitlines()
        demangle = dict(zip(names, dm))
    except Exception:
        pass
    print(f"# {os.path.relpath(LIB, ROOT)}: SASS instruction counts per kernel (cuobjdump -sass, sm_90a).  Columns: " + " ".join(OPS) + " | total")
    for n in sorted(names, key=lambda k: -counts[k]["HGMMA"] * 100000 - counts[k]["_total"]):
        c = counts[n]
        short = re.sub(r"\(.*", "", demangle.get(n, n).replace("(int)", "").replace("(bool)", "")).replace("void ", "").replace("ppv::", "")
        print(f"{short:60s} " + " ".join(f"{c[o]:5d}" for o in OPS) + f" | {c['_total']:6d}")
    tot = collections.Counter()
    for c in counts.values():
        tot.update(c)
    print(f"{'TOTAL':60s} " + " ".join(f"{tot[o]:5d}" for o in OPS) + f" | {tot['_total']:6d}")


if __name__ == "__main__":
    main()
