"""Opcode census of the shipped library: per kernel, how many tensor-core / TMA instructions its SASS holds.
    python tools/sass_census.py [tensorrt_laboratory_b200/libb200infer.so] > sass_census.txt
HGMMA = wgmma f16, IGMMA = wgmma s8, WARPSYNC/WARPGROUP = warpgroup fences, UTMALDG / UTMASTG = TMA tensor load / store,
UBLKCP = cp.async.bulk, HMMA = the legacy mma.sync path (must be absent)."""
import collections
import os
import re
import subprocess
import sys

OPS = ["HGMMA", "IGMMA", "WARPGROUP", "UTMALDG", "UTMASTG", "UBLKCP", "SYNCS", "HMMA", "IMMA", "ATOMG", "REDG", "MEMBAR"]


def main():
    lib = sys.argv[1] if len(sys.argv) > 1 else os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                                              "tensorrt_laboratory_b200", "libb200infer.so")
    sass = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    demangle = {}
    counts = collections.OrderedDict()
    cur = None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            counts[cur] = collections.Counter()
            continue
        if cur is None:
            continue
        m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
        if m:
            op = m.group(1).split(".")[0]
            counts[cur][op] += 1
            counts[cur]["_total"] += 1
    names = list(counts)
    try:
        out = subprocess.run(["c++filt"] + names, capture_output=True, text=True, check=True).stdout.splitlines()
        demangle = dict(zip(names, out))
    except Exception:
        demangle = {n: n for n in names}
    totals = collections.Counter()
    print(f"# SASS opcode census of {os.path.basename(lib)} ({len(names)} kernels); columns: " + " ".join(OPS) + " | instructions")
    for n in names:
        c = counts[n]
        if not any(c[o] for o in OPS[:9]) and "tcgen05" not in demangle[n]:
            for o in OPS:
                totals[o] += c[o]
            continue
        short = re.sub(r"\(.*", "", demangle[n])
        print(f"{short:90s} " + " ".join(f"{c[o]:5d}" for o in OPS) + f" | {c['_total']}")
        for o in OPS:
            totals[o] += c[o]
    print("# whole library: " + ", ".join(f"{o}={totals[o]}" for o in OPS))


if __name__ == "__main__":
    main()
