"""SASS mnemonic census of every kernel in liquid_cache_b200/lib/liblc_gpu.so (cuobjdump -sass): which kernels stage by TMA
(UBLKCP + SYNCS), which stream with vector loads (LDG.E.128 / .64), where shared memory, votes, shuffles, atomics and spills
(STL / LDL) sit. Run here after a build:  python profiles/sass_census.py > sass_census.txt"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "liquid_cache_b200", "lib", "liblc_gpu.so")
COLS = ["UBLKCP", "SYNCS", "LDG.E.128", "LDG.E.64", "LDG.E", "LDG.other", "STG", "LDS", "STS", "VOTE", "SHFL", "ATOMS", "ATOMG/RED", "BAR", "LDL", "STL", "total"]


def main():
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    demangle = lambda n: subprocess.run(["c++filt", n], capture_output=True, text=True).stdout.strip()  # noqa: E731
    cur, counts = None, collections.OrderedDict()
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            counts[cur] = collections.Counter()
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
        if not m or cur is None:
            continue
        op = m.group(1)
        c = counts[cur]
        c["total"] += 1
        if op.startswith("UBLKCP"): c["UBLKCP"] += 1
        elif op.startswith("SYNCS"): c["SYNCS"] += 1
        elif op.startswith("LDG"):
            if ".128" in op: c["LDG.E.128"] += 1
            elif ".64" in op: c["LDG.E.64"] += 1
            elif re.search(r"\.(U8|S8|U16|S16)", op): c["LDG.other"] += 1
            else: c["LDG.E"] += 1
        elif op.startswith("STG"): c["STG"] += 1
        elif op.startswith("LDS"): c["LDS"] += 1
        elif op.startswith("STS"): c["STS"] += 1
        elif op.startswith("VOTE"): c["VOTE"] += 1
        elif op.startswith("SHFL"): c["SHFL"] += 1
        elif op.startswith("ATOMS"): c["ATOMS"] += 1
        elif op.startswith("ATOMG") or op.startswith("RED") or op.startswith("ATOM."): c["ATOMG/RED"] += 1
        elif op.startswith("BAR"): c["BAR"] += 1
        elif op.startswith("LDL"): c["LDL"] += 1
        elif op.startswith("STL"): c["STL"] += 1
    print(f"# {os.path.relpath(LIB, ROOT)}: static SASS instruction counts per kernel (sm_90a)")
    print("kernel".ljust(58) + " ".join(c.rjust(9) for c in COLS))
    for fn, c in counts.items():
        name = demangle(fn)
        name = name.replace("(anonymous namespace)::", "")
        name = re.sub(r"\(.*", "", name).replace("void ", "").replace("lc::", "")
        print(name[:57].ljust(58) + " ".join(str(c.get(k, 0)).rjust(9) for k in COLS))


if __name__ == "__main__":
    sys.exit(main())
