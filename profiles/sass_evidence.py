"""Static evidence from the built library (no GPU needed): per kernel, registers / shared memory and the SASS mnemonics that
show which hardware paths it uses (wgmma, TMA tensor / bulk copies, multicast, multimem, PDL).

    python profiles/sass_evidence.py
"""
import os
import re
import subprocess
import sys
from collections import Counter, OrderedDict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "nano-vllm_b200", "lib", "libb200attn.so")
WATCH = ["HGMMA", "WARPGROUP", "UTMALDG", "UTMAPF", "UBLKCP", "SYNCS", "MULTICAST", "MULTIMEM", "LDGMC", "REDG", "ACQBULK", "PREEXIT",
         "HMMA", "LDSM", "MUFU.EX2", "CCTL", "ERRBAR", "ATOM"]


def demangle(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.splitlines()
    return dict(zip(names, out))


def main():
    res = subprocess.run(["cuobjdump", "--dump-resource-usage", LIB], capture_output=True, text=True).stdout
    usage = OrderedDict()
    cur = None
    for ln in res.splitlines():
        m = re.match(r"\s*Function (\S+):", ln)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", ln)
        if m and cur:
            usage[cur] = tuple(int(x) for x in m.groups())
            cur = None
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
    counts = {}
    cur = None
    for ln in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", ln)
        if m:
            cur = m.group(1)
            counts[cur] = Counter()
            continue
        if cur is None:
            continue
        m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\d\s+)?([A-Z0-9_.]+)", ln)
        if m:
            op = m.group(1)
            counts[cur]["_total"] += 1
            for w in WATCH:
                if op.startswith(w) or ("." + w) in op:
                    counts[cur][w] += 1
    names = demangle(list(usage))
    print(f"# {os.path.relpath(LIB, ROOT)}: {len(usage)} kernels (sm_90a).  Columns: registers/thread, static shared bytes, SASS instructions, watched mnemonics")
    rows = []
    for k, (reg, stack, sh, local) in usage.items():
        c = counts.get(k, Counter())
        short = re.sub(r"\(anonymous namespace\)::", "", names.get(k, k))
        short = re.sub(r"\(.*$", "", short)
        short = re.sub(r"^void ", "", short)
        marks = " ".join(f"{w}x{c[w]}" for w in WATCH if c[w])
        rows.append((short, reg, sh, stack, local, c["_total"], marks))
    for short, reg, sh, stack, local, tot, marks in sorted(rows):
        spill = f" STACK {stack}" if stack else ""
        print(f"{short[:78]:78s} reg {reg:3d}  smem {sh:5d}{spill}  sass {tot:5d}  {marks}")


if __name__ == "__main__":
    sys.exit(main())
