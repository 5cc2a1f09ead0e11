#!/usr/bin/env python
"""tools/sass_excerpt.py [libhbcu.so] -- per-kernel SASS evidence: architecture of every cubin, and for each
kernel the instruction mnemonics that prove how it moves data and does its arithmetic (TMA: UTMALDG + mbarrier SYNCS;
packed bytes: VABSDIFF4/IDP; vector loads; FP64), with the first occurrence of each as an excerpt line."""
import collections
import re
import subprocess
import sys
from pathlib import Path

so = sys.argv[1] if len(sys.argv) > 1 else str(Path(__file__).resolve().parent.parent / "handbrake_b200" / "lib" / "libhbcu.so")
txt = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
arch = collections.Counter(re.findall(r"arch = (sm_\w+)", txt))
print(f"# {Path(so).name}: cubins by architecture: {dict(arch)}")
WATCH = ["UTMALDG", "SYNCS", "VABSDIFF4", "IDP", "LDG.E.128", "LDS.128", "LDG.E.64", "STG.E.128",
         "DADD", "DMUL", "DFMA", "SHFL", "ATOM", "RED", "MUFU", "LDGSTS"]
cur, body = None, []


def flush():
    if cur is None:
        return
    ops = collections.Counter()
    first = {}
    for line in body:
        m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(@!?U?P\w+\s+)?([A-Z0-9_.]+)(.*?);", line)
        if not m:
            continue
        op = m.group(2)
        ops[op.split(".")[0]] += 1
        for w in WATCH:
            if op.startswith(w) and w not in first:
                first[w] = (op + m.group(3)).strip()
    name = subprocess.run(["c++filt", cur], capture_output=True, text=True).stdout.strip()
    name = re.sub(r"\(anonymous namespace\)::", "", name)
    print(f"\n{name[:150]}\n    {sum(ops.values())} instructions; top: " + ", ".join(f"{k} {v}" for k, v in ops.most_common(8)))
    for w in WATCH:
        if w in first:
            print(f"    {w:<10} x{sum(v for k, v in ops.items() if k == w.split('.')[0]) if '.' not in w else ''}  e.g. {first[w][:110]}")


for line in txt.splitlines():
    m = re.match(r"\s+Function : (\S+)", line)
    if m:
        flush()
        cur, body = m.group(1), []
    elif cur is not None:
        body.append(line)
flush()
