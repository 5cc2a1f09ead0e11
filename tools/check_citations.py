"""Checks that every `file.c:line[-line]` citation of the reference in this repo points inside an existing file of
$HANDBRAKE_SRC/libhb (a HandBrake source tree).  usage: python tools/check_citations.py"""
import os
import re
import sys
from pathlib import Path

REPO = Path(__file__).resolve().parent.parent
REF = Path(os.environ.get("HANDBRAKE_SRC", ".")) / "libhb"
PAT = re.compile(r"\b((?:handbrake/|templates/|platform/macosx/)?[A-Za-z0-9_]+\.[ch]):(\d+)(?:-(\d+))?")


def main():
    if not REF.exists():
        print("no reference tree here; nothing to check")
        return 0
    lengths = {}
    for f in REF.rglob("*.[ch]"):
        n = sum(1 for _ in f.open(errors="replace"))
        lengths.setdefault(f.name, []).append((str(f.relative_to(REF)), n))
    bad = 0
    own = {p.name for p in REPO.rglob("*.[ch]") if ".git" not in p.parts} | {p.name for p in REPO.rglob("*.cu")}
    files = [p for p in REPO.rglob("*") if p.suffix in (".md", ".c", ".h", ".cu", ".py") and ".git" not in p.parts and "gpurun_out" not in p.parts
             and p.name not in ("SURVEY.md", "PAPERS.md", "SNIPPETS.md")]
    total = 0
    for p in files:
        for m in PAT.finditer(p.read_text(errors="replace")):
            name, a, b = m.group(1), int(m.group(2)), int(m.group(3) or m.group(2))
            base = name.split("/")[-1]
            cands = [n for rel, n in lengths.get(base, []) if rel.endswith(name)]
            if not cands:
                if base in own:
                    continue                      # a citation of one of our own files
                print(f"{p.relative_to(REPO)}: {m.group(0)}: no such reference file")
                bad += 1
                continue
            total += 1
            if b < a or b > max(cands):
                print(f"{p.relative_to(REPO)}: {m.group(0)}: beyond the file's {max(cands)} lines")
                bad += 1
    print(f"{total} citations checked, {bad} bad")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
