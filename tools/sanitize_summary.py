#!/usr/bin/env python
"""Summarise captures/sanitize_*.log into profiles/r02_sanitizer.md (hazards / errors by source location)."""
import collections
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "captures")
lines = ["# compute-sanitizer (`bash scripts/sanitize.sh` on a GPU machine; target `tools/sanitize_target.py`)", "",
         "Every kernel family at small sizes (6000 points), each call checked against the oracle inside the target.", ""]
for tool in ("memcheck", "racecheck", "synccheck"):
    path = os.path.join(OUT, f"sanitize_{tool}.log")
    if not os.path.exists(path):
        lines += [f"## {tool}", "", "(no log)", ""]
        continue
    txt = open(path, errors="replace").read()
    finished = "all checks passed" in txt
    summ = re.findall(r"=========\s+((?:ERROR|RACECHECK|LEAK) SUMMARY:[^\n]*)", txt)
    lines += [f"## {tool}", "", f"target finished: **{finished}**; " + "; ".join(summ), ""]
    if tool == "racecheck":
        loc = collections.Counter()
        for m in re.finditer(r"Race reported between (\w+) access at (.*?) in (\S+:\d+)\s*\n((?:=========\s+and .*\n)+)", txt):
            first = f"{m.group(1)} {m.group(3)}"
            for mm in re.finditer(r"and (\w+) access at .*? in (\S+:\d+) \[(\d+) hazards\]", m.group(4)):
                loc[(first, f"{mm.group(1)} {mm.group(2)}")] += int(mm.group(3))
        if loc:
            lines += ["| first access | second access | hazards |", "|---|---|---:|"]
            for (a, b), n in loc.most_common():
                lines.append(f"| {a} | {b} | {n} |")
            lines.append("")
    if tool == "memcheck":
        errs = collections.Counter(re.findall(r"=========\s+(Invalid [^\n]*|Misaligned[^\n]*|Leaked \d+ bytes)", txt))
        for e, n in errs.most_common(10):
            lines.append(f"* {n} x {e}")
        lines.append("")
open(os.path.join(ROOT, "profiles", "r02_sanitizer.md"), "w").write("\n".join(lines) + "\n")
print("\n".join(lines))
