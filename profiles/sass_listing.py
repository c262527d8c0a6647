#!/usr/bin/env python3
"""profiles/sass_r02.md: per-kernel SASS statistics of the shipped library (run here, no GPU needed):
static instruction count, spill instructions (STL/LDL), async-copy / barrier mnemonics (UBLKCP = cp.async.bulk, SYNCS = mbarrier,
LDGSTS = cp.async), top opcodes."""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
so = os.path.join(ROOT, "zstd-rs_b200", "libb200zstd.so")
tag = sys.argv[1] if len(sys.argv) > 1 else "r02"
out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
funcs, cur = {}, None
for line in out.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        cur = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip().split("(")[0]
        funcs[cur] = []
        continue
    m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(.*?);", line)
    if m and cur:
        funcs[cur].append(m.group(1).strip())
lines = [f"# SASS of the shipped library (`cuobjdump -sass zstd-rs_b200/libb200zstd.so`, sm_90a), {tag}", "",
         "Per kernel: static instruction count, local-memory (spill) instructions, the asynchronous-copy / barrier mnemonics that show",
         "which hardware paths are used (`UBLKCP` = cp.async.bulk = TMA bulk copy, `SYNCS` = mbarrier, `LDGSTS` = cp.async), and the 14 most",
         "frequent opcodes.  Regenerate with `python profiles/sass_listing.py`.", ""]
for f, ins in funcs.items():
    ops, full = collections.Counter(), collections.Counter()
    for i in ins:
        t = i.split()
        op = t[1] if t[0].startswith("@") and len(t) > 1 else t[0]
        ops[op.split(".")[0]] += 1
        full[op] += 1
    grouped = collections.Counter()
    for k, v in full.items():
        if re.match(r"(UBLKCP|UTMA|SYNCS|LDGSTS|LDL|STL|ATOMS|REDS|MEMBAR|ERRBAR|BAR\.|NANOSLEEP|REDUX|VOTE|SHFL|POPC|CCTL|LDS|STS|LDG|STG)", k):
            grouped[re.match(r"[A-Z0-9]+", k).group(0)] += v
    lines.append(f"## {f}")
    lines.append(f"static instructions: {len(ins)}; spills: STL {grouped.get('STL', 0)}, LDL {grouped.get('LDL', 0)}")
    lines.append("memory / sync mnemonics: " + ", ".join(f"{k} {v}" for k, v in sorted(grouped.items())))
    det = [f"{k} x{v}" for k, v in sorted(full.items()) if re.match(r"(UBLKCP|UTMA|SYNCS|LDGSTS)", k)]
    if det:
        lines.append("async-copy detail: " + ", ".join(det))
    lines.append("top opcodes: " + ", ".join(f"{k} {v}" for k, v in ops.most_common(14)))
    lines.append("")
open(os.path.join(ROOT, "profiles", f"sass_{tag}.md"), "w").write("\n".join(lines) + "\n")
print("wrote profiles/sass_%s.md" % tag)
