#!/usr/bin/env python
"""Summarise `nvcc -Xptxas -v` output: kernel (demangled) -> registers / spills / smem."""
import re, subprocess, sys
txt = open(sys.argv[1]).read()
pat = re.compile(r"Compiling entry function '([^']+)' for 'sm_90a'\n.*\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n.*?Used (\d+) registers(.*)")
names = [m.group(1) for m in pat.finditer(txt)]
dem = subprocess.run(["c++filt"] + names, capture_output=True, text=True).stdout.splitlines() if names else []
flt = sys.argv[2] if len(sys.argv) > 2 else ""
for m, d in zip(pat.finditer(txt), dem):
    d = d.replace("b200adj::", "").replace("void ", "")
    d = re.sub(r"\(.*\)$", "", d)
    if flt and not re.search(flt, d):
        continue
    print(f"{d:90s} regs={m.group(5):>3s} stack={m.group(2)} spill_st={m.group(3)} spill_ld={m.group(4)} {m.group(6).strip(', ')}")
