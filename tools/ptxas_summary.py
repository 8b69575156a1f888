#!/usr/bin/env python
"""Registers / spills / shared memory per kernel from the ptxas logs of the last build
(surfelmeshing_b200/build/*.ptxas.log)."""
import re
import sys
from pathlib import Path

root = Path(__file__).resolve().parents[1] / "surfelmeshing_b200" / "build"
for log in sorted(root.glob("*.ptxas.log")):
    t = log.read_text()
    for m in re.finditer(r"Compiling entry function '([^']+)' for 'sm_90a'\n.*?(\d+) bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads\n.*?Used (\d+) registers(?:, used \d+ barriers)?(?:, (\d+) bytes smem)?", t, re.S):
        name = re.sub(r"_ZN3smb\d+_GLOBAL__N__[0-9a-f]+_\d+_\w+?_cu_[0-9a-f]{8}\d+", "", m.group(1))[:44]
        print(f"{log.name.split('.')[0]:10s} {name:46s} regs {m.group(5):>3s} stack {m.group(2):>4s} spill {m.group(3)}/{m.group(4)} smem {m.group(6)}")
