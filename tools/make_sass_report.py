#!/usr/bin/env python
"""probe_out/<tag>_sass.md: per-kernel SASS evidence from the built library (cuobjdump -sass): counts of the
memory / async-copy / SFU mnemonics that the design claims, and the instruction window around the TMA load."""
import re
import subprocess
import sys
from collections import Counter, OrderedDict
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
LIB = ROOT / "surfelmeshing_b200" / "libsurfel_b200.so"
KEYS = ["UTMALDG", "SYNCS", "LDG.E.128", "LDG.E.64", "LDG.E.U16", "LDG.E ", "STG.E.128", "LDS.128", "LDS.64", "LDS ", "STS.128",
        "RED.E.ADD.F32x4", "REDG.E.ADD.F32x4", "RED.E.MIN", "ATOMG", "RED.E.ADD", "MUFU.EX2", "MUFU.RCP", "MUFU.RSQ", "MUFU.SQRT",
        "SHFL", "VOTE", "BAR.SYNC", "ACQBULK", "FFMA", "FMUL", "FADD"]


def main():
    tag = sys.argv[1] if len(sys.argv) > 1 else "r02"
    sass = subprocess.run(["cuobjdump", "-sass", str(LIB)], capture_output=True, text=True, check=True).stdout
    kernels = OrderedDict()
    name = None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            raw = m.group(1)
            short = re.sub(r"_ZN3smb\d+_GLOBAL__N__[0-9a-f]+_\d+_\w+?_cu_[0-9a-f]{8}\d+", "", raw)
            short = re.sub(r"ENS_.*|ENS0_.*|EvNS.*|Eiii.*|EiiPK.*", "", short)
            name = short
            kernels.setdefault(name, [])
            continue
        if name and re.search(r"/\*[0-9a-f]{4}\*/", line):
            kernels[name].append(re.sub(r"/\* 0x[0-9a-f]+ \*/", "", line).strip())
    out = [f"# {tag}: SASS evidence (`cuobjdump -sass surfelmeshing_b200/libsurfel_b200.so`, sm_90a only)\n",
           "Instruction counts per kernel (static code, not executed counts). `UTMALDG` = `cp.async.bulk.tensor` (TMA) load, "
           "`SYNCS` = mbarrier operations, `LDG.E.128` / `STG.E.128` = 128-bit global accesses, `REDG.E.ADD.F32x4` = vector float "
           "atomics, `MUFU.*` = SFU approximations mirrored from the reference's fast-math SASS.\n",
           "| kernel | instr | " + " | ".join(k.strip() for k in KEYS) + " |", "|---|---:|" + "---:|" * len(KEYS)]
    for k, lines in kernels.items():
        if not k.startswith("k_"):
            continue
        c = Counter()
        for ln in lines:
            for key in KEYS:
                if key in ln:
                    c[key] += 1
        out.append(f"| {k} | {len(lines)} | " + " | ".join(str(c[key]) if c[key] else "" for key in KEYS) + " |")
    for k, lines in kernels.items():
        if k.startswith("k_erode_normals_radii") and any("UTMALDG" in ln for ln in lines):
            i = next(i for i, ln in enumerate(lines) if "UTMALDG" in ln)
            out += ["", f"## TMA tile fill of `{k}` (window around the load)\n", "```"] + lines[max(0, i - 14): i + 12] + ["```"]
            break
    (ROOT / "probe_out").mkdir(exist_ok=True)
    (ROOT / "probe_out" / f"{tag}_sass.md").write_text("\n".join(out) + "\n")
    print(ROOT / "probe_out" / f"{tag}_sass.md")


if __name__ == "__main__":
    main()
