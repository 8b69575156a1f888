"""Build recipe for libsurfel_b200.so (hand-written sm_90a kernels + the C ABI).

`python -m surfelmeshing_b200.build` compiles every .cu under csrc/ with nvcc for
sm_90a (H100) only (no fallback architectures) and links them in-tree into
surfelmeshing_b200/libsurfel_b200.so, so that the package is importable from the
repository tree.

`python -m surfelmeshing_b200.build --out variants/lib_x.so [-- extra nvcc flags]` builds a variant
of the library for an A/B run (tools/ab_probe.py --lib x=variants/lib_x.so) from a patched source
tree or with extra nvcc flags, its objects in a directory of their own next to the output
(variants/lib_x.objs/), so the product's incremental build is left alone.

Flags: -ftz=true -fmad=false. The kernels spell out every fp32 operation (csrc/sm_math.cuh)
in the order of the reference's -use_fast_math SASS; -fmad=false guarantees the compiler
contracts nothing on its own. -ffp-contract=off does the same for the host compiler, whose default
would fuse the documented products and sums of sm_outlier_filter_transforms on hosts with FMA units.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
CSRC = PKG_DIR / "csrc"
LIB_PATH = PKG_DIR / "libsurfel_b200.so"
SOURCES = ["api.cu", "pipeline.cu", "transfer.cu", "preprocess.cu", "integrate.cu", "regularize.cu", "knn.cu",
           "render.cu", "track.cu", "mesh.cu", "reloc.cu"]
HEADERS = ["sm_math.cuh", "sm_kernels.cuh", "sm_handle.cuh", "sm_knn.cuh", "../../include/surfel_b200.h"]

NVCC_FLAGS = [
    "-std=c++17",
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo",
    "-ftz=true", "-fmad=false", "-prec-div=true", "-prec-sqrt=true",
    "-Xcompiler", "-fPIC",
    "-Xcompiler", "-ffp-contract=off",   # host code too (sm_outlier_filter_transforms documents its order)
    "-Xptxas", "-v",
]


def _nvcc() -> str:
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not Path(nvcc).exists():
        raise RuntimeError("nvcc not found: libsurfel_b200.so cannot be built (there is no CPU fallback)")
    return nvcc


def _stale(target: Path, deps) -> bool:
    if not target.exists():
        return True
    t = target.stat().st_mtime
    return any(Path(d).stat().st_mtime > t for d in deps)


def build(force: bool = False, verbose: bool = False, out: Path = LIB_PATH, extra_flags=()) -> Path:
    """Compile csrc/*.cu -> `out` (incremental) with NVCC_FLAGS + `extra_flags`. Returns the library path."""
    nvcc = _nvcc()
    out = Path(out).resolve()
    obj_dir = PKG_DIR / "build" if out == LIB_PATH else out.with_suffix(".objs")
    obj_dir.mkdir(parents=True, exist_ok=True)
    flags = [*NVCC_FLAGS, *extra_flags]
    flags_stamp = obj_dir / "nvcc_flags"
    force = force or not flags_stamp.exists() or flags_stamp.read_text() != " ".join(flags)
    headers = [CSRC / h for h in HEADERS] + [Path(__file__)]
    objects = []
    for src in SOURCES:
        obj = obj_dir / (src.replace(".cu", ".o"))
        objects.append(obj)
        if force or _stale(obj, [CSRC / src] + headers):
            cmd = [nvcc, *flags, "-c", str(CSRC / src), "-o", str(obj)]
            res = subprocess.run(cmd, capture_output=True, text=True)
            if verbose or res.returncode != 0:
                sys.stderr.write(" ".join(cmd) + "\n" + res.stdout + res.stderr)
            if res.returncode != 0:
                raise RuntimeError(f"nvcc failed on {src}")
            (obj_dir / (src + ".ptxas.log")).write_text(res.stderr)
    flags_stamp.write_text(" ".join(flags))
    if force or _stale(out, objects):
        cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-o", str(out), *map(str, objects)]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            sys.stderr.write(" ".join(cmd) + "\n" + res.stdout + res.stderr)
            raise RuntimeError("link failed")
    return out


def main(argv) -> None:
    import argparse
    split = argv.index("--") if "--" in argv else len(argv)
    ap = argparse.ArgumentParser(prog="python -m surfelmeshing_b200.build",
                                 usage="%(prog)s [--force] [--out LIB] [-- extra nvcc flags...]")
    ap.add_argument("--force", action="store_true", help="recompile every source")
    ap.add_argument("--out", type=Path, default=LIB_PATH, help="library to build (default: the product, in-tree)")
    args = ap.parse_args(argv[:split])
    print(build(force=args.force, verbose=True, out=args.out, extra_flags=argv[split + 1:]))


if __name__ == "__main__":
    main(sys.argv[1:])
