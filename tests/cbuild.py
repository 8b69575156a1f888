"""Builds the tests' plain-C sources (TEST INFRASTRUCTURE) with the host C compiler on first use, into one per-user
cache directory under the system's temporary directory, so the repository tree stays untouched.

A build is keyed by the compiler's path, the flags and the bytes of the source and of every file it reaches through
`#include "…"`, so an edit to any of them builds anew instead of loading a stale binary."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import re
import shutil
import subprocess
import tempfile
from pathlib import Path

# The restatements' flags: -ffp-contract=off stops the compiler fusing a multiply and an add written apart.
WALK_FLAGS = ("-O2", "-fPIC", "-shared", "-std=gnu11", "-ffp-contract=off")

_INCLUDE = re.compile(rb'^\s*#\s*include\s*"([^"]+)"', re.M)
_loaded = {}


def ptr(a):
    """The address of a numpy array's data, as a ctypes argument."""
    return a.ctypes.data_as(C.c_void_p)


def sources(source) -> list[Path]:
    """`source` and every file it reaches through `#include "…"`, each name resolved next to the file that has it."""
    found = [Path(source).resolve()]
    for path in found:   # grows while it is walked
        for name in _INCLUDE.findall(path.read_bytes()):
            included = (path.parent / name.decode()).resolve()
            if not included.is_file():
                raise FileNotFoundError(f'{path}: #include "{name.decode()}" is not next to it')
            if included not in found:
                found.append(included)
    return found


def cache_key(source, flags, cc) -> str:
    h = hashlib.sha256()
    for part in (cc, *flags):
        h.update(part.encode() + b"\0")
    for path in sources(source):
        data = path.read_bytes()
        h.update(len(data).to_bytes(8, "little") + data)
    return h.hexdigest()[:16]


def build(source, flags) -> Path:
    """The path of `source` compiled with `flags`: an executable, or a shared library when the flags say -shared."""
    source = Path(source)
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        raise RuntimeError(f"a C compiler is needed to build {source.name}")
    out_dir = Path(tempfile.gettempdir()) / f"surfel_cbuild_{os.getuid()}"
    out_dir.mkdir(parents=True, exist_ok=True)
    path = out_dir / f"{source.stem}_{cache_key(source, flags, cc)}{'.so' if '-shared' in flags else ''}"
    if not path.exists():
        tmp = out_dir / f"{path.name}.{os.getpid()}.tmp"
        res = subprocess.run([cc, *flags, "-o", str(tmp), str(source), "-lm"], capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError(f"{source.name} does not build:\n{res.stderr}")
        os.replace(tmp, path)
    return path


def library(source, flags, signatures=None) -> C.CDLL:
    """`source` built as a shared library and loaded once per process, with `signatures` {name: (restype,
    argtypes)} set."""
    key = (Path(source).resolve(), tuple(flags))
    if key not in _loaded:
        lib = C.CDLL(str(build(source, flags)))
        for name, (restype, argtypes) in (signatures or {}).items():
            getattr(lib, name).restype = restype
            getattr(lib, name).argtypes = argtypes
        _loaded[key] = lib
    return _loaded[key]
