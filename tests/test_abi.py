"""The C-ABI library loads and exports exactly what include/surfel_b200.h declares."""
import ctypes as C
import re
import subprocess
from pathlib import Path

import pytest
import torch

from surfelmeshing_b200 import _lib

ROOT = Path(__file__).resolve().parents[1]


def header_symbols():
    text = (ROOT / "include" / "surfel_b200.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(sm_[a-z0-9_]+)\s*\(", text)))


def test_header_declares_the_bound_symbols():
    assert header_symbols() == _lib.EXPORTED_SYMBOLS


def test_library_exports_every_declared_symbol(product):
    out = subprocess.run(["nm", "-D", "--defined-only", str(product.path)], capture_output=True, text=True, check=True)
    exported = set(re.findall(r"\bT (sm_[a-z0-9_]+)", out.stdout))
    missing = [s for s in header_symbols() if s not in exported]
    assert not missing, f"not exported: {missing}"
    # nothing of the oracle is linked into the product
    assert "smref_" not in out.stdout and "cw_" not in out.stdout


def test_library_is_sm90a_only(product):
    out = subprocess.run(["cuobjdump", "--list-elf", str(product.path)], capture_output=True, text=True)
    archs = set(re.findall(r"sm_(\d+a?)", out.stdout))
    assert archs == {"90a"}, archs


def test_default_params_match_reference_defaults(product):
    ip = _lib.IntegrateParams()
    pp = _lib.PreprocessParams()
    product.fn["default_integrate_params"](C.byref(ip))
    product.fn["default_preprocess_params"](C.byref(pp))
    d_ip, d_pp = _lib.IntegrateParams.defaults(), _lib.PreprocessParams.defaults()
    for name, _ in ip._fields_:
        assert getattr(ip, name) == getattr(d_ip, name), name
    for name, _ in pp._fields_:
        assert getattr(pp, name) == getattr(d_pp, name), name
    assert ip.surfel_integration_active_window_size == 2**31 - 1 and ip.measurement_blending_radius == 12
    assert pp.outlier_filtering_frame_count == 8 and pp.depth_erosion_radius == 2


def test_struct_layouts():
    assert C.sizeof(_lib.IntegrateParams) == 44
    assert C.sizeof(_lib.PreprocessParams) == 52
    assert C.sizeof(_lib.StreamStats) == 48


@pytest.mark.skipif(torch.cuda.is_available(), reason="only meaningful on a box without a GPU")
def test_no_cpu_fallback(product):
    """Without a CUDA device the product refuses to work instead of falling back to the CPU."""
    handle = C.c_void_p()
    status = product.fn["create"](C.byref(handle), 1000, 64, 48, 52.5, 52.5, 32.0, 24.0)
    assert status == _lib.SM_ERR_CUDA
    assert product.fn["last_error"]()


def test_missing_library_fails_loudly(tmp_path):
    with pytest.raises(ImportError):
        _lib.Library(tmp_path / "libsurfel_b200.so", "sm_", product=True)


def test_library_reads_no_environment():
    """The library has one configuration: tuning goes through sm_configure or a separate build, never through
    environment variables that only some processes see."""
    csrc = ROOT / "surfelmeshing_b200" / "csrc"
    readers = [f"{p.name}:{i}" for p in sorted(csrc.iterdir()) if p.is_file()
               for i, line in enumerate(p.read_text().splitlines(), 1) if "getenv" in line]
    assert not readers, readers


def test_every_configure_key_is_documented():
    """sm_configure accepts named knobs: each key the library tests for appears in the header's description."""
    source = (ROOT / "surfelmeshing_b200" / "csrc" / "api.cu").read_text()
    keys = sorted(set(re.findall(r'k == "([a-z_0-9]+)"', source)))
    assert len(keys) >= 9
    header = (ROOT / "include" / "surfel_b200.h").read_text()
    missing = [k for k in keys if f'"{k}"' not in header]
    assert not missing, missing
