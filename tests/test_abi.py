"""The C-ABI library loads and exports exactly what include/surfel_b200.h declares, and _lib mirrors the header's
structures, constants and defaults."""
import ctypes as C
import re
import subprocess
from pathlib import Path

import pytest
import torch

from surfelmeshing_b200 import _lib
from tests import cbuild

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


def values(s) -> dict:
    """A structure's fields by name, with nested structures as dicts and arrays as lists."""
    out = {}
    for name, _ in s._fields_:
        v = getattr(s, name)
        out[name] = values(v) if isinstance(v, C.Structure) else list(v) if isinstance(v, C.Array) else v
    return out


# Every ctypes structure of _lib: the C typedef it mirrors and its size.
STRUCTS = {
    _lib.IntegrateParams: ("sm_integrate_params", 44),
    _lib.PreprocessParams: ("sm_preprocess_params", 52),
    _lib.StreamDesc: ("sm_stream_desc", 56),
    _lib.TransferToken: ("sm_transfer_token", 24),
    _lib.TransferStats: ("sm_transfer_stats", 32),
    _lib.VisualizationParams: ("sm_visualization_params", 36),
    _lib.StreamStats: ("sm_stream_stats", 48),
    _lib.SessionStatus: ("sm_session_status", 16),
    _lib.RenderParams: ("sm_render_params", 32),
    _lib.TrackParams: ("sm_track_params", 44),
    _lib.TrackResult: ("sm_track_result", 20),
    _lib.TrackRGBDParams: ("sm_track_rgbd_params", 12),
    _lib.TrackRGBDResult: ("sm_track_rgbd_result", 28),
    _lib.MeshParams: ("sm_mesh_params", 12),
    _lib.MeshStats: ("sm_mesh_stats", 32),
    _lib.MeshUpdateStats: ("sm_mesh_update_stats", 80),
    _lib.RelocParams: ("sm_reloc_params", 96),
    _lib.RelocResult: ("sm_reloc_result", 40),
    _lib.HoleParams: ("sm_hole_params", 12),
    _lib.HoleStats: ("sm_hole_stats", 56),
    _lib.SimplifyParams: ("sm_simplify_params", 32),
    _lib.SimplifyStats: ("sm_simplify_stats", 72),
    _lib.TextureParams: ("sm_texture_params", 16),
    _lib.TextureStats: ("sm_texture_stats", 56),
    _lib.TextureViewDesc: ("sm_texture_view", 96),
    _lib.TextureGainParams: ("sm_texture_gain_params", 24),
    _lib.TextureGainStats: ("sm_texture_gain_stats", 40),
    _lib.ComponentParams: ("sm_component_params", 24),
    _lib.ComponentStats: ("sm_component_stats", 48),
    _lib.MeshComponent: ("sm_mesh_component", 48),
    _lib.CompactStats: ("sm_compact_stats", 40),
}
# Every integer constant of _lib: the header's name for it (None: the header states it only in prose) and its value.
CONSTANTS = {
    "SM_OK": ("SM_OK", 0),
    "SM_ERR_CUDA": ("SM_ERR_CUDA", -1),
    "SM_ERR_INVALID_ARGUMENT": ("SM_ERR_INVALID_ARGUMENT", -2),
    "SM_ERR_CAPACITY": ("SM_ERR_CAPACITY", -3),
    "INVALID_SURFEL_INDEX": ("SM_INVALID_SURFEL_INDEX", 0xFFFFFFFF),
    "ROW_COUNT": ("SM_ROW_COUNT", 25),
    "RENDER_UNMESHED_SURFELS": ("SM_RENDER_UNMESHED_SURFELS", 1),
    "DISK_INDEX_FLAG": (None, 0x80000000),
    "TRACK_CLOUD": ("SM_TRACK_CLOUD", 0),
    "TRACK_PREVIOUS_FRAME": ("SM_TRACK_PREVIOUS_FRAME", 1),
    "RELOC_MAX_CANDIDATES": ("SM_RELOC_MAX_CANDIDATES", 8),
    "MESH_MAX_UMBRELLA": ("SM_MESH_MAX_UMBRELLA", 16),
    "MESH_ALL": ("SM_MESH_ALL", 0),
    "MESH_ADDED": ("SM_MESH_ADDED", 1),
    "MESH_REMOVED": ("SM_MESH_REMOVED", 2),
    "MESH_MAX_HOLE": ("SM_MESH_MAX_HOLE", 16),
    "MESH_MAX_VALENCE": ("SM_MESH_MAX_VALENCE", 32),
    "SIMPLIFY_MAX_ROUNDS": ("SM_SIMPLIFY_MAX_ROUNDS", 1024),
    "SIMPLIFY_STOP_TARGET": ("SM_SIMPLIFY_STOP_TARGET", 1),
    "SIMPLIFY_STOP_CONVERGED": ("SM_SIMPLIFY_STOP_CONVERGED", 2),
    "SIMPLIFY_STOP_MAX_ROUNDS": ("SM_SIMPLIFY_STOP_MAX_ROUNDS", 3),
    "TEXTURE_MAX_TILE": ("SM_TEXTURE_MAX_TILE", 512),
    "TEXTURE_MAX_VIEWS": ("SM_TEXTURE_MAX_VIEWS", 1024),
    "TEXTURE_MAX_ATLAS_SIDE": ("SM_TEXTURE_MAX_ATLAS_SIDE", 32768),
}
# Defaults pinned to literal values: changing one takes an edit here as well as in the library and in defaults().
DEFAULT_VALUES = {
    _lib.IntegrateParams: dict(measurement_blending_radius=12, surfel_integration_active_window_size=2**31 - 1),
    _lib.PreprocessParams: dict(outlier_filtering_frame_count=8, depth_erosion_radius=2),
    _lib.TrackParams: dict(levels=3, iterations=[4, 5, 10, 0], model_source=_lib.TRACK_CLOUD),
    _lib.RelocParams: dict(level=3, ferns=512, candidates=1,
                           track={**values(_lib.TrackParams.defaults()), "max_point_distance": C.c_float(0.1).value}),
    _lib.MeshParams: dict(neighbor_radius_factor=2.0, max_angle_between_normals_deg=90.0, max_triangle_angle_deg=170.0),
    _lib.HoleParams: dict(max_hole_edges=8, max_angle_between_normals_deg=90.0, max_triangle_angle_deg=180.0),
    _lib.SimplifyParams: dict(target_triangles=0, max_cost=1e-6, max_angle_between_normals_deg=90.0,
                              max_triangle_angle_deg=170.0, max_rounds=64),
    _lib.ComponentParams: dict(min_triangles=10, min_area=0.0, keep_largest=0),
}


def test_table_covers_the_mirror():
    structs = {v for v in vars(_lib).values()
               if isinstance(v, type) and issubclass(v, C.Structure) and v.__module__ == _lib.__name__}
    assert sorted(s.__name__ for s in structs ^ set(STRUCTS)) == []
    constants = {name for name, v in vars(_lib).items() if type(v) is int and name.isupper()}
    assert sorted(constants ^ set(CONSTANTS)) == []


def test_mirror_matches_the_header(tmp_path):
    """sizeof and the offset of every field of each mirrored structure, and the value of every named constant, as
    the compiler sees them in include/surfel_b200.h."""
    lines = [f'  printf("%s %zu\\n", "{c}", sizeof({c}));' for c, _ in STRUCTS.values()]
    lines += [f'  printf("%s %zu\\n", "{c}.{f}", offsetof({c}, {f}));'
              for s, (c, _) in STRUCTS.items() for f, _ in s._fields_]
    lines += [f'  printf("%s %lld\\n", "{h}", (long long)({h}));' for h, _ in CONSTANTS.values() if h]
    source = tmp_path / "abi.c"
    source.write_text(f'#include <stddef.h>\n#include <stdio.h>\n#include "{ROOT / "include" / "surfel_b200.h"}"\n'
                      "int main(void) {\n" + "\n".join(lines) + "\n  return 0;\n}\n")
    out = subprocess.run([str(cbuild.build(source, ()))], capture_output=True, text=True, check=True).stdout
    compiled = {k: int(v) for k, v in (line.rsplit(" ", 1) for line in out.splitlines())}
    wrong = []
    for s, (c, size) in STRUCTS.items():
        if not C.sizeof(s) == compiled[c] == size:
            wrong.append(f"sizeof {s.__name__} {C.sizeof(s)}, {c} {compiled[c]}, pinned {size}")
        wrong += [f"{s.__name__}.{f} at {getattr(s, f).offset}, {c}.{f} at {compiled[f'{c}.{f}']}"
                  for f, _ in s._fields_ if getattr(s, f).offset != compiled[f"{c}.{f}"]]
    for name, (h, value) in CONSTANTS.items():
        header = compiled[h] if h else value
        if not getattr(_lib, name) == header == value:
            wrong.append(f"{name} {getattr(_lib, name)}, {h} {header}, pinned {value}")
    assert not wrong, "\n".join(wrong)


@pytest.mark.parametrize("params", [s for s in STRUCTS if hasattr(s, "defaults")], ids=lambda s: s.__name__)
def test_defaults_match_the_library(product, params):
    """Each defaults() is what the library's sm_default_*_params writes."""
    p = params()
    product.fn["default_" + STRUCTS[params][0][3:]](C.byref(p))
    got = values(p)
    assert got == values(params.defaults())
    for name, value in DEFAULT_VALUES.get(params, {}).items():
        assert got[name] == value, name


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


def test_library_defines_sm_cuda_once():
    """Every translation unit reports a failed CUDA call the same way, through the one SM_CUDA of sm_kernels.cuh."""
    csrc = ROOT / "surfelmeshing_b200" / "csrc"
    definitions = [f"{p.name}:{i}" for p in sorted(csrc.iterdir()) if p.is_file()
                   for i, line in enumerate(p.read_text().splitlines(), 1) if re.match(r"\s*#\s*define\s+SM_CUDA\b", line)]
    assert [d.split(":")[0] for d in definitions] == ["sm_kernels.cuh"], definitions


def test_library_selects_no_compile_time_variant():
    """The committed sources build one product: a preprocessor conditional may only tell device from host
    compilation (__CUDA_ARCH__). A variant is a patched tree or extra nvcc flags in a separate build."""
    csrc = ROOT / "surfelmeshing_b200" / "csrc"
    switches = []
    for p in sorted(csrc.iterdir()):
        if not p.is_file():
            continue
        for i, line in enumerate(p.read_text().splitlines(), 1):
            m = re.match(r"\s*#\s*(if|ifdef|ifndef|elif)\b(.*)", line)
            if not m:
                continue
            names = set(re.findall(r"[A-Za-z_]\w*", m.group(2).split("//")[0])) - {"defined"}
            if names != {"__CUDA_ARCH__"}:
                switches.append(f"{p.name}:{i}: {line.strip()}")
    assert not switches, switches


def test_every_configure_key_is_documented():
    """sm_configure accepts named knobs: each key the library tests for appears in the header's description."""
    source = (ROOT / "surfelmeshing_b200" / "csrc" / "api.cu").read_text()
    keys = sorted(set(re.findall(r'k == "([a-z_0-9]+)"', source)))
    assert len(keys) >= 9
    header = (ROOT / "include" / "surfel_b200.h").read_text()
    missing = [k for k in keys if f'"{k}"' not in header]
    assert not missing, missing
