"""The arrival key that picks a pixel's supporting surfel (csrc/sm_kernels.cuh) is a bijection on the
slots: host-side round trip over 5.7 M (slot, kind, pixel) triples per wave size, against the plain
division formulas."""
import shutil
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]


def test_tiebreak_key_roundtrip(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not Path(nvcc).exists():
        pytest.skip("needs nvcc (host compilation of the shared header)")
    exe = tmp_path / "tiebreak_check"
    build = subprocess.run([nvcc, "-std=c++17", "-O2", "-I", str(ROOT / "surfelmeshing_b200" / "csrc"), "-o", str(exe),
                            str(ROOT / "tests" / "stubs" / "tiebreak_check.cu")], capture_output=True, text=True)
    assert build.returncode == 0, build.stderr
    run = subprocess.run([str(exe)], capture_output=True, text=True)
    assert run.returncode == 0, run.stdout
    assert run.stdout.count(" 0 bad") == 8, run.stdout


def test_tiebreak_rule_reproduces_the_measured_statistics(tmp_path):
    """The default rule, sampled on the host: the win rates it produces for pairs of supporters against what was
    measured on the reference's kernels on an H100 (DESIGN.md section 4: same warp 100 %, across the warps of a block
    ~49 %, across blocks 50 - 74 % (67 % on average), different waves 100 %; a secondary association beats a primary
    one of its wave 2.9 % of the time, fewer in the first wave, whose blocks start together, than in the later ones)."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not Path(nvcc).exists():
        pytest.skip("needs nvcc (host compilation of the shared header)")
    exe = tmp_path / "tiebreak_stats"
    build = subprocess.run([nvcc, "-std=c++17", "-O2", "-I", str(ROOT / "surfelmeshing_b200" / "csrc"), "-I", str(ROOT / "include"),
                            "-o", str(exe), str(ROOT / "tests" / "stubs" / "tiebreak_stats.cu")], capture_output=True, text=True)
    assert build.returncode == 0, build.stderr
    run = subprocess.run([str(exe)], capture_output=True, text=True)
    assert run.returncode == 0, run.stderr
    stats = {k: float(v) for k, v in (line.split() for line in run.stdout.strip().splitlines())}
    print(stats)
    assert stats["other_wave"] == 1.0
    assert stats["wave0_same_warp"] == 1.0 and stats["wave2_same_warp"] == 1.0
    assert abs(stats["wave0_same_block"] - 0.5 - 0.125) < 0.02      # 25 % of the pixels in slot order, the rest a coin flip
    assert abs(stats["wave0_other_block"] - 0.625) < 0.02           # 25 % in slot order; measured 67 % on average
    assert abs(stats["wave2_other_block"] - 0.725) < 0.02           # 45 % in slot order
    assert 0.005 < stats["wave0_secondary_wins"] < 0.011            # 1.5 % early secondaries, half of them ahead
    assert 0.007 < stats["wave1_secondary_wins"] < 0.014            # 2 %
    assert 0.014 < stats["wave2_secondary_wins"] < 0.026            # 4 %; measured 2.9 % over all waves
