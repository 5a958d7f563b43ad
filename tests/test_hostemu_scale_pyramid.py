"""The ScalePyramid octave kernel (csrc/octave_vwalk.cuh) on the host emulator (tools/hostemu): every instantiated chain
in both stage-0 modes, images whose smallest side equals the largest tap count, widths 28, 60 and 132, heights that are
not a multiple of the 16-row step, and grids with segments that start in the middle of a band, with finite and NaN /
+-Inf / -0 / subnormal texels -- compared bit for bit (-0 and +0 differ) with a scalar level-by-level restatement."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tools", "hostemu")


@pytest.mark.skipif(shutil.which("g++") is None or shutil.which("make") is None or not os.path.exists("/usr/local/cuda/include/cuda.h"),
                    reason="needs g++, make and the CUDA headers")
def test_octave_kernel_on_the_host_emulator():
    build = subprocess.run(["make", "-C", EMU], capture_output=True, text=True, timeout=600)
    assert build.returncode == 0, build.stdout[-2000:] + build.stderr[-4000:]
    run = subprocess.run([os.path.join(EMU, "run_emu"), "--octave"], capture_output=True, text=True, timeout=900)
    tail = run.stdout[-3000:] + run.stderr[-2000:]
    assert run.returncode == 0 and "PASSED: 0 failing comparisons" in run.stdout and "FAIL " not in run.stdout, tail
    lines = [ln for ln in run.stdout.splitlines() if ln.startswith("ok   ")]
    assert len(lines) == 22, tail  # eleven cases, finite and special texels
    for what in ("[13,11,13,17,21,25]", "[13,11,13,17,21]", "[11,11,13,17,21,25]", "[0,11,13,17,21,25]", "[0,11,13,17,21]",
                 "special texels", "x25x28 ", "x97x60 ", "x70x132 "):
        assert any(what in ln for ln in lines), what
