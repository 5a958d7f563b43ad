"""The LAF patch extraction kernel (csrc/laf_patches.cuh) on the host emulator (tools/hostemu): levels the pyramid did not
build, non-finite LAFs, C = 3, PS = 1 and 64, odd level sizes, a strided level 0, both functions and normalisations, and
grids that do not divide the patch count -- compared bit for bit (NaN against NaN) with a scalar restatement in the
kernel's op order."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tools", "hostemu")


@pytest.mark.skipif(shutil.which("g++") is None or shutil.which("make") is None or not os.path.exists("/usr/local/cuda/include/cuda.h"),
                    reason="needs g++, make and the CUDA headers")
def test_patch_extraction_kernel_on_the_host_emulator():
    build = subprocess.run(["make", "-C", EMU], capture_output=True, text=True, timeout=600)
    assert build.returncode == 0, build.stdout[-2000:] + build.stderr[-4000:]
    run = subprocess.run([os.path.join(EMU, "run_emu"), "--patches"], capture_output=True, text=True, timeout=900)
    tail = run.stdout[-3000:] + run.stderr[-2000:]
    assert run.returncode == 0 and "PASSED: 0 failing comparisons" in run.stdout and "FAIL " not in run.stdout, tail
    lines = [ln for ln in run.stdout.splitlines() if ln.startswith("ok   ")]
    assert len(lines) == 8, tail
    for what in ("levels=2 norm pyramid", "C=3", "non-finite", "strided", "PS=1 ", "PS=64", "97x131", "simple", "raw"):
        assert any(what in ln for ln in lines), what
