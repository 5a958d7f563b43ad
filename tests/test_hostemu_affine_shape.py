"""The affine shape kernels (csrc/affine_shape.cuh) on the host emulator (tools/hostemu): P = 3 to 64, constant, stripe and
anti-correlated (negative b) patches, special texels, a non-default eps; LAFs at levels the pyramid did not build, non-finite
LAFs, both preserve_orientation values, more images than LAF sets, and grids that do not divide the keypoint count --
compared bit for bit (NaN against NaN) with a scalar restatement in the kernels' op order."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tools", "hostemu")


@pytest.mark.skipif(shutil.which("g++") is None or shutil.which("make") is None or not os.path.exists("/usr/local/cuda/include/cuda.h"),
                    reason="needs g++, make and the CUDA headers")
def test_affine_shape_kernels_on_the_host_emulator():
    build = subprocess.run(["make", "-C", EMU], capture_output=True, text=True, timeout=600)
    assert build.returncode == 0, build.stdout[-2000:] + build.stderr[-4000:]
    run = subprocess.run([os.path.join(EMU, "run_emu"), "--affine"], capture_output=True, text=True, timeout=900)
    tail = run.stdout[-3000:] + run.stderr[-2000:]
    assert run.returncode == 0 and "PASSED: 0 failing comparisons" in run.stdout and "FAIL " not in run.stdout, tail
    lines = [ln for ln in run.stdout.splitlines() if ln.startswith("ok   ")]
    assert len(lines) == 9, tail
    for what in ("patch_affine_shape_kernel", "P=64", "P=3 ", "special texels", "eps=0.000100", "laf_affine_shape_kernel", "preserve",
                 "upright", "non-finite", "extra images", "levels=1"):
        assert any(what in ln for ln in lines), what
