"""The non-maximum-suppression kernels (csrc/nms.cuh) on the host emulator (tools/hostemu): every instantiated 2-D K in
the mask and values forms, edge tiles, tiles that lie wholly inside the halo (H or W below K, 1 x 1, 2 x 2), grids that do
not divide the tiles, and the 3-D kernel in its three modes on a permuted (B, C, L, H, W) source with 1 to 5 levels, with
quantised (heavily tied) and NaN / +-Inf / -0 / subnormal texels -- compared bit for bit with a scalar restatement."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tools", "hostemu")


@pytest.mark.skipif(shutil.which("g++") is None or shutil.which("make") is None or not os.path.exists("/usr/local/cuda/include/cuda.h"),
                    reason="needs g++, make and the CUDA headers")
def test_nms_kernels_on_the_host_emulator():
    build = subprocess.run(["make", "-C", EMU], capture_output=True, text=True, timeout=600)
    assert build.returncode == 0, build.stdout[-2000:] + build.stderr[-4000:]
    run = subprocess.run([os.path.join(EMU, "run_emu"), "--nms"], capture_output=True, text=True, timeout=900)
    tail = run.stdout[-3000:] + run.stderr[-2000:]
    assert run.returncode == 0 and "PASSED: 0 failing comparisons" in run.stdout and "FAIL " not in run.stdout, tail
    lines = [ln for ln in run.stdout.splitlines() if ln.startswith("ok   ")]
    assert len(lines) == 60, tail
    for k in range(3, 32, 2):
        for form in ("mask", "values"):
            assert any(f"nms2d_kernel K={k} {form} " in ln for ln in lines), (k, form)
    for what in ("nms3d_kernel mask", "nms3d_kernel values", "(minima)", "special texels", "x1x1 ", "x2x2 "):
        assert any(what in ln for ln in lines), what
