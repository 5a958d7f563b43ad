"""The feature-response kernels (csrc/corner_vwalk.cuh for Harris / GFTT, grad_tiled_kernel's Hessian epilogue) on the host
emulator (tools/hostemu): edge bands, images whose height leaves a last tile with a box entirely below the image, 4 x 4
images, segments that start in the middle of a band, both stencil modes, sigmas, and NaN / +-Inf / -0 / subnormal texels --
compared bit for bit (-0 and +0 differ) with a scalar restatement of the composition."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tools", "hostemu")


@pytest.mark.skipif(shutil.which("g++") is None or shutil.which("make") is None or not os.path.exists("/usr/local/cuda/include/cuda.h"),
                    reason="needs g++, make and the CUDA headers")
def test_response_kernels_on_the_host_emulator():
    build = subprocess.run(["make", "-C", EMU], capture_output=True, text=True, timeout=600)
    assert build.returncode == 0, build.stdout[-2000:] + build.stderr[-4000:]
    run = subprocess.run([os.path.join(EMU, "run_emu"), "--responses"], capture_output=True, text=True, timeout=900)
    tail = run.stdout[-3000:] + run.stderr[-2000:]
    assert run.returncode == 0 and "PASSED: 0 failing comparisons" in run.stdout and "FAIL " not in run.stdout, tail
    lines = [ln for ln in run.stdout.splitlines() if ln.startswith("ok   ")]
    assert len(lines) == 24, tail  # twelve cases, eager and lazy completion
    for what in ("corner_vwalk_kernel Harris sobel", "corner_vwalk_kernel Harris diff", "corner_vwalk_kernel GFTT sobel", "corner_vwalk_kernel GFTT diff",
                 "grad_tiled_kernel<GRAD_HESS> K=3", "grad_tiled_kernel<GRAD_HESS> K=5", "special texels", "x4x4 ", "x65x68 ", "x66x132 "):
        assert any(what in ln for ln in lines), what
