"""Special values through the tiled kernels on the host emulator (tools/hostemu, run_emu --specials): NaN, +-Inf, -0,
subnormal, 1e-38 and 3e38 texels and a plane of -0 through the separable and 2-D filters, pyrdown, the derivative kernels,
SSIM, remap and the fused undistort, compared bit for bit with -0 != +0; the headline forward kernel (both tile shapes, every
interpolation) also under degenerate matrices (NaN / Inf entries, beyond-int and 1e30 translations, the zero matrix, a
denominator exactly 0 on a column, ~1e-20 or negative everywhere); the tiled backward with special texels and special
upstream gradients, with the same non-finite classes as the fp64 scalar backward."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tools", "hostemu")


@pytest.mark.skipif(shutil.which("g++") is None or shutil.which("make") is None or not os.path.exists("/usr/local/cuda/include/cuda.h"),
                    reason="needs g++, make and the CUDA headers")
def test_special_values_on_the_host_emulator():
    build = subprocess.run(["make", "-C", EMU], capture_output=True, text=True, timeout=600)
    assert build.returncode == 0, build.stdout[-2000:] + build.stderr[-4000:]
    run = subprocess.run([os.path.join(EMU, "run_emu"), "--specials"], capture_output=True, text=True, timeout=900)
    tail = run.stdout[-3000:] + run.stderr[-2000:]
    assert run.returncode == 0 and "PASSED: 0 failing comparisons" in run.stdout and "FAIL " not in run.stdout, tail
    for kernel in ("sepfilter_tiled_kernel (verified", "sepfilter_tiled_kernel<LERP>", "filter2d_tiled_kernel (verified", "filter2d_tiled_kernel<5, DOWN2>",
                   "grad_tiled_kernel", "ssim_vwalk_kernel", "remap_tiled_kernel (verified", "remap_tiled_kernel<LENS>", "warp_fwd_tma (headline",
                   "warp_fwd_tma<DYN>", "warp_bwd_tma2 (per-warp pipelines", "warp_bwd_tma2<STRIDE1>"):
        for sp in ("specials=1", "specials=2"):
            assert any(kernel in ln and sp in ln for ln in run.stdout.splitlines() if ln.startswith("ok   ")), (kernel, sp)
    for tile, interp in (("tile 64x32", "interp=0"), ("tile 32x32", "interp=0"), ("tile 64x32", "interp=1"), ("tile 64x32", "interp=2")):
        assert any(tile in ln and interp in ln and "specials=2" in ln for ln in run.stdout.splitlines() if ln.startswith("ok   warp_fwd_tma (headline")), (tile, interp)
