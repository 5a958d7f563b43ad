"""The TMA-pipelined filter kernels executed on the CPU (tools/hostemu): the kernel templates of kornia_b200/csrc are
compiled by g++ against a shim and run one fiber per CUDA thread, then compared bit for bit with scalar loops.  Covers the
hardware-verified kernels (which validates the emulator) and any kernel under development before it spends GPU time."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tools", "hostemu")


@pytest.mark.skipif(shutil.which("g++") is None or shutil.which("make") is None or not os.path.exists("/usr/local/cuda/include/cuda.h"),
                    reason="needs g++, make and the CUDA headers")
def test_kernels_on_the_host_emulator():
    build = subprocess.run(["make", "-C", EMU], capture_output=True, text=True, timeout=600)
    assert build.returncode == 0, build.stdout[-2000:] + build.stderr[-4000:]
    run = subprocess.run([os.path.join(EMU, "run_emu")], capture_output=True, text=True, timeout=600)
    tail = run.stdout[-3000:] + run.stderr[-2000:]
    assert run.returncode == 0 and "PASSED: 0 failing comparisons" in run.stdout, tail
    for kernel in ("sepfilter_tiled_kernel", "sepfilter_tiled_kernel<LERP>", "filter2d_tiled_kernel<5, DOWN2>", "grad_tiled_kernel", "ssim_vwalk_kernel",
                   "remap_tiled_kernel<LENS>", "warp_bwd_tma2 (per-warp pipelines", "warp_fwd_tma (headline",
                   "warp_fwd_u8hwc", "warp_u8_tiled_kernel vs warp_fwd_u8hwc", "unit_from_byte == float(u) / 255.0f for all 256 bytes"):
        assert kernel in run.stdout, kernel
    assert "FAIL" not in run.stdout, tail


@pytest.mark.skipif(shutil.which("g++") is None or shutil.which("make") is None or not os.path.exists("/usr/local/cuda/include/cuda.h"),
                    reason="needs g++, make and the CUDA headers")
def test_filter_kernels_on_random_shapes():
    """300 random (kernel, border, shape, grid, completion mode) draws: images smaller than a tile, one-row last tiles,
    more CTAs than bands, segments that start inside a band."""
    build = subprocess.run(["make", "-C", EMU], capture_output=True, text=True, timeout=600)
    assert build.returncode == 0, build.stdout[-2000:] + build.stderr[-4000:]
    run = subprocess.run([os.path.join(EMU, "run_emu"), "--fuzz", "300"], capture_output=True, text=True, timeout=900)
    assert run.returncode == 0 and "PASSED: 0 failing comparisons" in run.stdout and "FAIL " not in run.stdout, run.stdout[-3000:] + run.stderr[-2000:]
