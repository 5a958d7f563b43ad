"""The sub-pixel refinement kernel (csrc/quad_interp.cuh) on the host emulator (tools/hostemu): the conv form (radius 1
and 2) and the iterative form, with and without a mask, at n_iters 0, 1 and 5, both thresholds and allow_scale_steps,
partial edge tiles, D / H / W below 3 and special texels on a permuted (B, C, L, H, W) source -- compared bit for bit
(NaN against NaN) with a scalar restatement."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tools", "hostemu")


@pytest.mark.skipif(shutil.which("g++") is None or shutil.which("make") is None or not os.path.exists("/usr/local/cuda/include/cuda.h"),
                    reason="needs g++, make and the CUDA headers")
def test_quad_kernel_on_the_host_emulator():
    build = subprocess.run(["make", "-C", EMU], capture_output=True, text=True, timeout=600)
    assert build.returncode == 0, build.stdout[-2000:] + build.stderr[-4000:]
    run = subprocess.run([os.path.join(EMU, "run_emu"), "--quad"], capture_output=True, text=True, timeout=900)
    tail = run.stdout[-3000:] + run.stderr[-2000:]
    assert run.returncode == 0 and "PASSED: 0 failing comparisons" in run.stdout and "FAIL " not in run.stdout, tail
    lines = [ln for ln in run.stdout.splitlines() if ln.startswith("ok   ")]
    assert len(lines) == 36, tail
    for what in ("conv r=1 nms", "conv r=2 mask", "iterative nms", "iterative mask", "n_iters=0", "n_iters=1", " flat", "special texels",
                 "x2x9x9 ", "x2x9 ", "x3x3x3 "):
        assert any(what in ln for ln in lines), what
