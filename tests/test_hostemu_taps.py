"""The zero-skipping filter2d kernel (csrc/filter2d_taps.cuh) on the host emulator (tools/hostemu): its fixed list of cases
-- K 9 to 31, the three borders, Bk 1 / B / cycling, grids that do not divide the strips, boxes with NaN, +-Inf, -0,
subnormal texels and products that underflow -- compared bit for bit (-0 and +0 differ) with the dense K x K loop in the
generic kernel's FMA order."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tools", "hostemu")


@pytest.mark.skipif(shutil.which("g++") is None or shutil.which("make") is None or not os.path.exists("/usr/local/cuda/include/cuda.h"),
                    reason="needs g++, make and the CUDA headers")
def test_taps_kernel_on_the_host_emulator():
    build = subprocess.run(["make", "-C", EMU], capture_output=True, text=True, timeout=600)
    assert build.returncode == 0, build.stdout[-2000:] + build.stderr[-4000:]
    run = subprocess.run([os.path.join(EMU, "run_emu"), "--taps"], capture_output=True, text=True, timeout=900)
    tail = run.stdout[-3000:] + run.stderr[-2000:]
    assert run.returncode == 0 and "PASSED: 0 failing comparisons" in run.stdout and "FAIL " not in run.stdout, tail
    lines = [ln for ln in run.stdout.splitlines() if ln.startswith("ok   filter2d_taps_kernel vs the dense loop")]
    assert len(lines) == 18, tail  # nine cases, eager and lazy completion
    for k in ("K=9 ", "K=15 ", "K=21 ", "K=31 "):
        assert any(k in ln for ln in lines), k
    for b in ("border=0", "border=1", "border=2"):
        assert any(b in ln for ln in lines), b
