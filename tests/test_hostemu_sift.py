"""The per-patch gradient-histogram kernels (csrc/siftdesc.cuh, csrc/patch_orientation.cuh) on the host emulator
(tools/hostemu): every SIFT configuration of the reference's tests and the envelope's edges, the orientation at 19 and 32
pixels with 36 and 8 bins and at the bin-count edges, odd batch sizes, grids that do not divide N, strided batches and
special texels -- compared bit for bit (NaN against NaN) with a scalar restatement that sums in the kernels' order."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tools", "hostemu")


@pytest.mark.skipif(shutil.which("g++") is None or shutil.which("make") is None or not os.path.exists("/usr/local/cuda/include/cuda.h"),
                    reason="needs g++, make and the CUDA headers")
def test_sift_and_orientation_kernels_on_the_host_emulator():
    build = subprocess.run(["make", "-C", EMU], capture_output=True, text=True, timeout=600)
    assert build.returncode == 0, build.stdout[-2000:] + build.stderr[-4000:]
    run = subprocess.run([os.path.join(EMU, "run_emu"), "--sift", "--orient"], capture_output=True, text=True, timeout=900)
    tail = run.stdout[-3000:] + run.stderr[-2000:]
    assert run.returncode == 0 and "PASSED: 0 failing comparisons" in run.stdout and "FAIL " not in run.stdout, tail
    lines = [ln for ln in run.stdout.splitlines() if ln.startswith("ok   ")]
    assert len(lines) == 24, tail
    for what in ("P=41 A=8 S=4", "P=32 A=8 S=4", "P=15 A=8 S=4", "P=19 A=5 S=3", "P=6 A=4 S=1 l2", "P=64 A=8 S=4", "A=16 S=8",
                 "P=19 A=36", "P=32 A=36", "P=19 A=8", "A=64", "A=2 ", "special texels"):
        assert any(what in ln for ln in lines), what
