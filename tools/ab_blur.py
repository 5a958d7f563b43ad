"""A/B of the two one-pass separable kernels on the cfg3 workload in ONE process, interleaved (same clocks, same thermal state):
sepfilter_tiled (strips left to right) vs sepfilter_vwalk (bands top to bottom), or with a second argument the named switch off / on
(any switch of kornia_b200.config that selects a blur kernel).  python tools/ab_blur.py [B] [switch]"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import kornia_b200 as K  # noqa: E402

B = int(sys.argv[1]) if len(sys.argv) > 1 else 256
SWITCH = sys.argv[2] if len(sys.argv) > 2 else "sep_vwalk"
x = torch.rand(B, 3, 1080, 1920, device="cuda")


def t(n=10):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(n):
        K.gaussian_blur2d(x, (k, k), (2.0, 2.0))
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / n


for k in (5, 7, 9, 11, 13, 17):
    res = {0: [], 1: []}
    for rep in range(4):
        for v in (0, 1):
            K.config.set(SWITCH, v)
            if SWITCH != "sep_vwalk":
                K.config.set("sep_vwalk", 0)
            t(3)
            res[v].append(t())
    K.config.reset()
    a, b = min(res[0]), min(res[1])
    gb = 24.0 * B * 1080 * 1920 / 1e6
    print(f"k={k:2d} B={B}: {SWITCH}=0 {a:.3f} ms ({gb / a / 3350 * 100:.1f} %)  {SWITCH}=1 {b:.3f} ms ({gb / b / 3350 * 100:.1f} %)  all: {['%.3f' % v for v in res[0]]} {['%.3f' % v for v in res[1]]}", flush=True)
