"""Kernel time of warp_perspective per (mode, padding): tiled kernel vs generic kernel, B=64x3x1080x1920."""
import os, sys, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench
import kornia_b200 as K
from kornia_b200 import _lib
dev = "cuda"
B = 64
src = torch.rand(B, 3, 1080, 1920, device=dev)
M = bench.make_homographies(B, 1000).to(dev)
fv = torch.tensor([0.1, 0.5, 0.9], device=dev)
def t(fn, n=10):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(n): fn()
    e.record(); torch.cuda.synchronize()
    return s.elapsed_time(e) / n
rows = []
for mode in ("bilinear", "nearest", "bicubic"):
    for pad in ("zeros", "border", "reflection", "fill"):
        f = lambda: K.warp_perspective(src, M, (1080, 1920), mode=mode, padding_mode=pad, fill_value=fv)
        a = t(f); va = _lib.last_warp_variant()
        K.config.set("tma", 0)
        b = t(f, 3); vb = _lib.last_warp_variant()
        K.config.reset()
        gbs = 24.0 * B * 1080 * 1920 / a / 1e6
        rows.append(dict(mode=mode, pad=pad, tiled_ms=a, generic_ms=b, speedup=b / a, tiled_GBps=gbs, frac_of_3350=gbs / 3350, variants=[va, vb]))
        print(f"{mode:9s} {pad:11s} tiled {a:7.3f} ms ({gbs:5.0f} GB/s, {gbs/3350*100:4.1f}%)  generic {b:7.3f} ms  x{b/a:.2f}  [{va}/{vb}]", flush=True)
json.dump(rows, open("gpurun_out/modes.json", "w"), indent=1)
