"""Kernel-level timing of filter2d (3x3, 5x5, 7x7) and gaussian blur variants at B=64x3x1080x1920: tiled vs generic."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import kornia_b200 as K
dev = "cuda"
B = 64
x = torch.rand(B, 3, 1080, 1920, device=dev)
def t(fn, n=10):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(n): fn()
    e.record(); torch.cuda.synchronize()
    return s.elapsed_time(e) / n
for k in (3, 5, 7):
    kern = torch.randn(1, k, k, device=dev)
    f = lambda: K.filter2d(x, kern)
    a = t(f)
    K.config.set("tiled_filter", 0); b = t(f, 3); K.config.reset()
    gbs = 24.0 * B * 1080 * 1920 / a / 1e6
    print(f"filter2d {k}x{k} reflect: tiled {a:.3f} ms ({gbs:.0f} GB/s, {gbs/3350*100:.1f}%)  generic {b:.3f} ms  x{b/a:.2f}", flush=True)
for k in (3, 5, 11, 17):
    f = lambda: K.gaussian_blur2d(x, (k, k), (2.0, 2.0))
    a = t(f)
    gbs = 24.0 * B * 1080 * 1920 / a / 1e6
    print(f"gaussian_blur2d {k}x{k} separable: {a:.3f} ms ({gbs:.0f} GB/s, {gbs/3350*100:.1f}%)", flush=True)
# remap with a smooth (undistortion-like) map
ys, xs = torch.meshgrid(torch.arange(1080, dtype=torch.float32, device=dev), torch.arange(1920, dtype=torch.float32, device=dev), indexing="ij")
r2 = ((xs - 960) / 960) ** 2 + ((ys - 540) / 540) ** 2
mx = (960 + (xs - 960) * (1 + 0.02 * r2))[None].contiguous()
my = (540 + (ys - 540) * (1 + 0.02 * r2))[None].contiguous()
f = lambda: K.remap(x, mx, my, align_corners=True)
a = t(f)
K.config.set("tma", 0); b = t(f, 3); K.config.reset()
gbs = 24.0 * B * 1080 * 1920 / a / 1e6   # shared map: 8 B/pixel of map traffic is read once and stays in L2
print(f"remap (shared radial map): tiled {a:.3f} ms ({gbs:.0f} GB/s of image traffic, {gbs/3350*100:.1f}%)  generic {b:.3f} ms  x{b/a:.2f}", flush=True)
mxb, myb = mx.expand(B, -1, -1).contiguous(), my.expand(B, -1, -1).contiguous()
f = lambda: K.remap(x, mxb, myb, align_corners=True)
a = t(f)
gbs = 32.0 * B * 1080 * 1920 / a / 1e6
print(f"remap (per-sample maps): tiled {a:.3f} ms ({gbs:.0f} GB/s, {gbs/3350*100:.1f}%)", flush=True)
