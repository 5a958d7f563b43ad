"""Timing of the filter / affine family (SURVEY.md 8f rows 2-3) at B x 3 x 1080 x 1920 fp32 on one GPU: this
library vs the reference's torch composition (the oracle module, i.e. the same ATen calls the reference makes)
on the same device.  CUDA events, 3 warm-ups, inputs (>= 1.6 GB) larger than L2.  Prints one line per op with the
algorithmic bytes moved per second and the fraction of the HBM roofline (3.35 TB/s, H100 SXM data sheet)."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import kornia_b200 as K  # noqa: E402
from oracle import kornia_restated as R  # noqa: E402

dev = "cuda"
B = int(os.environ.get("FAMILY_B", "64"))
H, W = 1080, 1920
peak = 3350.0
x = torch.rand(B, 3, H, W, device=dev)
elems = B * 3 * H * W


def t(fn, n=10):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(n):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / n


rows = []


def line(name, ours, theirs, bytes_per_elem):
    a = t(ours)
    b = t(theirs, 3)
    gbs = bytes_per_elem * elems / a / 1e6
    rows.append(dict(op=name, ms=round(a, 3), torch_ms=round(b, 3), speedup=round(b / a, 2), gbs=round(gbs), frac=round(gbs / peak, 3),
                     algorithmic_bytes_per_element=bytes_per_elem))
    print(f"{name:34s} {a:8.3f} ms  {gbs:6.0f} GB/s ({gbs / peak * 100:5.1f}%)   torch composition {b:8.3f} ms  x{b / a:.2f}", flush=True)


with torch.no_grad():
    line("spatial_gradient sobel order1", lambda: K.filters.spatial_gradient(x), lambda: R.spatial_gradient(x), 12)
    line("spatial_gradient sobel order2", lambda: K.filters.spatial_gradient(x, "sobel", 2), lambda: R.spatial_gradient(x, "sobel", 2), 16)
    line("sobel magnitude", lambda: K.filters.sobel(x), lambda: R.sobel(x), 8)
    line("box_blur 5x5", lambda: K.filters.box_blur(x, 5), lambda: R.box_blur(x, 5), 8)
    line("box_blur 5x5 separable", lambda: K.filters.box_blur(x, 5, separable=True), lambda: R.box_blur(x, 5, separable=True), 8)
    line("laplacian 5x5", lambda: K.filters.laplacian(x, 5), lambda: R.laplacian(x, 5), 8)
    line("unsharp_mask 5x5", lambda: K.filters.unsharp_mask(x, (5, 5), (1.5, 1.5)), lambda: R.unsharp_mask(x, (5, 5), (1.5, 1.5)), 8)
    y = (x + 0.1 * torch.randn_like(x)).clamp(0, 1)
    line("ssim window 11 (fused, FMA bound)", lambda: K.metrics.ssim(x, y, 11), lambda: R.ssim(x, y, 11), 12)
    line("ssim window 5", lambda: K.metrics.ssim(x, y, 5), lambda: R.ssim(x, y, 5), 12)
    leaf = x[:8].clone().requires_grad_(True)
    with torch.enable_grad():
        composed = t(lambda: K.metrics.ssim(leaf, y[:8], 11), 5)
    print(f"ssim window 11, differentiable composition (B=8): {composed:.3f} ms", flush=True)
    del y, leaf
    ang = torch.linspace(-30, 30, B, device=dev)
    line("rotate +-30 deg bilinear", lambda: K.geometry.transform.rotate(x, ang), lambda: R.rotate(x, ang), 8)
    small = torch.linspace(-4, 4, B, device=dev)
    line("rotate +-4 deg bilinear", lambda: K.geometry.transform.rotate(x, small), lambda: R.rotate(x, small), 8)
    boxes = torch.tensor([[[100.0, 50.0], [1800.0, 60.0], [1790.0, 1000.0], [90.0, 1010.0]]], device=dev).expand(B, 4, 2).contiguous()
    line("crop_and_resize -> 1080x1920", lambda: K.geometry.transform.crop_and_resize(x, boxes, (H, W)),
         lambda: R.crop_and_resize(x, boxes, (H, W)), 8)
    # RandomPerspective data path: corner points -> homography -> warp (one fused launch for the homography vs ~45 torch launches)
    quad = torch.tensor([[0.0, 0.0], [W - 1.0, 0.0], [W - 1.0, H - 1.0], [0.0, H - 1.0]], device=dev).expand(B, 4, 2).contiguous()
    quad_to = quad + 8.0 * torch.randn(B, 4, 2, device=dev)
    KT = K.geometry.transform
    line("points -> H -> warp_perspective", lambda: K.warp_perspective(x, KT.get_perspective_transform(quad, quad_to), (H, W)),
         lambda: R.warp_perspective(x, R.perspective_from_points(quad, quad_to), (H, W)), 8)
    fused_h = t(lambda: KT.get_perspective_transform(quad, quad_to), 50)
    K.config.set("torch_prelude", 1)
    torch_h = t(lambda: KT.get_perspective_transform(quad, quad_to), 20)
    K.config.reset()
    print(f"get_perspective_transform alone (B={B}): fused {fused_h * 1e3:.1f} us, torch op sequence {torch_h * 1e3:.1f} us", flush=True)
    rows.append(dict(op="get_perspective_transform", fused_us=round(fused_h * 1e3, 1), torch_us=round(torch_h * 1e3, 1)))
out = os.path.join(ROOT, "gpurun_out", "family_bench.json")
os.makedirs(os.path.dirname(out), exist_ok=True)
json.dump(dict(B=B, shape=[B, 3, H, W], peak_gbs=peak, rows=rows), open(out, "w"), indent=1)
