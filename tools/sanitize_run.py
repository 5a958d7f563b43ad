"""Small workload for compute-sanitizer (memcheck / racecheck / synccheck): tiled forward (3 interpolations),
tiled backward, tiled separable filter, the derivative stencils, at sizes with several tiles per CTA and partial edge tiles."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import kornia_b200 as K
dev = "cuda"
g = torch.Generator().manual_seed(0)
B, C, H, W = 3, 3, 100, 192
src = torch.rand(B, C, H, W, generator=g).to(dev)
M = (torch.eye(3)[None].repeat(B, 1, 1) + 0.01 * torch.randn(B, 3, 3, generator=g))
M[:, 2, :2] *= 0.01
M = M.to(dev)
for mode in ("bilinear", "nearest", "bicubic"):
    for pad in ("zeros", "fill"):
        K.warp_perspective(src, M, (90, 200), mode=mode, padding_mode=pad, fill_value=torch.tensor([0.1, 0.2, 0.3], device=dev))
# many strips (400 x 3 >= 8 x the SM count): the run-time work distribution of the headline kernel (warp_fwd_tma<DYN>)
many = torch.rand(400, 3, 96, 192, generator=g).to(dev)
Mmany = M[:1].expand(400, -1, -1).contiguous()
K.warp_perspective(many, Mmany, (96, 192))
K.warp_affine(many, Mmany[:, :2].contiguous(), (96, 192), align_corners=False)
sm, mm = many.clone().requires_grad_(True), Mmany.clone().requires_grad_(True)   # ... and of the backward kernel (warp_bwd_tma2<DYN>)
torch.autograd.grad(K.warp_perspective(sm, mm, (96, 192)).sum(), [sm, mm])
del many, sm, mm
s = src.clone().requires_grad_(True)
m = M.clone().requires_grad_(True)
out = K.warp_perspective(s, m, (H, W))
torch.autograd.grad(out.sum(), [s, m])
for pad in ("zeros", "border", "reflection"):  # 'reflection': INNER and border tiles, a sample shifted out of the image by 30 rows
    Ms = M.clone()
    Ms[0, 1, 2] += 30.0
    K.warp_perspective(src, Ms, (H, W), padding_mode=pad)
    K.warp_perspective(src, Ms, (H, W), mode="nearest", padding_mode=pad, align_corners=False)
# remap: the pipelined persistent kernel (zeros / border, maps through TMA), the one-CTA-per-tile kernel (reflection; odd width)
ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
mx = (xs + 3.0 * torch.sin(ys / 9.0) - 4.0)[None].repeat(B, 1, 1).to(dev)
my = (ys + 2.5 * torch.cos(xs / 11.0) + 1.0)[None].repeat(B, 1, 1).to(dev)
for pad in ("zeros", "border", "reflection"):
    K.remap(src, mx, my, padding_mode=pad, align_corners=True)
    K.remap(src, mx[:1], my[:1], padding_mode=pad)
    K.remap(src, mx[:, :90, :150].contiguous(), my[:, :90, :150].contiguous(), padding_mode=pad)   # w % 4 != 0: not TMA-addressable
K.gaussian_blur2d(src, (11, 11), (2.0, 2.0))
K.gaussian_blur2d(src, (5, 5), (1.0, 1.0), "replicate")
# image derivatives: odd width (scalar path), aligned width (vector path), backward, fused magnitude, 5x5 stencils
for shape in ((2, 3, 33, 45), (1, 2, 16, 256), (2, 1, 1, 7), (3, 1, 2, 2)):
    xg = torch.rand(*shape, generator=g).to(dev).requires_grad_(True)
    for mode, order in (("sobel", 1), ("sobel", 2), ("diff", 2)):
        K.filters.spatial_gradient(xg, mode, order).sum().backward()
    K.filters.sobel(xg.detach())
    K.filters.sobel(xg).sum().backward()
for ws in (3, 7, 11):
    K.metrics.ssim(src, src.flip(-1).contiguous(), ws)
odd = torch.rand(2, 1, 45, 67, generator=g).to(dev)
K.metrics.ssim(odd, odd.flip(-2).contiguous(), 5, padding="valid")
K.filters.box_blur(src, (3, 5))
K.filters.laplacian(src, 5)
K.geometry.transform.rotate(src, torch.tensor([10.0, 20.0, 30.0], device=dev))
K.geometry.transform.center_crop(src, (50, 60))
# callers added after the round-1 GPU budget was spent: pyramids, resize, undistort (all on the default kernels)
KT, KC = K.geometry.transform, K.geometry.calibration
KT.pyrdown(src)
KT.pyrup(src[:, :, :40, :64].contiguous())
KT.build_laplacian_pyramid(src, 3)
KT.resize(src, (40, 77), antialias=True)
cam = torch.tensor([[150.0, 0.0, 96.0], [0.0, 150.0, 50.0], [0.0, 0.0, 1.0]], device=dev).expand(B, 3, 3).contiguous()
KC.undistort_image(src, cam, torch.tensor([[-0.2, 0.05, 0.001, -0.002, 0.01]], device=dev).expand(B, 5).contiguous())
# uint8 ingest warps: the tiled kernel (W % 4 == 0), the per-tap kernel (odd width; switch u8_tiled = 0), partial tiles, every padding
for shape in ((3, 100, 192, 3), (2, 33, 45, 3), (2, 70, 132, 1), (1, 5, 4, 3), (2, 40, 64, 4)):
    frames = torch.randint(0, 256, shape, generator=g, dtype=torch.uint8).to(dev)
    Mq = M[: shape[0]].clone()
    for tiled in (1, 0):
        K.config.set("u8_tiled", tiled)
        for pad in ("zeros", "border", "reflection"):
            KT.warp_perspective_from_uint8(frames, Mq, (shape[1] + 3, shape[2] - 1), padding_mode=pad)
            KT.warp_affine_from_uint8(frames, Mq[:, :2].contiguous(), (shape[1], shape[2]), padding_mode=pad, align_corners=False)
    K.config.reset()
    if shape[3] == 3:
        KT.warp_perspective_from_uint8(frames, Mq, (shape[1], shape[2]), mode="bicubic", padding_mode="fill", fill_value=torch.tensor([0.1, 0.2, 0.3]))
        KT.warp_perspective_from_uint8(frames, Mq, (shape[1], shape[2]), padding_mode="fill", fill_value=torch.tensor([0.1, 0.2, 0.3]))
for shape in ((3, 100, 192, 3), (2, 70, 132, 1), (1, 33, 45, 3)):  # the last one: odd width -> conversion + fp32 path
    frames = torch.randint(0, 256, shape, generator=g, dtype=torch.uint8).to(dev)
    camq = torch.tensor([[0.8 * shape[2], 0.0, shape[2] / 2], [0.0, 0.8 * shape[2], shape[1] / 2], [0.0, 0.0, 1.0]], device=dev).expand(shape[0], 3, 3).contiguous()
    KC.undistort_image_from_uint8(frames, camq, torch.tensor([[-0.2, 0.05, 0.001, -0.002, 0.01]], device=dev).expand(shape[0], 5).contiguous())
# ScalePyramid: the octave kernel (blur and copy stages, a band of 4 columns, more CTAs than bands), tiny octaves composed
KT.ScalePyramid(min_size=8)(torch.rand(2, 1, 100, 132, generator=g).to(dev))
# non-maximum suppression: the 2-D kernel in both forms (explicit 5 x 5 and general 15 x 15, odd width, partial tiles), the
# 3-D kernel on a permuted (B, C, L, H, W) view in both nms3d forms and as nms3d_minmax
KG = K.geometry
resp = torch.rand(2, 2, 70, 133, generator=g).to(dev)
KG.nms2d(resp, (5, 5), True)
KG.NonMaximaSuppression2d((15, 15)).to(dev)(resp)
octv = torch.rand(1, 5, 2, 37, 61, generator=g).to(dev).permute(0, 2, 1, 3, 4)
KG.nms3d(octv, (3, 3, 3), True)
KG.nms3d(octv, (3, 3, 3))
KG.nms3d_minmax(octv)
# sub-pixel refinement on rough permuted (B, C, L, H, W) views with an odd width and partial tiles, so keypoints walk and
# read patches across tiles: the conv form with nms3d_minmax's mask (C = 1, as the conv form must view its input) and the
# iterative form computing its own NMS
rough = torch.randn(1, 5, 1, 37, 61, generator=g).to(dev).permute(0, 2, 1, 3, 4)
KG.conv_quad_interp3d(rough, 5, 10.0, 0.3, KG.nms3d_minmax(rough)[0], 2)
KG.iterative_quad_interp3d(torch.randn(1, 5, 2, 37, 61, generator=g).to(dev).permute(0, 2, 1, 3, 4), 5, 10.0, 0.3)
# per-patch gradient histograms: SIFT on a batch-strided view of odd-sized patches (a grid that does not divide N) and the
# dominant orientation at the reference's LAFOrienter size
with torch.no_grad():
    K.feature.SIFTDescriptor(19, 5, 3)(torch.rand(37, 1, 23, 23, generator=g).to(dev)[::2, :, 2:21, 1:20])
    K.feature.PatchDominantGradientOrientation(19)(torch.rand(41, 1, 19, 19, generator=g).to(dev))
torch.cuda.synchronize()
print("sanitize workload done")
