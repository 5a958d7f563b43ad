"""ORACLE for ScalePyramid (test infrastructure, not product code): the reference's octave builder
(kornia/geometry/transform/pyramid.py:151-404) restated with the same ATen calls -- per level a reflect F.pad and a
grouped F.conv2d for the rows, then the same for the columns, the clamped gaussian_blur2d of oracle/kornia_restated.py
on levels smaller than the kernel, bilinear ``align_corners=True`` octave seeds and ``torch.stack``.  It runs on whatever
device its argument lives on; on CUDA it is the reference composition tools/bench_scale_pyramid.py times the octave
kernel against."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from oracle import kornia_restated as R


def kernel_size(sigma: float) -> int:
    k = int(2.0 * 4.0 * sigma + 1.0)
    return k + 1 if k % 2 == 0 else k


def gaussian1d(sigma: float, ksize: int) -> torch.Tensor:
    x = torch.arange(ksize, dtype=torch.float64) - ksize // 2
    k = torch.exp(-0.5 * x**2 / sigma**2)
    return (k / k.sum()).float()


def blur(x: torch.Tensor, k: torch.Tensor) -> torch.Tensor:
    """Separable reflect-bordered blur with a 1-D kernel: rows, then columns."""
    K, C = k.shape[0], x.shape[1]
    k = k.to(device=x.device, dtype=x.dtype)
    rows = F.conv2d(F.pad(x, (K // 2, K // 2, 0, 0), mode="reflect"), k.view(1, 1, 1, K).expand(C, 1, 1, K).contiguous(), groups=C)
    return F.conv2d(F.pad(rows, (0, 0, K // 2, K // 2), mode="reflect"), k.view(1, 1, K, 1).expand(C, 1, K, 1).contiguous(), groups=C)


def kernels(n_levels=3, init_sigma=1.6, double_image=False, extra_levels=3):
    """(initial kernel or None, level kernels): the buffers _gk_init, _gk_0 ... of the reference module."""
    step = 2 ** (1.0 / float(n_levels))
    assumed = 1.0 if double_image else 0.5
    init = None
    if init_sigma > assumed:
        s = max(math.sqrt(init_sigma**2 - assumed**2), 0.01)
        init = gaussian1d(s, kernel_size(s))
    levels, cur = [], init_sigma
    for _ in range(n_levels + extra_levels - 1):
        d = cur * math.sqrt(step**2 - 1.0)
        levels.append(gaussian1d(d, kernel_size(d)))
        cur *= step
    return init, levels


def scale_pyramid(x, n_levels=3, init_sigma=1.6, min_size=15, double_image=False, extra_levels=3):
    """(pyr, sigmas, pixel_dists) as the reference's ScalePyramid(...)(x) returns them."""
    step = 2 ** (1.0 / float(n_levels))
    L = n_levels + extra_levels
    init, ks = kernels(n_levels, init_sigma, double_image, extra_levels)
    bs = x.shape[0]
    pixel_distance, cur_sigma = 1.0, 0.5
    if double_image:
        x = F.interpolate(x, scale_factor=2.0, mode="bilinear", align_corners=True)
        pixel_distance, cur_sigma = 0.5, 1.0
    if init_sigma > cur_sigma:
        s = max(math.sqrt(init_sigma**2 - cur_sigma**2), 0.01)
        ksize, min_dim = kernel_size(s), min(x.shape[2], x.shape[3])
        if ksize <= min_dim:
            x = blur(x, init)
        else:
            ksize = min(ksize, min_dim if min_dim % 2 == 1 else min_dim - 1)
            x = R.gaussian_blur2d(x, (ksize, ksize), torch.tensor([[s, s]], device=x.device, dtype=x.dtype))
        cur_sigma = init_sigma
    sigmas = [torch.full((bs, L), cur_sigma, device=x.device, dtype=x.dtype)]
    pds = [torch.full((bs, L), pixel_distance, device=x.device, dtype=x.dtype)]
    pyr = [[x]]
    while True:
        cur = init_sigma
        for lvl in range(1, L):
            prev = pyr[-1][-1]
            min_dim = min(prev.shape[2], prev.shape[3])
            if ks[lvl - 1].shape[0] <= min_dim:
                new = blur(prev, ks[lvl - 1])
            else:
                d = cur * math.sqrt(step**2 - 1.0)
                ksize = min_dim if min_dim % 2 == 1 else min_dim - 1
                new = R.gaussian_blur2d(prev, (ksize, ksize), torch.tensor([[d, d]], device=x.device, dtype=x.dtype))
            cur *= step
            pyr[-1].append(new)
            sigmas[-1][:, lvl] = cur
            pds[-1][:, lvl] = pixel_distance
        top = pyr[-1][-extra_levels]
        H, W = top.shape[2], top.shape[3]
        if min(H // 2, W // 2) <= min_size:
            break
        pyr.append([F.interpolate(top, size=(H // 2, W // 2), mode="bilinear", align_corners=True)])
        pixel_distance *= 2.0
        sigmas.append(torch.full((bs, L), init_sigma, device=x.device, dtype=x.dtype))
        pds.append(torch.full((bs, L), pixel_distance, device=x.device, dtype=x.dtype))
    return [torch.stack(p, 2) for p in pyr], sigmas, pds
