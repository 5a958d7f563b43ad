"""Plain-torch restatement of the reference's non-maximum suppression (kornia/geometry/subpix/nms.py), written from its
semantics rather than its op sequence: keep = x > M, M the NaN-propagating maximum (torch.amax) of a neighbour set.

* 2-D K = 3, 5, 7: the K*K - 1 neighbours; the outer (K - 1) / 2 ring is False.
* 2-D other square sizes: the neighbours of the replicate-padded image and 0; a window holding a non-finite texel is False.
* 2-D even or non-square sizes: the reference's conv output does not view as (B, C, -1, H, W): the same RuntimeError.
* 3-D (3, 3, 3) and nms3d_minmax: the 26 neighbours (x < amin for the minima); border levels, rows and columns are False.
* Values: x * mask.to(x.dtype).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F


def _values(x, mask, mask_only):
    return mask if mask_only else x * mask.to(x.dtype)


def _windows2d(xp, kh, kw):
    return xp.unfold(2, kh, 1).unfold(3, kw, 1)  # (B, C, H', W', kh, kw)


def nms2d(x: torch.Tensor, kernel_size, mask_only: bool = False) -> torch.Tensor:
    B, C, H, W = x.shape
    ky, kx = kernel_size
    if (ky, kx) in ((3, 3), (5, 5), (7, 7)):
        r = ky // 2
        mask = torch.zeros(B, C, H, W, dtype=torch.bool)
        if H > 2 * r and W > 2 * r:
            win = _windows2d(x, ky, kx).reshape(B, C, H - 2 * r, W - 2 * r, ky * kx)
            c = win[..., (ky * kx) // 2]
            nb = torch.cat([win[..., : (ky * kx) // 2], win[..., (ky * kx) // 2 + 1:]], -1)
            mask[..., r:H - r, r:W - r] = c > nb.amax(-1)
        return _values(x, mask, mask_only)
    # the reference's padding mixes the two axes and its weight swaps them: reproduce the shape its .view sees
    py, px = (ky - 1) // 2, (kx - 1) // 2
    HP, WP = H + px + py, W + px + py
    if ky != kx:
        torch.empty(B * C, ky * kx, HP - kx + 1, WP - ky + 1).view(B, C, -1, H, W)
    xp = F.pad(x, (px, py, px, py), mode="replicate")
    win = _windows2d(xp, ky, kx).reshape(B * C, -1, ky * kx)
    if win.shape[1] != H * W:  # even sizes: the reference's view raises
        torch.empty(B * C, ky * kx, win.shape[1]).view(B, C, -1, H, W)
    win = win.reshape(B, C, H, W, ky * kx)
    finite = torch.isfinite(win).all(-1)
    nb = win.clone()
    nb[..., (ky * kx) // 2] = 0.0
    mask = finite & (x > nb.amax(-1))
    return _values(x, mask, mask_only)


def _interior3d(x, greater):
    B, C, D, H, W = x.shape
    mask = torch.zeros(B, C, D, H, W, dtype=torch.bool)
    if D > 2 and H > 2 and W > 2:
        win = x.unfold(2, 3, 1).unfold(3, 3, 1).unfold(4, 3, 1).reshape(B, C, D - 2, H - 2, W - 2, 27)
        c = win[..., 13]
        nb = torch.cat([win[..., :13], win[..., 14:]], -1)
        mask[..., 1:-1, 1:-1, 1:-1] = c > nb.amax(-1) if greater else c < nb.amin(-1)
    return mask


def nms3d(x: torch.Tensor, kernel_size, mask_only: bool = False) -> torch.Tensor:
    if tuple(kernel_size) != (3, 3, 3):
        # the reference pads by k on each side: its conv output does not view as (B, C, -1, D, H, W)
        B, C, D, H, W = x.shape
        kd, ky, kx = kernel_size
        torch.empty(B, C * kd * ky * kx, D + kd + 1, H + ky + 1, W + kx + 1).view(B, C, -1, D, H, W)
    return _values(x, _interior3d(x, True), mask_only)


def nms3d_minmax(x: torch.Tensor):
    return _interior3d(x, True), _interior3d(x, False)
