"""Plain-torch restatement of the reference's sub-pixel refinement (kornia/geometry/subpix/spatial_soft_argmax.py), written
from its semantics rather than its op sequence: the quadratic fit is evaluated densely over every interior voxel (one
rounding per operation, in the reference's order), and the conv form's lookup table is stated as a dilation of the mask.

* The maxima: the given mask, else nms3d(x, (3, 3, 3), True) (strictly above the NaN-propagating max of the 26
  neighbours; border False).  D, H or W < 3: the grid and the copy.
* Per iteration: the fit at the position clamped to [1, n - 2]; the conv form also needs a mask-True voxel within L-inf
  ``dilation_radius`` of that position.  A failed keypoint keeps its last shift and stops; a solved one moves along x,
  then y, then (allow_scale_steps) the level where the shift exceeds the threshold (fp32 comparison), each move valid
  only inside [1, n - 2], the position clamped to [0, n - 1].
* valid = still valid and every |shift| <= 1.5: coords = position + shift, else the grid; y = x[position] +
  0.5 * (valid ? g . s : 0), + bonus * valid when the bonus is > 0.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F


def _maxima(x):
    B, C, D, H, W = x.shape
    mask = torch.zeros(B, C, D, H, W, dtype=torch.bool)
    win = x.unfold(2, 3, 1).unfold(3, 3, 1).unfold(4, 3, 1).reshape(B, C, D - 2, H - 2, W - 2, 27)
    nb = torch.cat([win[..., :13], win[..., 14:]], -1)
    mask[..., 1:-1, 1:-1, 1:-1] = win[..., 13] > nb.amax(-1)
    return mask


def _dense_fit(v):
    """(sx, sy, ss, gds, solved) of every interior voxel of the (N, D, H, W) volume, as (N, D - 2, H - 2, W - 2)."""
    D, H, W = v.shape[1:]

    def at(dd, dh, dw):
        return v[:, 1 + dd:D - 1 + dd, 1 + dh:H - 1 + dh, 1 + dw:W - 1 + dw]

    c, xm, xp, ym, yp, sm, sp = at(0, 0, 0), at(0, 0, -1), at(0, 0, 1), at(0, -1, 0), at(0, 1, 0), at(-1, 0, 0), at(1, 0, 0)
    gx, gy, gs = 0.5 * (xp - xm), 0.5 * (yp - ym), 0.5 * (sp - sm)
    dxx, dyy, dss = xp - 2.0 * c + xm, yp - 2.0 * c + ym, sp - 2.0 * c + sm
    dxy = 0.25 * (at(0, 1, 1) - at(0, 1, -1) - at(0, -1, 1) + at(0, -1, -1))
    dxs = 0.25 * (at(1, 0, 1) - at(1, 0, -1) - at(-1, 0, 1) + at(-1, 0, -1))
    dys = 0.25 * (at(1, 1, 0) - at(1, -1, 0) - at(-1, 1, 0) + at(-1, -1, 0))
    b0, b1, b2 = -gx, -gy, -gs
    m00 = dyy * dss - dys * dys
    m01 = dxy * dss - dys * dxs
    m02 = dxy * dys - dyy * dxs
    det = dxx * m00 - dxy * m01 + dxs * m02
    solved = det.abs() > 1e-7
    det = torch.where(solved, det, torch.ones_like(det))
    sx = (b0 * m00 - dxy * (b1 * dss - dys * b2) + dxs * (b1 * dys - dyy * b2)) / det
    sy = (dxx * (b1 * dss - dys * b2) - b0 * m01 + dxs * (dxy * b2 - b1 * dxs)) / det
    ss = (dxx * (dyy * b2 - b1 * dys) - dxy * (dxy * b2 - b1 * dxs) + b0 * m02) / det
    return gx, gy, gs, sx, sy, ss, solved


def refine(x, n_iters=5, strict_maxima_bonus=10.0, max_subpixel_shift=0.6, mask=None, dilation_radius=None, allow_scale_steps=True,
           max_candidates=None):
    """The conv form when ``dilation_radius`` is given, else the iterative form."""
    B, C, D, H, W = x.shape
    grid = torch.stack(torch.meshgrid(torch.arange(D), torch.arange(W), torch.arange(H), indexing="ij")).to(x.dtype)
    coords = grid.permute(0, 1, 3, 2).expand(B, C, 3, D, H, W).clone()
    y = x.clone()
    if D < 3 or H < 3 or W < 3:
        return coords, y
    m = (mask if mask is not None else _maxima(x)).reshape(B * C, D, H, W)
    v = x.reshape(B * C, D, H, W)
    n, d, h, w = (t.clone() for t in torch.nonzero(m, as_tuple=True))
    if max_candidates is not None and n.numel() > max_candidates:
        keep = torch.topk(v[n, d, h, w], max_candidates).indices
        n, d, h, w = n[keep], d[keep], h[keep], w[keep]
    d0, h0, w0 = d.clone(), h.clone(), w.clone()
    gx, gy, gs, sx_a, sy_a, ss_a, ok_a = _dense_fit(v)
    gds_a = gx * sx_a + gy * sy_a + gs * ss_a
    if dilation_radius is not None:
        k = 2 * dilation_radius + 1
        near = F.max_pool3d(m.float().unsqueeze(1), k, 1, dilation_radius).squeeze(1) > 0
    lim = torch.tensor(max_subpixel_shift, dtype=x.dtype)
    valid = torch.ones(n.shape, dtype=torch.bool)
    shift = torch.zeros(3, n.numel(), dtype=x.dtype)  # x, y, level
    gds = torch.zeros(n.numel(), dtype=x.dtype)
    for _ in range(n_iters):
        di, hi, wi = d.clamp(1, D - 2), h.clamp(1, H - 2), w.clamp(1, W - 2)
        at = (n, di - 1, hi - 1, wi - 1)
        ok = ok_a[at] if dilation_radius is None else ok_a[at] & near[n, di, hi, wi]
        valid = valid & ok
        s = torch.stack([sx_a[at], sy_a[at], ss_a[at]])
        shift = torch.where(valid, s, shift)
        gds = torch.where(valid, gds_a[at], gds)
        for axis, (pos, size) in enumerate(((w, W), (h, H), (d, D))):
            if axis == 2 and not allow_scale_steps:
                break
            new = pos + (valid & (s[axis] > lim)).long() - (valid & (s[axis] < -lim)).long()
            valid = valid & (new >= 1) & (new <= size - 2)
            pos.copy_(new.clamp(0, size - 1))
    valid = valid & (shift.abs() <= 1.5).all(0)
    b, c = n // C, n % C
    for axis, (pos, pos0) in enumerate(((d, d0), (w, w0), (h, h0))):
        coords[b, c, axis, d0, h0, w0] = torch.where(valid, pos.to(x.dtype) + shift[(2, 0, 1)[axis]], pos0.to(x.dtype))
    val = v[n, d, h, w] + 0.5 * torch.where(valid, gds, torch.zeros_like(gds))
    if strict_maxima_bonus > 0:
        val = val + strict_maxima_bonus * valid.to(x.dtype)
    y[b, c, d0, h0, w0] = val
    return coords, y
