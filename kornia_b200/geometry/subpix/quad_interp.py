"""Drop-in ``conv_quad_interp3d``, ``iterative_quad_interp3d``, ``ConvQuadInterp3d``, ``IterativeQuadInterp3d`` and
``AdaptiveQuadInterp3d`` (reference: kornia/geometry/subpix/spatial_soft_argmax.py).

Sub-pixel refinement of the maxima of a (B, C, D, H, W) scale-space response.  Every NMS maximum (the given
``precomputed_nms_mask``, else ``nms3d(input, (3, 3, 3), True)``) fits a quadratic to its 3 x 3 x 3 patch, solves for the
shift by Cramer's rule and, for up to ``n_iters`` iterations, steps one voxel along x, then y, then (``allow_scale_steps``)
the level wherever the shift exceeds ``max_subpixel_shift``.  The conv form looks the solve up in a table built over the
L-inf ``dilation_radius`` ball around every maximum, so a keypoint whose clamped position lies outside every ball becomes
invalid; the iterative form solves wherever the keypoint goes.  ``coords_max`` (B, C, 3, D, H, W) holds [level, x, y],
``y_max`` the input with the corrected response (plus ``strict_maxima_bonus`` on valid keypoints) at the maxima.

fp32 CUDA calls that need no gradient, with no mask or a contiguous bool mask of the input's shape, run as ONE CUDA kernel
(csrc/quad_interp.cuh) for the conv form with ``dilation_radius >= 1`` and the iterative form without ``max_candidates``:
no host synchronisation, so the call replays in a CUDA graph and compiles without a graph break.  The kernel is
bit-identical to ``_composed_*``: the reference's op sequence, which every other call runs and which is also the
differentiable path."""
from __future__ import annotations

from typing import Optional

import torch
from torch import nn

from ... import _ops
from .nms import nms3d

__all__ = ["conv_quad_interp3d", "iterative_quad_interp3d", "ConvQuadInterp3d", "IterativeQuadInterp3d", "AdaptiveQuadInterp3d"]

# the 3 x 3 x 3 patch, flattened as k = (dd + 1) * 9 + (dh + 1) * 3 + (dw + 1); the centre is k = 13
_PATCH = [(dd, dh, dw) for dd in (-1, 0, 1) for dh in (-1, 0, 1) for dw in (-1, 0, 1)]
_PATCH_D = torch.tensor([o[0] for o in _PATCH], dtype=torch.long)
_PATCH_H = torch.tensor([o[1] for o in _PATCH], dtype=torch.long)
_PATCH_W = torch.tensor([o[2] for o in _PATCH], dtype=torch.long)


def _k(dd: int, dh: int, dw: int) -> int:
    return (dd + 1) * 9 + (dh + 1) * 3 + (dw + 1)


def _check_input(input) -> None:
    if not torch.is_tensor(input):
        raise TypeError(f"Input type is not a torch.Tensor. Got {type(input)}")
    if input.ndim != 5:
        raise ValueError(f"Invalid input shape, expected BxCxDxHxW. Got: {input.shape}")


def _grid_and_copy(input: torch.Tensor):
    """The dense outputs before refinement: the [level, x, y] grid and ``input.clone()``."""
    B, C, D, H, W = input.shape
    coords_max = torch.empty(B, C, 3, D, H, W, device=input.device, dtype=input.dtype)
    coords_max[:, :, 0] = torch.arange(D, device=input.device, dtype=input.dtype).view(D, 1, 1)
    coords_max[:, :, 1] = torch.arange(W, device=input.device, dtype=input.dtype).view(1, 1, W)
    coords_max[:, :, 2] = torch.arange(H, device=input.device, dtype=input.dtype).view(1, H, 1)
    return coords_max, input.clone()


def _patch_offsets(H: int, W: int, device) -> torch.Tensor:
    return _PATCH_D.to(device) * (H * W) + _PATCH_H.to(device) * W + _PATCH_W.to(device)


def _solve_cramer_sym3x3(dxx, dyy, dss, dxy, dxs, dys, r0, r1, r2, eps: float = 1e-7):
    """(sx, sy, ss, solved) of [[dxx, dxy, dxs], [dxy, dyy, dys], [dxs, dys, dss]] s = r by Cramer's rule; an entry with
    |det| <= eps is unsolved and divided by 1."""
    cf00 = dyy * dss - dys * dys
    cf01 = dxy * dss - dys * dxs
    cf02 = dxy * dys - dyy * dxs
    det = dxx * cf00 - dxy * cf01 + dxs * cf02
    solved = det.abs() > eps
    safe_det = torch.where(solved, det, torch.ones_like(det))
    t1 = r1 * dss - dys * r2
    t3 = dxy * r2 - r1 * dxs
    sx = (r0 * cf00 - dxy * t1 + dxs * (r1 * dys - dyy * r2)) / safe_det
    sy = (dxx * t1 - r0 * cf01 + dxs * t3) / safe_det
    ss = (dxx * (dyy * r2 - r1 * dys) - dxy * t3 + r0 * cf02) / safe_det
    return sx, sy, ss, solved


def _fit(patch: torch.Tensor):
    """Gradient and solve of (N, 27) patches: (gx, gy, gs, sx, sy, ss, solved)."""
    def p(dd, dh, dw):
        return patch[:, _k(dd, dh, dw)]

    c2 = 2.0 * p(0, 0, 0)
    gx = 0.5 * (p(0, 0, 1) - p(0, 0, -1))
    gy = 0.5 * (p(0, 1, 0) - p(0, -1, 0))
    gs = 0.5 * (p(1, 0, 0) - p(-1, 0, 0))
    dxx = p(0, 0, 1) - c2 + p(0, 0, -1)
    dyy = p(0, 1, 0) - c2 + p(0, -1, 0)
    dss = p(1, 0, 0) - c2 + p(-1, 0, 0)
    dxy = 0.25 * (p(0, 1, 1) - p(0, 1, -1) - p(0, -1, 1) + p(0, -1, -1))
    dxs = 0.25 * (p(1, 0, 1) - p(1, 0, -1) - p(-1, 0, 1) + p(-1, 0, -1))
    dys = 0.25 * (p(1, 1, 0) - p(1, -1, 0) - p(-1, 1, 0) + p(-1, -1, 0))
    sx, sy, ss, solved = _solve_cramer_sym3x3(dxx, dyy, dss, dxy, dxs, dys, -gx, -gy, -gs)
    return gx, gy, gs, sx, sy, ss, solved


def _step(cur, shift, valid, limit, n):
    """One move along an axis: +-1 where a valid keypoint's shift exceeds the limit, valid only inside [1, n - 2], the
    position then clamped to [0, n - 1]."""
    new = cur + (valid & (shift > limit)).long() - (valid & (shift < -limit)).long()
    return new.clamp(0, n - 1), valid & (new >= 1) & (new <= n - 2)


class _Walk:
    """The per-keypoint state of the iteration loop, shared by both forms."""

    def __init__(self, d, h, w, dtype):
        N = d.shape[0]
        self.d, self.h, self.w = d.clone(), h.clone(), w.clone()
        self.valid = torch.ones(N, dtype=torch.bool, device=d.device)
        zeros = torch.zeros(N, device=d.device, dtype=dtype)
        self.sx, self.sy, self.ss, self.gds = zeros, zeros.clone(), zeros.clone(), zeros.clone()

    def clamped(self, D, H, W):
        return self.d.clamp(1, D - 2), self.h.clamp(1, H - 2), self.w.clamp(1, W - 2)

    def update(self, sx, sy, ss, gds, limit, allow_scale_steps, D, H, W):
        valid = self.valid
        self.sx = torch.where(valid, sx, self.sx)
        self.sy = torch.where(valid, sy, self.sy)
        self.ss = torch.where(valid, ss, self.ss)
        self.gds = torch.where(valid, gds, self.gds)
        self.w, valid = _step(self.w, sx, valid, limit, W)
        self.h, valid = _step(self.h, sy, valid, limit, H)
        if allow_scale_steps:
            self.d, valid = _step(self.d, ss, valid, limit, D)
        self.valid = valid


def _write_back(walk, coords_max, y_max, values, bc, d0, h0, w0, C, strict_maxima_bonus):
    """Coordinates and corrected responses of the keypoints into the dense outputs (``values``: the (BC, D, H, W) input)."""
    valid = walk.valid & (walk.sx.abs() <= 1.5) & (walk.sy.abs() <= 1.5) & (walk.ss.abs() <= 1.5)
    dtype = y_max.dtype
    b, c = bc // C, bc % C
    coords_max[b, c, 0, d0, h0, w0] = torch.where(valid, walk.d.to(dtype) + walk.ss, d0.to(dtype))
    coords_max[b, c, 1, d0, h0, w0] = torch.where(valid, walk.w.to(dtype) + walk.sx, w0.to(dtype))
    coords_max[b, c, 2, d0, h0, w0] = torch.where(valid, walk.h.to(dtype) + walk.sy, h0.to(dtype))
    correction = 0.5 * torch.where(valid, walk.gds, torch.zeros_like(walk.gds))
    y_max[b, c, d0, h0, w0] = values[bc, walk.d, walk.h, walk.w] + correction
    if strict_maxima_bonus > 0:
        y_max[b, c, d0, h0, w0] += strict_maxima_bonus * valid.to(dtype)


def _composed_conv_quad_interp3d(input, n_iters, strict_maxima_bonus, max_subpixel_shift, precomputed_nms_mask, dilation_radius,
                                 allow_scale_steps):
    """conv_quad_interp3d as the reference computes it: solves on the dilated maxima, a lookup table, then the walk."""
    B, C, D, H, W = input.shape
    coords_max, y_max = _grid_and_copy(input)
    if D < 3 or H < 3 or W < 3:
        return coords_max, y_max
    device, dtype = input.device, input.dtype
    BC, HW, DHW = B * C, H * W, D * H * W
    nms_mask = precomputed_nms_mask if precomputed_nms_mask is not None else nms3d(input, (3, 3, 3), True)
    bc, d0, h0, w0 = torch.where(nms_mask.view(BC, D, H, W))
    # every interior voxel within L-inf dilation_radius of a maximum (duplicates solve alike)
    r = dilation_radius
    offs = torch.arange(-r, r + 1, device=device, dtype=torch.long)
    od, oh, ow = (o.reshape(-1) for o in torch.meshgrid(offs, offs, offs, indexing="ij"))
    dd = (d0.unsqueeze(1) + od.unsqueeze(0)).reshape(-1)
    hh = (h0.unsqueeze(1) + oh.unsqueeze(0)).reshape(-1)
    ww = (w0.unsqueeze(1) + ow.unsqueeze(0)).reshape(-1)
    bb = bc.unsqueeze(1).expand(-1, od.shape[0]).reshape(-1)
    inner = (dd >= 1) & (dd <= D - 2) & (hh >= 1) & (hh <= H - 2) & (ww >= 1) & (ww <= W - 2)
    bb, dd, hh, ww = bb[inner], dd[inner], hh[inner], ww[inner]
    flat = input.view(-1)  # the reference's view: an input that cannot be viewed raises here
    at = bb * DHW + dd * HW + hh * W + ww
    gx, gy, gs, sx_t, sy_t, ss_t, solved_t = _fit(flat[at.unsqueeze(1) + _patch_offsets(H, W, device).unsqueeze(0)])
    gds_t = gx * sx_t + gy * sy_t + gs * ss_t
    table = torch.full((BC * DHW,), -1, dtype=torch.int32, device=device)
    table[at] = torch.arange(at.shape[0], dtype=torch.int32, device=device)
    walk = _Walk(d0, h0, w0, dtype)
    for _ in range(n_iters):
        di, hi, wi = walk.clamped(D, H, W)
        row = table[bc * DHW + di * HW + hi * W + wi].long()
        hit = row >= 0
        row = row.clamp(min=0)
        walk.valid = walk.valid & (solved_t[row] & hit)
        vf = walk.valid.to(dtype)
        walk.update(sx_t[row] * vf, sy_t[row] * vf, ss_t[row] * vf, gds_t[row], max_subpixel_shift, allow_scale_steps, D, H, W)
    _write_back(walk, coords_max, y_max, input.view(BC, D, H, W), bc, d0, h0, w0, C, strict_maxima_bonus)
    return coords_max, y_max


def _composed_iterative_quad_interp3d(input, n_iters, strict_maxima_bonus, max_subpixel_shift, allow_scale_steps, precomputed_nms_mask,
                                      max_candidates):
    """iterative_quad_interp3d as the reference computes it: the patch is gathered and solved at every step."""
    B, C, D, H, W = input.shape
    coords_max, y_max = _grid_and_copy(input)
    if D < 3 or H < 3 or W < 3:
        return coords_max, y_max
    dtype = input.dtype
    values = input.reshape(B * C, D, H, W)
    HW, DHW = H * W, D * H * W
    nms_mask = (precomputed_nms_mask if precomputed_nms_mask is not None else nms3d(input, (3, 3, 3), True)).view(B * C, D, H, W)
    bc, d0, h0, w0 = torch.where(nms_mask)
    if max_candidates is not None and bc.shape[0] > max_candidates:  # the strongest maxima by pre-refinement response
        _, top = torch.topk(values[bc, d0, h0, w0], k=max_candidates)
        bc, d0, h0, w0 = bc[top], d0[top], h0[top], w0[top]
    offsets = _patch_offsets(H, W, input.device)
    flat = values.reshape(-1)
    walk = _Walk(d0, h0, w0, dtype)
    for _ in range(n_iters):
        di, hi, wi = walk.clamped(D, H, W)
        gx, gy, gs, sx, sy, ss, solved = _fit(flat[(bc * DHW + di * HW + hi * W + wi).unsqueeze(1) + offsets.unsqueeze(0)])
        walk.valid = walk.valid & solved
        vf = walk.valid.to(dtype)
        sx, sy, ss = sx * vf, sy * vf, ss * vf
        walk.update(sx, sy, ss, gx * sx + gy * sy + gs * ss, max_subpixel_shift, allow_scale_steps, D, H, W)
    _write_back(walk, coords_max, y_max, values, bc, d0, h0, w0, C, strict_maxima_bonus)
    return coords_max, y_max


def _fused(input, mask, n_iters, strict_maxima_bonus, max_subpixel_shift, radius, allow_scale_steps):
    """The kernel's (coords_max, y_max), or None when the call takes the composition (``radius`` 0: the iterative form).
    The conv form keeps the composition's ``input.view(-1)``, so an input that cannot be viewed raises as there."""
    if not (input.dtype == torch.float32 and input.is_cuda and not (torch.is_grad_enabled() and input.requires_grad)):
        return None
    if mask is not None and not (mask.dtype == torch.bool and mask.shape == input.shape and mask.device == input.device and mask.is_contiguous()):
        return None
    if type(n_iters) is not int or not -(2**31) <= n_iters < 2**31 or type(radius) is not int:
        return None
    if not all(isinstance(v, (int, float)) for v in (strict_maxima_bonus, max_subpixel_shift)):
        return None
    if radius > 0 and min(input.shape[2:]) >= 3:
        input.view(-1)
    return _ops.ops.quad_interp3d_fwd(input, mask, n_iters, float(max_subpixel_shift), float(strict_maxima_bonus), radius,
                                      bool(allow_scale_steps))


def conv_quad_interp3d(
    input: torch.Tensor,
    n_iters: int = 5,
    strict_maxima_bonus: float = 10.0,
    max_subpixel_shift: float = 0.6,
    precomputed_nms_mask: Optional[torch.Tensor] = None,
    dilation_radius: int = 1,
    allow_scale_steps: bool = True,
) -> tuple[torch.Tensor, torch.Tensor]:
    r"""Sub-pixel refinement of the 3-D maxima of ``input`` (B, C, D, H, W) by quadratic interpolation, with the solves
    tabulated over the L-inf ``dilation_radius`` ball around every maximum: ``(coords_max, y_max)``.

    ``coords_max`` (B, C, 3, D, H, W) holds [level, x, y]: refined at the maxima, the grid elsewhere.  ``y_max`` is the
    input with the quadratically corrected response, plus ``strict_maxima_bonus`` when it is positive, at the valid maxima.
    ``precomputed_nms_mask`` (bool, the input's shape) replaces the internal ``nms3d``.
    """
    _check_input(input)
    if isinstance(dilation_radius, int) and dilation_radius >= 1:  # a radius <= 0 can index the composition's empty table
        out = _fused(input, precomputed_nms_mask, n_iters, strict_maxima_bonus, max_subpixel_shift, dilation_radius, allow_scale_steps)
        if out is not None:
            return out
    return _composed_conv_quad_interp3d(input, n_iters, strict_maxima_bonus, max_subpixel_shift, precomputed_nms_mask, dilation_radius,
                                        allow_scale_steps)


def iterative_quad_interp3d(
    input: torch.Tensor,
    n_iters: int = 5,
    strict_maxima_bonus: float = 10.0,
    max_subpixel_shift: float = 0.6,
    allow_scale_steps: bool = True,
    precomputed_nms_mask: Optional[torch.Tensor] = None,
    max_candidates: Optional[int] = None,
) -> tuple[torch.Tensor, torch.Tensor]:
    r"""Sub-pixel refinement of the 3-D maxima of ``input`` (B, C, D, H, W) by quadratic interpolation, re-solving the
    3 x 3 x 3 patch wherever a keypoint moves: ``(coords_max, y_max)`` as :func:`conv_quad_interp3d` returns them.

    ``max_candidates`` keeps only that many maxima, the strongest before refinement; the others keep the grid and input.
    """
    _check_input(input)
    if max_candidates is None:
        out = _fused(input, precomputed_nms_mask, n_iters, strict_maxima_bonus, max_subpixel_shift, 0, allow_scale_steps)
        if out is not None:
            return out
    return _composed_iterative_quad_interp3d(input, n_iters, strict_maxima_bonus, max_subpixel_shift, allow_scale_steps,
                                             precomputed_nms_mask, max_candidates)


class ConvQuadInterp3d(nn.Module):
    r"""Module form of :func:`conv_quad_interp3d`."""

    def __init__(
        self,
        n_iters: int = 5,
        strict_maxima_bonus: float = 10.0,
        max_subpixel_shift: float = 0.6,
        dilation_radius: int = 1,
        allow_scale_steps: bool = True,
    ) -> None:
        super().__init__()
        self.n_iters = n_iters
        self.strict_maxima_bonus = strict_maxima_bonus
        self.max_subpixel_shift = max_subpixel_shift
        self.dilation_radius = dilation_radius
        self.allow_scale_steps = allow_scale_steps

    def __repr__(self) -> str:
        return (
            f"{self.__class__.__name__}(n_iters={self.n_iters}, strict_maxima_bonus={self.strict_maxima_bonus}, "
            f"max_subpixel_shift={self.max_subpixel_shift}, dilation_radius={self.dilation_radius}, "
            f"allow_scale_steps={self.allow_scale_steps})"
        )

    def forward(self, x: torch.Tensor, precomputed_nms_mask: Optional[torch.Tensor] = None) -> tuple[torch.Tensor, torch.Tensor]:
        """Refined coordinates and responses of the maxima of ``x`` (B, C, D, H, W)."""
        return conv_quad_interp3d(x, self.n_iters, self.strict_maxima_bonus, self.max_subpixel_shift, precomputed_nms_mask,
                                  self.dilation_radius, self.allow_scale_steps)


class IterativeQuadInterp3d(nn.Module):
    r"""Module form of :func:`iterative_quad_interp3d`."""

    def __init__(
        self,
        n_iters: int = 5,
        strict_maxima_bonus: float = 10.0,
        max_subpixel_shift: float = 0.6,
        allow_scale_steps: bool = True,
        max_candidates: Optional[int] = None,
    ) -> None:
        super().__init__()
        self.n_iters = n_iters
        self.strict_maxima_bonus = strict_maxima_bonus
        self.max_subpixel_shift = max_subpixel_shift
        self.allow_scale_steps = allow_scale_steps
        self.max_candidates = max_candidates

    def __repr__(self) -> str:
        return (
            f"{self.__class__.__name__}(n_iters={self.n_iters}, strict_maxima_bonus={self.strict_maxima_bonus}, "
            f"max_subpixel_shift={self.max_subpixel_shift}, allow_scale_steps={self.allow_scale_steps}, "
            f"max_candidates={self.max_candidates})"
        )

    def forward(self, x: torch.Tensor, precomputed_nms_mask: Optional[torch.Tensor] = None) -> tuple[torch.Tensor, torch.Tensor]:
        """Refined coordinates and responses of the maxima of ``x`` (B, C, D, H, W)."""
        return iterative_quad_interp3d(x, self.n_iters, self.strict_maxima_bonus, self.max_subpixel_shift, self.allow_scale_steps,
                                       precomputed_nms_mask=precomputed_nms_mask, max_candidates=self.max_candidates)


class AdaptiveQuadInterp3d(nn.Module):
    r"""Sub-pixel refinement that picks its form: ``mode`` "conv" (:func:`conv_quad_interp3d`), "patch"
    (:func:`iterative_quad_interp3d`) or "auto" (conv on CUDA inputs, patch otherwise).  ``dilation_radius`` applies to the
    conv form and ``max_candidates`` to the patch form."""

    MODES = ("patch", "conv", "auto")

    def __init__(
        self,
        mode: str = "auto",
        n_iters: int = 5,
        strict_maxima_bonus: float = 10.0,
        max_subpixel_shift: float = 0.6,
        dilation_radius: int = 1,
        allow_scale_steps: bool = True,
        max_candidates: Optional[int] = None,
    ) -> None:
        super().__init__()
        if mode not in self.MODES:
            raise ValueError(f"mode must be one of {self.MODES}, got '{mode}'")
        self.mode = mode
        self.n_iters = n_iters
        self.strict_maxima_bonus = strict_maxima_bonus
        self.max_subpixel_shift = max_subpixel_shift
        self.dilation_radius = dilation_radius
        self.allow_scale_steps = allow_scale_steps
        self.max_candidates = max_candidates

    def __repr__(self) -> str:
        return (
            f"{self.__class__.__name__}(mode='{self.mode}', n_iters={self.n_iters}, "
            f"strict_maxima_bonus={self.strict_maxima_bonus}, max_subpixel_shift={self.max_subpixel_shift}, "
            f"dilation_radius={self.dilation_radius}, allow_scale_steps={self.allow_scale_steps}, "
            f"max_candidates={self.max_candidates})"
        )

    def forward(self, x: torch.Tensor, precomputed_nms_mask: Optional[torch.Tensor] = None) -> tuple[torch.Tensor, torch.Tensor]:
        """Refined coordinates and responses of the maxima of ``x`` (B, C, D, H, W) by the form ``mode`` selects."""
        if self.mode == "conv" or (self.mode == "auto" and x.is_cuda):
            return conv_quad_interp3d(x, self.n_iters, self.strict_maxima_bonus, self.max_subpixel_shift, precomputed_nms_mask,
                                      self.dilation_radius, self.allow_scale_steps)
        return iterative_quad_interp3d(x, self.n_iters, self.strict_maxima_bonus, self.max_subpixel_shift, self.allow_scale_steps,
                                       precomputed_nms_mask=precomputed_nms_mask, max_candidates=self.max_candidates)
