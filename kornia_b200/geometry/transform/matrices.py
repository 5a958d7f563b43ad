"""Small (B,2,3)/(B,3,3) matrix builders used by the warp callers (reference:
kornia/geometry/transform/imgwarp.py:397-527,529-622, kornia/geometry/conversions.py:117-148,
1640-1688).  Nine numbers per sample: kept as the reference's torch op sequence so the matrices
handed to the CUDA warp are the ones the reference would build on the same device, and autograd
reaches angles / centres / corner points."""
from __future__ import annotations

import torch

from ...core.check import check, check_shape
from .._prelude import inverse3x3

_PI = torch.tensor(3.14159265358979323846)  # fp32 constant, as kornia.constants.pi


def deg2rad(tensor: torch.Tensor) -> torch.Tensor:
    if not isinstance(tensor, torch.Tensor):
        raise TypeError(f"Input type is not a torch.Tensor. Got {type(tensor)}")
    return tensor * _PI.to(tensor.device).type(tensor.dtype) / 180.0


def rad2deg(tensor: torch.Tensor) -> torch.Tensor:
    if not isinstance(tensor, torch.Tensor):
        raise TypeError(f"Input type is not a torch.Tensor. Got {type(tensor)}")
    return 180.0 * tensor / _PI.to(tensor.device).type(tensor.dtype)


def angle_to_rotation_matrix(angle: torch.Tensor) -> torch.Tensor:
    """(*,) degrees -> (*,2,2) [[cos, sin], [-sin, cos]]."""
    rad = deg2rad(angle)
    c, s = torch.cos(rad), torch.sin(rad)
    return torch.stack([c, s, -s, c], dim=-1).view(*angle.shape, 2, 2)


def _eye3(like: torch.Tensor) -> torch.Tensor:
    return torch.eye(3, device=like.device, dtype=like.dtype)[None].repeat(like.shape[0], 1, 1)


def _fused_ok(*tensors: torch.Tensor) -> bool:
    """One-launch builders apply to CUDA fp32/fp64 inputs with batch >= 2 that need no gradient (torch's batched GEMM
    takes another path for a single sample; autograd keeps the torch op sequence)."""
    from .._prelude import FUSED_MIN_BATCH, torch_prelude_forced

    t0 = tensors[0]
    return (all(t.is_cuda for t in tensors) and t0.dtype in (torch.float32, torch.float64) and t0.shape[0] >= FUSED_MIN_BATCH
            and not (torch.is_grad_enabled() and any(t.requires_grad for t in tensors))
            and not torch_prelude_forced())


def _fused_rotation(center: torch.Tensor, angle: torch.Tensor, scale: torch.Tensor) -> torch.Tensor:
    from ... import _ops

    return _ops.ops.rotation_matrix2d(center, angle, scale)


def get_rotation_matrix2d(center: torch.Tensor, angle: torch.Tensor, scale: torch.Tensor) -> torch.Tensor:
    """(B,2,3) rotation by ``angle`` degrees (counter-clockwise on screen) and per-axis ``scale``
    about ``center`` (x, y): T(c) @ R @ S @ T(-c)."""
    for name, t in (("center", center), ("angle", angle), ("scale", scale)):
        if not isinstance(t, torch.Tensor):
            raise TypeError(f"Input {name} type is not a torch.Tensor. Got {type(t)}")
    if not (center.dim() == 2 and center.shape[1] == 2):
        raise ValueError(f"Input center must be a Bx2 torch.Tensor. Got {center.shape}")
    if angle.dim() != 1:
        raise ValueError(f"Input angle must be a B torch.Tensor. Got {angle.shape}")
    if not (scale.dim() == 2 and scale.shape[1] == 2):
        raise ValueError(f"Input scale must be a Bx2 torch.Tensor. Got {scale.shape}")
    if not (center.shape[0] == angle.shape[0] == scale.shape[0]):
        raise ValueError(f"Inputs must have same batch size dimension. Got center {center.shape}, angle {angle.shape} and scale "
                         f"{scale.shape}")
    if not (center.device == angle.device == scale.device) or not (center.dtype == angle.dtype == scale.dtype):
        raise ValueError(f"Inputs must have same device Got center ({center.device}, {center.dtype}), angle ({angle.device}, "
                         f"{angle.dtype}) and scale ({scale.device}, {scale.dtype})")
    if _fused_ok(center, angle, scale):
        return _fused_rotation(center, angle, scale)
    to_center, from_center, scaling, rotation = _eye3(center), _eye3(center), _eye3(center), _eye3(center)
    to_center[:, :2, 2] = center
    from_center[:, :2, 2] = -center
    scaling[:, 0, 0] *= scale[:, 0]
    scaling[:, 1, 1] *= scale[:, 1]
    rotation[:, :2, :2] = angle_to_rotation_matrix(angle)
    return (to_center @ rotation @ scaling @ from_center)[:, :2, :]


def _unit_square_to_quad(points: torch.Tensor) -> torch.Tensor:
    """(B,3,3) projective map taking (0,0),(1,0),(1,1),(0,1) onto the four ``points`` (B,4,2)
    (Heckbert's direct formulation, imgwarp.py:397-441)."""
    x0, y0 = points[..., 0, 0], points[..., 0, 1]
    x1, y1 = points[..., 1, 0], points[..., 1, 1]
    x2, y2 = points[..., 2, 0], points[..., 2, 1]
    x3, y3 = points[..., 3, 0], points[..., 3, 1]
    dx1, dx2, sx = x1 - x2, x3 - x2, x0 - x1 + x2 - x3
    dy1, dy2, sy = y1 - y2, y3 - y2, y0 - y1 + y2 - y3
    denom = dx1 * dy2 - dy1 * dx2
    g = (sx * dy2 - sy * dx2) / denom
    h = (dx1 * sy - dy1 * sx) / denom
    rows = [torch.stack([x1 - x0 + g * x1, x3 - x0 + h * x3, x0], dim=-1),
            torch.stack([y1 - y0 + g * y1, y3 - y0 + h * y3, y0], dim=-1),
            torch.stack([g, h, torch.ones_like(x0)], dim=-1)]
    return torch.stack(rows, dim=-2)


def _perspective_torch(points_src: torch.Tensor, points_dst: torch.Tensor) -> torch.Tensor:
    dtype = points_src.dtype
    work = dtype if dtype in (torch.float32, torch.float64) else torch.float32
    h = _unit_square_to_quad(points_dst.to(work)) @ inverse3x3(_unit_square_to_quad(points_src.to(work)))
    return (h / h[..., 2:3, 2:3]).to(dtype)


class _FusedPerspective(torch.autograd.Function):
    """kb200_perspective_from_points forward (one launch instead of ~45); the backward differentiates the
    torch op sequence on the saved corner points (18 numbers per sample)."""

    @staticmethod
    def forward(ctx, points_src, points_dst):
        from ... import _ops

        ctx.save_for_backward(points_src, points_dst)
        return _ops.ops.perspective_from_points(points_src, points_dst)

    @staticmethod
    def backward(ctx, gh):
        ps, pd = ctx.saved_tensors
        with torch.enable_grad():
            a = ps.detach().requires_grad_(ctx.needs_input_grad[0])
            b = pd.detach().requires_grad_(ctx.needs_input_grad[1])
            wrt = [t for t, need in zip((a, b), ctx.needs_input_grad) if need]
            grads = list(torch.autograd.grad(_perspective_torch(a, b), wrt, gh)) if wrt else []
        return tuple(grads.pop(0) if need else None for need in ctx.needs_input_grad)


def get_perspective_transform(points_src: torch.Tensor, points_dst: torch.Tensor) -> torch.Tensor:
    """(B,3,3) homography taking the four ``points_src`` (B,4,2; x,y) onto ``points_dst``, scaled so
    that H[2,2] = 1: H = Q(dst) @ Q(src)^-1 with Q the unit-square-to-quad map (imgwarp.py:444-527).
    CUDA fp32/fp64 points with batch >= 2 take one fused launch; anything else (CPU points, half
    precision, a single sample, the ``torch_prelude`` switch of kornia_b200.config) the reference's torch op sequence."""
    from .._prelude import FUSED_MIN_BATCH, torch_prelude_forced

    check_shape(points_src, ["B", "4", "2"])
    check_shape(points_dst, ["B", "4", "2"])
    check(points_src.shape == points_dst.shape, "Source data shape must match Destination data shape.")
    check(points_src.dtype == points_dst.dtype, "Source data type must match Destination data type.")
    fused_ok = (points_src.is_cuda and points_dst.is_cuda and points_src.dtype in (torch.float32, torch.float64)
                and points_src.shape[0] >= FUSED_MIN_BATCH and not torch_prelude_forced())
    if fused_ok:
        needs_grad = torch.is_grad_enabled() and (points_src.requires_grad or points_dst.requires_grad)
        if not needs_grad:
            from ... import _ops

            return _ops.ops.perspective_from_points(points_src, points_dst)
        if not torch.compiler.is_compiling():  # the backward re-differentiates the torch op sequence: eager only
            return _FusedPerspective.apply(points_src, points_dst)
    return _perspective_torch(points_src, points_dst)
