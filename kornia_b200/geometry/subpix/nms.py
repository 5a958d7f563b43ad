"""Drop-in ``nms2d``, ``nms3d``, ``nms3d_minmax``, ``NonMaximaSuppression2d`` and ``NonMaximaSuppression3d`` (reference:
kornia/geometry/subpix/nms.py).

The reference suppresses with one ATen kernel per neighbour comparison and per ``&`` (3 x 3, 5 x 5, 7 x 7 and the 3-D
(3, 3, 3) form), or with a one-hot ``F.conv2d`` that writes K*K neighbour planes before a ``max`` (every other 2-D
size).  Every form keeps a position when ``x > M``, M the NaN-propagating maximum of a neighbour set:

* 2-D K = 3, 5, 7: the K*K - 1 neighbours; the outer (K - 1) / 2 ring is False.
* 2-D other square odd K: the K*K - 1 neighbours of the replicate-padded image and 0 (the convolution's all-zero centre
  channel); a window, centre included, that holds a non-finite texel is False (0 * Inf and 0 * NaN make every channel
  NaN).  Even and non-square sizes raise the reference's ``RuntimeError``.
* 3-D (3, 3, 3) and ``nms3d_minmax``: the 26 neighbours (``x < min`` for the minima); border levels, rows and columns
  are False.  Other 3-D sizes raise the reference's ``RuntimeError``.

With ``mask_only=False`` the result is ``x * mask.to(x.dtype)``.  fp32 CUDA calls of the sizes above (K = 3 .. 31 in
2-D) that need no gradient, or ask only for the mask, run as ONE CUDA kernel (csrc/nms.cuh), bit-identical to
``_composed_*``: the reference's op sequence and shapes, with the general 2-D form's neighbour planes taken exactly by
``F.unfold`` instead of a convolution (which cuDNN may compute in TF32).  ``_composed_*`` is what every other call runs
and is also the differentiable path: the gradient of ``x * mask`` is ``g * mask``."""
from __future__ import annotations

import torch
import torch.nn.functional as F
from torch import nn

from ... import _ops

__all__ = ["nms2d", "nms3d", "nms3d_minmax", "NonMaximaSuppression2d", "NonMaximaSuppression3d"]

_FUSED_2D_SIZES = frozenset(range(3, 32, 2))  # csrc/nms.cu instantiations


def _get_nms_kernel2d(kx: int, ky: int) -> torch.Tensor:
    """Return neigh2channels conv kernel."""
    numel: int = ky * kx
    center: int = numel // 2
    weight = torch.eye(numel)
    weight[center, center] = 0
    return weight.view(numel, 1, ky, kx)


def _get_nms_kernel3d(kd: int, ky: int, kx: int) -> torch.Tensor:
    """Return neigh2channels conv kernel."""
    numel: int = kd * ky * kx
    center: int = numel // 2
    weight = torch.eye(numel)
    weight[center, center] = 0
    return weight.view(numel, 1, kd, ky, kx)


def _kernel_runs(x: torch.Tensor, mask_only: bool) -> bool:
    return x.dtype == torch.float32 and x.is_cuda and x.numel() > 0 and (mask_only or not (torch.is_grad_enabled() and x.requires_grad))


def _fused_nms2d(x: torch.Tensor, kernel_size, mask_only: bool):
    """The 2-D kernel's result, or None when the call takes the composition."""
    ky, kx = kernel_size
    if type(ky) is not int or ky != kx or ky not in _FUSED_2D_SIZES or not _kernel_runs(x, mask_only):
        return None
    return _ops.ops.nms2d_fwd(x.detach() if mask_only else x, ky, mask_only)


def _fused_nms3d(x: torch.Tensor, kernel_size, mask_only: bool):
    """The 3-D kernel's result, or None when the call takes the composition."""
    if tuple(kernel_size) != (3, 3, 3) or any(type(k) is not int for k in kernel_size) or not _kernel_runs(x, mask_only):
        return None
    return _ops.ops.nms3d_fwd(x.detach() if mask_only else x, mask_only)


def _strict_extremum(x: torch.Tensor, r: int, greater: bool) -> torch.Tensor:
    """The reference's explicit comparisons: ``x[..., r:-r, r:-r]`` against each of its (2r + 1)^2 - 1 neighbours in the
    last two dimensions (and, for a 5-D ``x`` with r = 1, in the level dimension), AND-reduced."""
    def sl(d):
        return slice(d, d - 2 * r if d < 2 * r else None)

    ct = x[..., sl(r), sl(r)] if x.dim() == 4 else x[..., sl(1), sl(1), sl(1)]
    offsets = [(dy, dx) for dy in range(2 * r + 1) for dx in range(2 * r + 1)]
    if x.dim() == 5:
        offsets = [(dz, dy, dx) for dz in range(3) for dy in range(3) for dx in range(3)]
    mask = None
    for off in offsets:
        if all(o == r for o in off):
            continue
        nb = x[(...,) + tuple(sl(o) for o in off)]
        m = ct > nb if greater else ct < nb
        mask = m if mask is None else mask & m
    return mask


def _composed_nms2d(x: torch.Tensor, kernel_size, padding, kernel: torch.Tensor, mask_only: bool) -> torch.Tensor:
    """NonMaximaSuppression2d.forward as the reference computes it (nms.py, forward of the 2-D module)."""
    B, CH, H, W = x.size()
    if kernel_size in ((3, 3), (5, 5), (7, 7)):
        r = kernel_size[0] // 2
        mask = torch.zeros(B, CH, H, W, device=x.device, dtype=torch.bool)
        mask[..., r:-r, r:-r] = _strict_extremum(x, r, True)
    else:
        x_padded = F.pad(x, list(padding)[::-1], mode="replicate")
        B, CH, HP, WP = x_padded.size()
        # the reference's one-hot F.conv2d with its (numel, 1, ky, kx) weight, as exact neighbour planes: channel j is
        # window texel j, the centre channel is 0, and a window holding a non-finite texel is NaN in every channel
        numel, kh, kw = kernel.shape[0], kernel.shape[-2], kernel.shape[-1]
        cols = F.unfold(x_padded.view(B * CH, 1, HP, WP), (kh, kw))
        bad = ~torch.isfinite(cols).all(dim=1, keepdim=True)
        nan = torch.full((), float("nan"), device=x.device, dtype=x.dtype)
        cols = torch.where(bad, nan, cols)
        cols[:, numel // 2] = torch.where(bad[:, 0], nan, torch.zeros((), device=x.device, dtype=x.dtype))
        neighborhood = cols.view(B, CH, -1, H, W)
        max_non_center = neighborhood.max(dim=2)[0]
        mask = x > max_non_center
    if mask_only:
        return mask
    return x * (mask.to(x.dtype))


def _composed_nms3d(x: torch.Tensor, kernel_size, padding, kernel: torch.Tensor, mask_only: bool) -> torch.Tensor:
    """NonMaximaSuppression3d.forward as the reference computes it (nms.py, forward of the 3-D module)."""
    B, CH, D, H, W = x.size()
    if kernel_size == (3, 3, 3):
        mask = torch.zeros(B, CH, D, H, W, device=x.device, dtype=torch.bool)
        mask[..., 1:-1, 1:-1, 1:-1] = _strict_extremum(x, 1, True)
    else:  # the reference pads by k rather than (k - 1) / 2: the view raises for every shape but degenerate ones
        max_non_center = (
            F.conv3d(F.pad(x, list(padding)[::-1], mode="replicate"), kernel.repeat(CH, 1, 1, 1, 1).to(x.device, x.dtype), stride=1, groups=CH)
            .view(B, CH, -1, D, H, W)
            .max(dim=2, keepdim=False)[0]
        )
        mask = x > max_non_center
    if mask_only:
        return mask
    return x * (mask.to(x.dtype))


def _composed_nms3d_minmax(input: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """nms3d_minmax as the reference computes it: the 26 strict comparisons each way on the interior."""
    B, CH, D, H, W = input.shape
    max_mask = torch.zeros(B, CH, D, H, W, device=input.device, dtype=torch.bool)
    min_mask = torch.zeros(B, CH, D, H, W, device=input.device, dtype=torch.bool)
    max_mask[..., 1:-1, 1:-1, 1:-1] = _strict_extremum(input, 1, True)
    min_mask[..., 1:-1, 1:-1, 1:-1] = _strict_extremum(input, 1, False)
    return max_mask, min_mask


class NonMaximaSuppression2d(nn.Module):
    r"""Apply non maxima suppression to filter.

    Flag `minima_are_also_good` is useful, when you want to detect both maxima and minima, e.g. for DoG
    """

    kernel: torch.Tensor

    def __init__(self, kernel_size: tuple[int, int]) -> None:
        super().__init__()
        self.kernel_size: tuple[int, int] = kernel_size
        self.padding: tuple[int, int, int, int] = self._compute_zero_padding2d(kernel_size)
        self.register_buffer("kernel", _get_nms_kernel2d(*kernel_size))

    @staticmethod
    def _compute_zero_padding2d(kernel_size: tuple[int, int]) -> tuple[int, int, int, int]:
        if not isinstance(kernel_size, tuple):
            raise AssertionError(type(kernel_size))
        if len(kernel_size) != 2:
            raise AssertionError(kernel_size)

        def pad(x: int) -> int:
            return (x - 1) // 2

        ky, kx = kernel_size
        return (pad(ky), pad(kx), pad(ky), pad(kx))

    def forward(self, x: torch.Tensor, mask_only: bool = False) -> torch.Tensor:
        """Keep only strict local maxima of the (B, C, H, W) response ``x`` within ``kernel_size``: the boolean mask when
        ``mask_only``, else ``x`` with the suppressed positions multiplied by 0."""
        if len(x.shape) != 4:
            raise AssertionError(x.shape)
        out = _fused_nms2d(x, self.kernel_size, mask_only)
        if out is not None:
            return out
        return _composed_nms2d(x, self.kernel_size, self.padding, self.kernel, mask_only)


class NonMaximaSuppression3d(nn.Module):
    r"""Apply non maxima suppression to filter."""

    def __init__(self, kernel_size: tuple[int, int, int]) -> None:
        super().__init__()
        self.kernel_size: tuple[int, int, int] = kernel_size
        self.padding: tuple[int, int, int, int, int, int] = self._compute_zero_padding3d(kernel_size)
        self.kernel = _get_nms_kernel3d(*kernel_size)

    @staticmethod
    def _compute_zero_padding3d(kernel_size: tuple[int, int, int]) -> tuple[int, int, int, int, int, int]:
        if not isinstance(kernel_size, tuple):
            raise AssertionError(type(kernel_size))
        if len(kernel_size) != 3:
            raise AssertionError(kernel_size)

        kd, ky, kx = kernel_size
        return (kd, kd, ky, ky, kx, kx)

    def forward(self, x: torch.Tensor, mask_only: bool = False) -> torch.Tensor:
        """Keep only strict local maxima of the (B, C, D, H, W) response ``x`` across depth, height and width: the boolean
        mask when ``mask_only``, else ``x`` with the suppressed positions multiplied by 0."""
        if len(x.shape) != 5:
            raise AssertionError(x.shape)
        out = _fused_nms3d(x, self.kernel_size, mask_only)
        if out is not None:
            return out
        return _composed_nms3d(x, self.kernel_size, self.padding, self.kernel, mask_only)


# functional api


def nms2d(input: torch.Tensor, kernel_size: tuple[int, int], mask_only: bool = False) -> torch.Tensor:
    r"""Apply non maxima suppression to filter.

    See :class:`~kornia_b200.geometry.subpix.NonMaximaSuppression2d` for details.
    """
    NonMaximaSuppression2d._compute_zero_padding2d(kernel_size)  # the constructor's checks, before the input's
    if len(input.shape) == 4:
        out = _fused_nms2d(input, kernel_size, mask_only)
        if out is not None:
            return out
    return NonMaximaSuppression2d(kernel_size)(input, mask_only)


def nms3d(input: torch.Tensor, kernel_size: tuple[int, int, int], mask_only: bool = False) -> torch.Tensor:
    r"""Apply non maxima suppression to filter.

    See :class:`~kornia_b200.geometry.subpix.NonMaximaSuppression3d` for details.
    """
    NonMaximaSuppression3d._compute_zero_padding3d(kernel_size)
    if len(input.shape) == 5:
        out = _fused_nms3d(input, kernel_size, mask_only)
        if out is not None:
            return out
    return NonMaximaSuppression3d(kernel_size)(input, mask_only)


def nms3d_minmax(input: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    r"""Local-maxima and local-minima masks of a (B, C, D, H, W) scale-space tensor in one pass: ``(max_mask, min_mask)``,
    each True where the voxel is strictly greater (smaller) than all 26 neighbours; the same as
    ``nms3d(input, (3, 3, 3), mask_only=True)`` and ``nms3d(-input, (3, 3, 3), mask_only=True)``."""
    if input.dim() != 5:
        raise AssertionError(input.shape)
    if _kernel_runs(input, True):
        return _ops.ops.nms3d_minmax_fwd(input.detach())
    return _composed_nms3d_minmax(input)
