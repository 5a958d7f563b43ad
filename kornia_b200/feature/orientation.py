"""Drop-in ``PatchDominantGradientOrientation`` (reference: kornia/feature/orientation.py).

The reference estimates the dominant gradient angle of an (N, 1, P, P) patch stack with about 290 ATen kernels: the
Sobel gradient, elementwise passes, and per angular bin two one-hot masks, casts, products, an add and an
``adaptive_avg_pool2d``, then a circular ``nn.Conv1d`` smoothing, ``max`` and the parabolic sub-bin fit.

An fp32 CUDA call with patch_size <= 64, 2 <= num_angular_bins <= 64 and patches of column stride 1 that needs no
gradient runs as ONE CUDA kernel (csrc/patch_orientation.cuh) that reads each patch once and writes its angle.  "Needs
no gradient" means grad mode is off, or neither the input, ``weighting`` nor ``angular_smooth.weight`` requires grad.
``angular_smooth.weight`` is a trainable parameter, as in the reference, so a default-constructed module called in grad
mode runs the composition; ``torch.inference_mode()``, ``torch.no_grad()`` or ``orienter.requires_grad_(False)`` selects
the kernel.  The kernel reads the module's current ``weighting`` and ``angular_smooth.weight``.

Every other call runs ``_composed_orientation``: the reference's op sequence over this library's ``SpatialGradient``,
with the circular smoothing taken exactly (a circular pad, ``unfold`` and a product with ``angular_smooth.weight``, not a
convolution cuDNN may run in TF32), so the gradients are the reference's.  It is also the differentiable path."""
from __future__ import annotations

import torch
import torch.nn.functional as F
from torch import nn

from .. import _ops
from ..core.check import check_shape
from ..filters.kernels import get_gaussian_discrete_kernel1d, get_gaussian_kernel2d
from ..filters.sobel import SpatialGradient
from .siftdesc import MAX_PATCH_SIZE, pi

__all__ = ["PatchDominantGradientOrientation"]

MAX_ANGULAR_BINS = 64  # the fused kernel's envelope (csrc/patch_orientation.cuh)


class PatchDominantGradientOrientation(nn.Module):
    """Dominant gradient orientation of (B, 1, patch_size, patch_size) patches, in radians: (B,).  Zero points right.

    Args:
        patch_size: size of the (square) input patch.
        num_angular_bins: number of histogram bins.
        eps: for safe division, and arctan.

    An fp32 CUDA call that needs no gradient runs one fused kernel (see the module docstring); a default module in grad
    mode has a trainable ``angular_smooth.weight`` and runs the differentiable composition.
    """

    def __init__(self, patch_size: int = 32, num_angular_bins: int = 36, eps: float = 1e-8) -> None:
        super().__init__()
        self.patch_size = patch_size
        self.num_ang_bins = num_angular_bins
        self.gradient = SpatialGradient("sobel", 1)
        self.eps = eps
        self.angular_smooth = nn.Conv1d(1, 1, kernel_size=5, padding=2, bias=False, padding_mode="circular")
        with torch.no_grad():
            self.angular_smooth.weight[:] = get_gaussian_discrete_kernel1d(5, 1.6)
        sigma: float = float(self.patch_size) / 6.0
        self.weighting = get_gaussian_kernel2d((self.patch_size, self.patch_size), (sigma, sigma), True)

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}(patch_size={self.patch_size}, num_ang_bins={self.num_ang_bins}, eps={self.eps})"

    def _fused_ok(self, patch: torch.Tensor) -> bool:
        w = self.angular_smooth.weight
        needs_grad = torch.is_grad_enabled() and (patch.requires_grad or w.requires_grad or self.weighting.requires_grad)
        return (patch.dtype == torch.float32 and patch.is_cuda and not needs_grad and self.patch_size <= MAX_PATCH_SIZE
                and 2 <= self.num_ang_bins <= MAX_ANGULAR_BINS and (patch.shape[-1] == 1 or patch.stride(-1) == 1) and w.numel() == 5
                and self.weighting.numel() == self.patch_size**2)

    def forward(self, patch: torch.Tensor) -> torch.Tensor:
        check_shape(patch, ["B", "1", "H", "W"])
        _, CH, W, H = patch.size()
        if (W != self.patch_size) or (H != self.patch_size) or (CH != 1):
            raise TypeError(f"input shape should be must be [Bx1x{self.patch_size}x{self.patch_size}]. Got {patch.size()}")
        self.weighting = self.weighting.to(patch.dtype).to(patch.device)
        self.angular_smooth = self.angular_smooth.to(patch.dtype).to(patch.device)
        if self._fused_ok(patch):
            return _ops.ops.patch_orientation_fwd(patch, self.weighting, self.angular_smooth.weight, self.num_ang_bins, float(self.eps))
        return _composed_orientation(self, patch)


def _composed_orientation(m: PatchDominantGradientOrientation, patch: torch.Tensor) -> torch.Tensor:
    """orientation.py forward: the reference's op sequence, with the circular smoothing taken exactly."""
    n = m.num_ang_bins
    grads = m.gradient(patch)
    gx = grads[:, :, 0]
    gy = grads[:, :, 1]
    mag = torch.sqrt(gx * gx + gy * gy + m.eps) * m.weighting
    ori = torch.atan2(gy, gx + m.eps) + 2.0 * pi
    o_big = float(n) * (ori + 1.0 * pi) / (2.0 * pi)
    bo0_big = torch.floor(o_big)
    wo1_big = o_big - bo0_big
    bo0_big = bo0_big % n
    bo1_big = (bo0_big + 1) % n
    wo0_big = (1.0 - wo1_big) * mag
    wo1_big = wo1_big * mag
    ang_bins = torch.cat([F.adaptive_avg_pool2d((bo0_big == i).to(patch.dtype) * wo0_big + (bo1_big == i).to(patch.dtype) * wo1_big, (1, 1))
                          for i in range(n)], 1).view(-1, 1, n)
    windows = F.pad(ang_bins, (2, 2), mode="circular").unfold(-1, 5, 1)  # (B, 1, n, 5)
    ang_bins = (windows * m.angular_smooth.weight.reshape(5)).sum(-1).view(-1, n)
    values, indices = ang_bins.max(1)
    indices_left = (n + indices - 1) % n
    indices_right = (indices + 1) % n
    left = torch.gather(ang_bins, 1, indices_left.reshape(-1, 1)).reshape(-1)
    center = values
    right = torch.gather(ang_bins, 1, indices_right.reshape(-1, 1)).reshape(-1)
    c_subpix = 0.5 * (left - right) / (left + right - 2.0 * center)
    return -((2.0 * pi * (indices.to(patch.dtype) + c_subpix) / float(n)) - pi)
