"""Drop-in ``PatchAffineShapeEstimator`` and ``LAFAffineShapeEstimator`` (reference: kornia/feature/affine_shape.py): the
Baumberg second-moment affine adaptation of Hessian-Affine / Harris-Affine detectors.

The reference's ``LAFAffineShapeEstimator`` runs about 90 small ATen launches per call around the patch extraction:
``make_upright``, an N x 1 x PS x PS patch stack, the Sobel gradient, weighting, products and means of
``PatchAffineShapeEstimator``, a batched ``torch.inverse`` of N 2 x 2 matrices in ``ellipse_to_laf``, the rescale and the
orientation restore.

An fp32 CUDA call that needs no gradient -- grad mode off, or no input (patch / img / laf) and no ``weighting`` requires
grad -- runs ONE CUDA kernel (csrc/affine_shape.cuh): ``PatchAffineShapeEstimator`` on the patch stack it is given, and
``LAFAffineShapeEstimator`` (after this library's ``pyrdown`` of the pyramid levels the extraction samples, a number that
depends on the shapes only) from the LAFs and the levels, never writing the patch stack.  ``LAFAffineShapeEstimator``
takes the kernel only when its ``affine_shape_detector`` is exactly this library's ``PatchAffineShapeEstimator`` of its
own ``patch_size``, PS <= 64, and the image (one channel) and LAFs are on one device.  Both kernels read the estimator's
current ``weighting`` and ``eps``.

Every other call runs ``_composed_patch_affine_shape`` / ``_composed_laf_affine_shape``: the reference's op sequence over
this library's ``SpatialGradient``, ``extract_patches_from_pyramid`` and LAF helpers.  It is the differentiable path, runs
a custom or AffNet ``affine_shape_detector``, and takes the calls for which the reference raises, so its errors come back."""
from __future__ import annotations

import math
from typing import Optional

import torch
from torch import nn

from .. import _ops
from ..core.check import check_shape
from ..filters.kernels import get_gaussian_kernel2d
from ..filters.sobel import SpatialGradient
from ..geometry.transform.pyramid import pyrdown
from .laf import (_built_levels, _check_laf, ellipse_to_laf, extract_patches_from_pyramid, get_laf_orientation, get_laf_scale, make_upright,
                  scale_laf, set_laf_orientation)
from .siftdesc import MAX_PATCH_SIZE

__all__ = ["PatchAffineShapeEstimator", "LAFAffineShapeEstimator"]


class PatchAffineShapeEstimator(nn.Module):
    """Second moment matrix of the Gaussian-weighted patch gradients, as the affine shape (a, b, c) / max(a, b, c) of
    (B, 1, patch_size, patch_size) patches: (B, 1, 3).  A degenerate shape (at least two moments below ``eps``) becomes the
    circle (1, 0, 1).

    Args:
        patch_size: the input image patch size.
        eps: for safe division.
    """

    def __init__(self, patch_size: int = 19, eps: float = 1e-10) -> None:
        super().__init__()
        self.patch_size: int = patch_size
        self.gradient: nn.Module = SpatialGradient("sobel", 1)
        self.eps: float = eps
        sigma: float = float(self.patch_size) / math.sqrt(2.0)
        self.weighting: torch.Tensor = get_gaussian_kernel2d((self.patch_size, self.patch_size), (sigma, sigma), True)

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}(patch_size={self.patch_size}, eps={self.eps})"

    def _fused_ok(self, patch: torch.Tensor) -> bool:
        P = self.patch_size
        needs_grad = torch.is_grad_enabled() and (patch.requires_grad or self.weighting.requires_grad)
        return (patch.dtype == torch.float32 and patch.is_cuda and not needs_grad and 1 <= P <= MAX_PATCH_SIZE
                and tuple(patch.shape[-2:]) == (P, P) and self.weighting.numel() == P * P)

    def forward(self, patch: torch.Tensor) -> torch.Tensor:
        check_shape(patch, ["B", "1", "H", "W"])
        self.weighting = self.weighting.to(patch.dtype).to(patch.device)
        if self._fused_ok(patch):
            return _ops.ops.patch_affine_shape_fwd(patch, self.weighting, float(self.eps))
        return _composed_patch_affine_shape(self, patch)


class LAFAffineShapeEstimator(nn.Module):
    """Replace the shape of LAFs (B, N, 2, 3) by the affine shape ``affine_shape_detector`` estimates on their patches of
    ``img`` (B, 1, H, W), keeping their scale and (with ``preserve_orientation``) their orientation.

    Args:
        patch_size: the input image patch size.
        affine_shape_detector: patch affine shape estimator, by default ``PatchAffineShapeEstimator(patch_size)``.
        preserve_orientation: if True, the original orientation is preserved.
    """

    def __init__(self, patch_size: int = 32, affine_shape_detector: Optional[nn.Module] = None, preserve_orientation: bool = True) -> None:
        super().__init__()
        self.patch_size = patch_size
        self.affine_shape_detector = affine_shape_detector or PatchAffineShapeEstimator(self.patch_size)
        self.preserve_orientation = preserve_orientation

    def __repr__(self) -> str:
        return (f"{self.__class__.__name__}"
                f"(patch_size={self.patch_size}, "
                f"affine_shape_detector={self.affine_shape_detector}, "
                f"preserve_orientation={self.preserve_orientation})")

    def _fused_ok(self, laf: torch.Tensor, img: torch.Tensor) -> bool:
        det, PS = self.affine_shape_detector, self.patch_size
        if type(det) is not PatchAffineShapeEstimator or det.patch_size != PS:
            return False
        w = det.weighting
        needs_grad = torch.is_grad_enabled() and (img.requires_grad or laf.requires_grad or w.requires_grad)
        return (img.is_cuda and laf.device == img.device and img.dtype == torch.float32 and laf.dtype == torch.float32 and not needs_grad
                and 1 <= PS <= MAX_PATCH_SIZE and w.numel() == PS * PS and laf.shape[0] > 0 and laf.shape[1] > 0
                and img.shape[0] >= laf.shape[0] and min(img.shape[-2:]) >= 2)

    def forward(self, laf: torch.Tensor, img: torch.Tensor) -> torch.Tensor:
        _check_laf(laf)
        check_shape(img, ["B", "1", "H", "W"])
        if self._fused_ok(laf, img):
            det, PS = self.affine_shape_detector, self.patch_size
            det.weighting = det.weighting.to(img.dtype).to(img.device)
            levels = [img]
            for _ in range(_built_levels(img.shape[-2], img.shape[-1], PS) - 1):
                levels.append(pyrdown(levels[-1]))
            return _ops.ops.laf_affine_shape_fwd(levels, laf, det.weighting, int(PS), float(det.eps), bool(self.preserve_orientation))
        return _composed_laf_affine_shape(self, laf, img)


def _composed_patch_affine_shape(m: PatchAffineShapeEstimator, patch: torch.Tensor) -> torch.Tensor:
    """affine_shape.py PatchAffineShapeEstimator.forward: the reference's op sequence."""
    grads = m.gradient(patch) * m.weighting
    gx = grads[:, :, 0]
    gy = grads[:, :, 1]
    ellipse_shape = torch.cat([gx.pow(2).mean(dim=2).mean(dim=2, keepdim=True),
                               (gx * gy).mean(dim=2).mean(dim=2, keepdim=True),
                               gy.pow(2).mean(dim=2).mean(dim=2, keepdim=True)], dim=2)
    bad_mask = ((ellipse_shape < m.eps).float().sum(dim=2, keepdim=True) >= 2).to(ellipse_shape.dtype)
    circular_shape = torch.tensor([1.0, 0.0, 1.0]).to(ellipse_shape.device).to(ellipse_shape.dtype).view(1, 1, 3)
    ellipse_shape = ellipse_shape * (1.0 - bad_mask) + circular_shape * bad_mask
    return ellipse_shape / ellipse_shape.max(dim=2, keepdim=True)[0]


def _composed_laf_affine_shape(m: LAFAffineShapeEstimator, laf: torch.Tensor, img: torch.Tensor) -> torch.Tensor:
    """affine_shape.py LAFAffineShapeEstimator.forward: the reference's op sequence."""
    _check_laf(laf)
    check_shape(img, ["B", "1", "H", "W"])
    B, N = laf.shape[:2]
    PS: int = m.patch_size
    patches = extract_patches_from_pyramid(img, make_upright(laf), PS, True).view(-1, 1, PS, PS)
    ellipse_shape = m.affine_shape_detector(patches)
    ellipses = torch.cat([laf.view(-1, 2, 3)[..., 2].unsqueeze(1), ellipse_shape], dim=2).view(B, N, 5)
    scale_orig = get_laf_scale(laf)
    if m.preserve_orientation:
        ori_orig = get_laf_orientation(laf)
    laf_out = ellipse_to_laf(ellipses)
    ellipse_scale = get_laf_scale(laf_out)
    laf_out = scale_laf(laf_out, scale_orig / ellipse_scale)
    if m.preserve_orientation:
        laf_out = set_laf_orientation(laf_out, ori_orig)
    return laf_out
