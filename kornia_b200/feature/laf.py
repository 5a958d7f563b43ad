"""Drop-in ``extract_patches_from_pyramid`` and ``extract_patches_simple``, with the helpers their composition needs:
``get_laf_scale``, ``normalize_laf``, ``denormalize_laf`` and ``generate_patch_grid_from_normalized_LAF``, and the LAF helpers
of the affine shape estimators (feature/affine_shape.py): ``make_upright``, ``scale_laf``, ``ellipse_to_laf``,
``get_laf_orientation``, ``set_laf_orientation`` and ``rotate_laf``, each the reference's op sequence (reference:
kornia/feature/laf.py).

The reference cuts patches out of a pyramid by looping over every level the image allows and, inside that, over every
image of the batch: each (level, image) pair builds an affine grid for ALL N keypoints, samples all of them with
``grid_sample`` and keeps, with ``torch.where``, only the patches whose scale picked that level -- about 25 ATen kernels
per (level, image), and every patch sampled 5-6 times at 1080p.

An fp32 CUDA call (image and LAFs on one device) that needs no gradient -- grad mode off, or neither ``img`` nor ``laf``
requires grad -- runs this library's ``pyrdown`` for the levels that are sampled and then ONE CUDA kernel
(csrc/laf_patches.cuh) that picks each patch's level, maps its grid and samples every channel, writing each output element
once.  The number of levels the reference samples depends only on the shapes, so it is computed on the host without a
device sync; a patch whose level is not among them stays zero, as in the reference.

Every other call runs ``_composed_extract_pyramid`` / ``_composed_extract_simple``: the reference's op sequence over
``F.affine_grid``, ``F.grid_sample`` and this library's ``pyrdown``, which is also the differentiable path."""
from __future__ import annotations

from typing import Union

import torch
import torch.nn.functional as F

from .. import _ops
from ..core.check import check_shape
from ..geometry.transform.matrices import angle_to_rotation_matrix, rad2deg
from ..geometry.transform.pyramid import pyrdown

__all__ = ["extract_patches_from_pyramid", "extract_patches_simple", "get_laf_scale", "normalize_laf", "denormalize_laf",
           "generate_patch_grid_from_normalized_LAF", "get_laf_orientation", "rotate_laf", "set_laf_orientation", "scale_laf", "make_upright",
           "ellipse_to_laf"]

def _check_laf(laf: torch.Tensor) -> None:
    """KORNIA_CHECK_LAF: a (B, N, 2, 3) tensor."""
    check_shape(laf, ["B", "N", "2", "3"])


def get_laf_scale(LAF: torch.Tensor) -> torch.Tensor:
    """(B, N, 1, 1) scale sqrt(|a d - c b + 1e-10|) of the LAFs' linear part [[a, b], [c, d]]."""
    _check_laf(LAF)
    eps = 1e-10
    out = LAF[..., 0:1, 0:1] * LAF[..., 1:2, 1:2] - LAF[..., 1:2, 0:1] * LAF[..., 0:1, 1:2] + eps
    return out.abs().sqrt()


def get_laf_orientation(LAF: torch.Tensor) -> torch.Tensor:
    """(B, N, 1) orientation of the LAFs in degrees: rad2deg(atan2(LAF[..., 0, 1], LAF[..., 0, 0]))."""
    _check_laf(LAF)
    angle_rad = torch.atan2(LAF[..., 0, 1], LAF[..., 0, 0])
    return rad2deg(angle_rad).unsqueeze(-1)


def rotate_laf(LAF: torch.Tensor, angles_degrees: torch.Tensor) -> torch.Tensor:
    """The LAFs with their linear part multiplied on the right by the rotation of ``angles_degrees`` (B, N, 1)."""
    _check_laf(LAF)
    B, N = LAF.shape[:2]
    rotmat = angle_to_rotation_matrix(angles_degrees).view(B * N, 2, 2)
    out_laf = LAF.clone()
    out_laf[:, :, :2, :2] = torch.bmm(LAF[:, :, :2, :2].reshape(B * N, 2, 2), rotmat).reshape(B, N, 2, 2)
    return out_laf


def set_laf_orientation(LAF: torch.Tensor, angles_degrees: torch.Tensor) -> torch.Tensor:
    """The LAFs rotated so that their orientation becomes ``angles_degrees`` (B, N, 1)."""
    _check_laf(LAF)
    ori = get_laf_orientation(LAF).reshape_as(angles_degrees)
    return rotate_laf(LAF, angles_degrees - ori)


def scale_laf(laf: torch.Tensor, scale_coef: Union[float, torch.Tensor]) -> torch.Tensor:
    """The LAFs with their linear part multiplied by ``scale_coef`` (a float or a broadcastable tensor); centres kept."""
    if not isinstance(scale_coef, (float, torch.Tensor)):
        raise TypeError(f"scale_coef should be float or torch.Tensor. Got {type(scale_coef)}")
    _check_laf(laf)
    centerless_laf = laf[:, :, :2, :2]
    return torch.cat([scale_coef * centerless_laf, laf[:, :, :, 2:]], dim=3)


def make_upright(laf: torch.Tensor, eps: float = 1e-9) -> torch.Tensor:
    """The LAFs with their rotation removed (the U * S of a 2 x 2 SVD U S V^T), scale and centre kept."""
    _check_laf(laf)
    det = get_laf_scale(laf)
    scale = det
    b2a2 = torch.sqrt(laf[..., 0:1, 1:2] ** 2 + laf[..., 0:1, 0:1] ** 2) + eps
    laf1_ell = torch.cat([(b2a2 / det).contiguous(), torch.zeros_like(det)], dim=3)
    laf2_ell = torch.cat([((laf[..., 1:2, 1:2] * laf[..., 0:1, 1:2] + laf[..., 1:2, 0:1] * laf[..., 0:1, 0:1]) / (b2a2 * det)),
                          (det / b2a2).contiguous()], dim=3)
    laf_unit_scale = torch.cat([torch.cat([laf1_ell, laf2_ell], dim=2), laf[..., :, 2:3]], dim=3)
    return scale_laf(laf_unit_scale, scale)


def ellipse_to_laf(ells: torch.Tensor) -> torch.Tensor:
    """(B, N, 2, 3) LAFs of (B, N, 5) ellipses [x, y, a, b, c]: the inverse of the lower-triangular square root
    [[sqrt|a|, 0], [b / (sqrt|a| + sqrt|c|), sqrt|c|]] of [[a, b], [b, c]], centred at (x, y)."""
    check_shape(ells, ["B", "N", "5"])
    B, N, _ = ells.shape
    a11 = ells[..., 2:3].abs().sqrt()
    a12 = torch.zeros_like(a11)
    a22 = ells[..., 4:5].abs().sqrt()
    a21 = ells[..., 3:4] / (a11 + a22).clamp(1e-9)
    A = torch.stack([a11, a12, a21, a22], dim=-1).view(B, N, 2, 2).inverse()
    return torch.cat([A, ells[..., :2].view(B, N, 2, 1)], dim=3)


def denormalize_laf(LAF: torch.Tensor, images: torch.Tensor) -> torch.Tensor:
    """LAFs from the [0, 1] scale to pixels of ``images``: linear part times min(H - 1, W - 1), centre times (W - 1, H - 1)."""
    _check_laf(LAF)
    _, _, h, w = images.size()
    wf = float(w - 1)
    hf = float(h - 1)
    min_size = min(hf, wf)
    coef = torch.ones(1, 1, 2, 3, dtype=LAF.dtype, device=LAF.device) * min_size
    coef[0, 0, 0, 2] = wf
    coef[0, 0, 1, 2] = hf
    return coef.expand_as(LAF) * LAF


def normalize_laf(LAF: torch.Tensor, images: torch.Tensor) -> torch.Tensor:
    """LAFs from pixels of ``images`` to the [0, 1] scale: the inverse coefficients of :func:`denormalize_laf`."""
    _check_laf(LAF)
    _, _, h, w = images.size()
    wf = float(w - 1)
    hf = float(h - 1)
    min_size = min(hf, wf)
    coef = torch.ones(1, 1, 2, 3, dtype=LAF.dtype, device=LAF.device) / min_size
    coef[0, 0, 0, 2] = 1.0 / wf
    coef[0, 0, 1, 2] = 1.0 / hf
    return coef.expand_as(LAF) * LAF


def generate_patch_grid_from_normalized_LAF(img: torch.Tensor, LAF: torch.Tensor, PS: int = 32) -> torch.Tensor:
    """(B * N, PS, PS, 2) ``grid_sample`` grid of the normalised LAFs on ``img``."""
    _check_laf(LAF)
    B, N, _, _ = LAF.size()
    _, ch, h, w = img.size()
    LAF_renorm = denormalize_laf(LAF, img)
    grid = F.affine_grid(LAF_renorm.view(B * N, 2, 3), [B * N, ch, PS, PS], align_corners=False)
    grid[..., :, 0] = 2.0 * grid[..., :, 0].clone() / float(w - 1) - 1.0
    grid[..., :, 1] = 2.0 * grid[..., :, 1].clone() / float(h - 1) - 1.0
    return grid


def _built_levels(h: int, w: int, PS: int) -> int:
    """How many pyramid levels the reference samples: max(1, min(h, w) // PS), cut at the first level (after level 0) whose
    shorter side is below PS -- that level is built but never sampled.  Depends on the shapes only (level l is h // 2^l)."""
    n = 1
    for _ in range(max(1, min(h, w) // PS) - 1):
        h, w = h // 2, w // 2
        if min(h, w) < PS:
            break
        n += 1
    return n


def _fused_ok(img: torch.Tensor, laf: torch.Tensor, PS: int, normalize: bool) -> bool:
    """fp32 image and LAFs on one CUDA device, no gradient needed.  The calls for which the reference raises -- no LAFs, an
    image batch smaller than the LAF batch, a one-pixel side to normalise by, PS < 1 -- run the composition, which raises
    the reference's own errors (affine_grid's, ``expand``'s, Python's division)."""
    needs_grad = torch.is_grad_enabled() and (img.requires_grad or laf.requires_grad)
    return (img.is_cuda and laf.device == img.device and img.dtype == torch.float32 and laf.dtype == torch.float32 and not needs_grad
            and img.dim() == 4 and img.shape[1] > 0 and laf.shape[0] > 0 and laf.shape[1] > 0 and img.shape[0] >= laf.shape[0]
            and PS >= 1 and not (normalize and min(img.shape[-2:]) < 2))


def extract_patches_simple(img: torch.Tensor, laf: torch.Tensor, PS: int = 32, normalize_lafs_before_extraction: bool = True) -> torch.Tensor:
    """(B, N, CH, PS, PS) patches of ``img`` (B, CH, H, W) at the LAFs ``laf`` (B, N, 2, 3), sampled from the image itself
    (no smoothing: aliases; prefer :func:`extract_patches_from_pyramid`).  Returns ``img.dtype``."""
    _check_laf(laf)
    if _fused_ok(img, laf, PS, normalize_lafs_before_extraction):
        return _ops.ops.extract_patches_fwd([img], laf, int(PS), bool(normalize_lafs_before_extraction), False)
    return _composed_extract_simple(img, laf, PS, normalize_lafs_before_extraction)


def extract_patches_from_pyramid(img: torch.Tensor, laf: torch.Tensor, PS: int = 32,
                                 normalize_lafs_before_extraction: bool = True) -> torch.Tensor:
    """(B, N, CH, PS, PS) patches of ``img`` (B, CH, H, W) at the LAFs ``laf`` (B, N, 2, 3), each sampled from the pyramid
    level its scale picks.  Returns ``laf.dtype``."""
    _check_laf(laf)
    if _fused_ok(img, laf, PS, normalize_lafs_before_extraction):
        _, _, h, w = img.shape
        levels = [img]
        for _ in range(_built_levels(h, w, PS) - 1):
            levels.append(pyrdown(levels[-1]))
        return _ops.ops.extract_patches_fwd(levels, laf, int(PS), bool(normalize_lafs_before_extraction), True)
    return _composed_extract_pyramid(img, laf, PS, normalize_lafs_before_extraction)


def _composed_extract_simple(img: torch.Tensor, laf: torch.Tensor, PS: int, normalize_lafs_before_extraction: bool) -> torch.Tensor:
    """laf.py extract_patches_simple: the reference's op sequence."""
    _check_laf(laf)
    nlaf = normalize_laf(laf, img) if normalize_lafs_before_extraction else laf
    _, ch, h, w = img.size()
    B, N, _, _ = laf.size()
    out = []
    for i in range(B):
        grid = generate_patch_grid_from_normalized_LAF(img[i:i + 1], nlaf[i:i + 1], PS).to(img.device)
        out.append(F.grid_sample(img[i:i + 1].expand(grid.size(0), ch, h, w), grid, padding_mode="border", align_corners=False))
    return torch.cat(out, dim=0).view(B, N, ch, PS, PS)


def _composed_extract_pyramid(img: torch.Tensor, laf: torch.Tensor, PS: int, normalize_lafs_before_extraction: bool) -> torch.Tensor:
    """laf.py extract_patches_from_pyramid: the reference's op sequence over this library's ``pyrdown``."""
    _check_laf(laf)
    nlaf = normalize_laf(laf, img) if normalize_lafs_before_extraction else laf
    B, N, _, _ = laf.size()
    _, ch, h, w = img.size()
    scale = 2.0 * get_laf_scale(denormalize_laf(nlaf, img)) / float(PS)
    max_level = min(h, w) // PS
    pyr_idx = scale.log2().clamp(min=0.0, max=max(0, max_level - 1)).long()
    out = torch.zeros(B, N, ch, PS, PS, dtype=nlaf.dtype, device=nlaf.device)
    cur_img = img
    num_levels = max(1, max_level)
    for cur_pyr_level in range(num_levels):
        _, ch_l, h_l, w_l = cur_img.size()
        for i in range(B):
            level_mask = (pyr_idx[i] == cur_pyr_level).view(N, 1, 1, 1)
            grid = generate_patch_grid_from_normalized_LAF(cur_img[i:i + 1], nlaf[i:i + 1], PS)
            patches = F.grid_sample(cur_img[i:i + 1].expand(N, ch_l, h_l, w_l), grid, padding_mode="border", align_corners=False)
            out[i] = torch.where(level_mask, patches.to(nlaf.dtype), out[i])
        if cur_pyr_level < num_levels - 1:
            cur_img = pyrdown(cur_img)
            if min(cur_img.size(2), cur_img.size(3)) < PS:
                break
    return out
