"""Warps that start from a decoder's output (SURVEY.md 8f row 4): interleaved uint8 (B,H,W,C) in, planar fp32 (B,C,h,w) out.

The reference has no single function for this; its users write the three steps

    x = kornia.image_to_tensor(frames, keepdim=False)   # kornia/image/utils.py:27   HWC -> CHW view
    x = x.float() / 255.0                                # kornia/io/io.py:108-111    _to_float32
    y = kornia.geometry.transform.warp_perspective(x, M, dsize, ...)            # imgwarp.py:69

which materialise the 4x larger fp32 image twice before the warp reads it.  ``warp_perspective_from_uint8`` and
``warp_affine_from_uint8`` are those three lines as one call and one kernel (csrc/warp_u8.cuh): every tap is converted
inside the sampler with the rounding the reference's conversion has on a CUDA device (torch evaluates ``x / 255.0`` there
as ``x * (1/255)`` in fp32; ``normalize="exact"`` selects the true division of its CPU backend, one ulp apart for 126 of
the 256 byte values), so the result equals the composition on the same device bit for bit; the arguments
after ``image`` are those of ``warp_perspective`` / ``warp_affine`` with the same meaning, defaults, validation order
and exceptions.  Forward only: a uint8 image carries no gradient, and a matrix that requires grad is refused (use the
composition on the differentiable fp32 path for that).

The kernel is also run on the host emulator (tools/hostemu); nothing else in the library calls it.
"""
from __future__ import annotations

from typing import Optional

import torch

from .. import _prelude as P
from ... import _lib, _ops
from .imgwarp import _mode_codes

__all__ = ["warp_perspective_from_uint8", "warp_affine_from_uint8"]


def _batched_hwc(image: torch.Tensor) -> torch.Tensor:
    if not isinstance(image, torch.Tensor):
        raise TypeError(f"Input image type is not a torch.Tensor. Got {type(image)}")
    if image.dtype != torch.uint8:
        raise TypeError(f"Input image must be uint8 (a decoder's output). Got {image.dtype}")
    if image.dim() == 3:  # (H,W,C) -> (1,H,W,C): image_to_tensor(keepdim=False)
        image = image.unsqueeze(0)
    if image.dim() != 4:
        raise ValueError(f"Input image must be a BxHxWxC or HxWxC torch.Tensor. Got {image.shape}")
    return image


def _normalize_code(normalize) -> int:
    """False -> 0 (float(byte)); True / 'device' -> 1 (times the fp32 reciprocal of 255); 'exact' -> 2 (divided by 255)."""
    if normalize is True or normalize == "device":
        return 1
    if normalize is False:
        return 0
    if normalize == "exact":
        return 2
    raise ValueError(f"normalize must be True, False, 'device' or 'exact'. Got {normalize!r}")


def _no_grad_matrix(M: torch.Tensor) -> None:
    if torch.is_grad_enabled() and M.requires_grad:
        raise RuntimeError("kornia_b200: the uint8 ingest warp is forward-only; for d/dM use warp_perspective / warp_affine on "
                           "image.permute(0, 3, 1, 2).float() / 255")


def warp_perspective_from_uint8(
    image: torch.Tensor,
    M: torch.Tensor,
    dsize: tuple[int, int],
    mode: str = "bilinear",
    padding_mode: str = "zeros",
    align_corners: bool = True,
    fill_value: Optional[torch.Tensor] = None,
    normalize=True,
) -> torch.Tensor:
    """``warp_perspective(image.permute(0,3,1,2).float() / 255, M, dsize, ...)`` for a uint8 (B,H,W,C) or (H,W,C) ``image``
    in one kernel; ``normalize=False`` skips the division (``.float()`` only), ``"exact"`` divides the way torch's CPU
    backend does.  ``M`` (B,3,3) fp32."""
    image = _batched_hwc(image)
    if not isinstance(M, torch.Tensor):
        raise TypeError(f"Input M type is not a torch.Tensor. Got {type(M)}")
    if not (M.dim() == 3 and tuple(M.shape[-2:]) == (3, 3)):
        raise ValueError(f"Input M must be a Bx3x3 torch.Tensor. Got {M.shape}")
    if fill_value is None:
        fill_value = torch.zeros(3)
    if padding_mode == "fill" and fill_value.shape != torch.Size([3]):
        raise ValueError(f"Padding_tensor only supported for 3 channels. Got {fill_value.shape}")
    interp, pad = _mode_codes(mode, padding_mode, allow_fill=True)
    norm = _normalize_code(normalize)
    _no_grad_matrix(M)
    B, H, W, C = image.shape
    h_out, w_out = int(dsize[0]), int(dsize[1])
    if M.shape[0] != B:
        raise RuntimeError(f"grid_sampler(): expected grid and input to have same batch size, but got input with sizes "
                           f"{[B, C, H, W]} and grid with sizes {[M.shape[0], h_out, w_out, 2]}")
    with torch.no_grad():
        m = P.sampling_matrix(M.to(torch.float32), (H, W), (h_out, w_out), affine=False)
        bx, by = P.meshgrid_axes(h_out, w_out, image.device, torch.float32)
    fill = None
    if pad == _lib.FILL:
        if C != 3:
            raise RuntimeError(f"The size of tensor a ({C}) must match the size of tensor b (3) at non-singleton dimension 1")
        fill = fill_value
    return _ops.warp_u8hwc(image, m, bx, by, fill, h_out, w_out, True, interp, pad, bool(align_corners), norm)


def warp_affine_from_uint8(
    image: torch.Tensor,
    M: torch.Tensor,
    dsize: tuple[int, int],
    mode: str = "bilinear",
    padding_mode: str = "zeros",
    align_corners: bool = True,
    fill_value: Optional[torch.Tensor] = None,
    normalize=True,
) -> torch.Tensor:
    """``warp_affine(image.permute(0,3,1,2).float() / 255, M, dsize, ...)`` for a uint8 (B,H,W,C) or (H,W,C) ``image`` in
    one kernel.  ``M`` (B,2,3) or (1,2,3) shared by the batch; ``fill_value`` (C,), (1,) or 0-d."""
    image = _batched_hwc(image)
    if not isinstance(M, torch.Tensor):
        raise TypeError(f"Input M type is not a torch.Tensor. Got {type(M)}")
    interp, pad = _mode_codes(mode, padding_mode, allow_fill=True)
    if not (M.dim() == 3 and tuple(M.shape[-2:]) == (2, 3)):  # conversions.py:375-376
        raise ValueError(f"Input matrix must be a Bx2x3 tensor. Got {M.shape}")
    norm = _normalize_code(normalize)
    _no_grad_matrix(M)
    B, H, W, C = image.shape
    h_out, w_out = int(dsize[0]), int(dsize[1])
    B_M = M.shape[0]
    if B_M != B and not (B_M == 1 and B > 1):
        raise RuntimeError(f"grid_sampler(): expected grid and input to have same batch size, but got input with sizes "
                           f"{[B, C, H, W]} and grid with sizes {[B_M, h_out, w_out, 2]}")
    with torch.no_grad():
        m = P.sampling_matrix(M.to(torch.float32), (H, W), (h_out, w_out), affine=True)
        bx, by = P.affine_axes(h_out, w_out, bool(align_corners), image.device, torch.float32)
    fill = None
    if pad == _lib.FILL:
        fill = torch.zeros(C) if fill_value is None else fill_value
        if fill.ndim == 0 or (fill.ndim == 1 and fill.numel() == 1):
            fill = fill.reshape(1).expand(C)
        elif fill.ndim != 1 or fill.numel() != C:
            raise RuntimeError(f"The size of tensor a ({C}) must match the size of tensor b ({fill.shape[-1] if fill.ndim else 1}) "
                               "at non-singleton dimension 1")
    return _ops.warp_u8hwc(image, m, bx, by, fill, h_out, w_out, False, interp, pad, bool(align_corners), norm)
