"""Drop-in ``undistort_image`` (reference: kornia/geometry/calibration/undistort.py:138-198; SURVEY.md 8f row 4):
every output pixel is pushed through the lens model (``distort_points``) to find where the distorted image holds
it, and the image is resampled there by ``remap`` -- the tiled TMA kernel of csrc/remap_tiled.cuh (bilinear,
zeros, align_corners=True).  When no gradient is needed and the tilt coefficients are zero, the one-kernel form runs instead
(kb200_undistort_forward: the lens model evaluated per pixel in registers, no maps, ~45 fewer elementwise passes):
bit-identical to maps + remap on the same device;
``config.set("fused_undistort", 0)`` selects the composition."""
from __future__ import annotations

import torch

from ... import _lib, _ops, config
from ..transform.imgwarp import remap
from .distort import distort_points

__all__ = ["undistort_image", "undistort_image_from_uint8"]


def _fused_request(image: torch.Tensor, K: torch.Tensor, dist: torch.Tensor, B: int):
    """(B,16) lens numbers fx, fy, cx, cy, k1, k2, p1, p2, k3, k4, k5, k6, s1..s4 when the one-kernel path
    (kb200_undistort_forward: the lens model evaluated per pixel inside the sampling kernel, no maps) may serve the call,
    else None (switch ``fused_undistort`` of kornia_b200.config, on by default).  Not taken when a gradient is needed or the
    tilt coefficients are set."""
    if not config.enabled("fused_undistort") or torch.compiler.is_compiling():
        return None
    if not (image.is_cuda and image.dtype == torch.float32):
        return None
    if torch.is_grad_enabled() and (image.requires_grad or K.requires_grad or dist.requires_grad):
        return None
    lens = pack_lens(K, dist, image)
    return lens if lens is not None and lens.shape[0] == B else None


def pack_lens(K: torch.Tensor, dist: torch.Tensor, like: torch.Tensor):
    """(B,16) rows fx, fy, cx, cy, k1, k2, p1, p2, k3, k4, k5, k6, s1, s2, s3, s4 -- the layout kb200_undistort_forward
    reads (csrc/remap_tiled.cuh:lens_distort) -- or None when the tilt coefficients are set."""
    d = dist.reshape(-1, dist.shape[-1]).to(like)
    if d.shape[-1] == 14 and bool((d[:, 12:] != 0).any()):
        return None
    if d.shape[-1] < 12:
        d = torch.nn.functional.pad(d, [0, 12 - d.shape[-1]])
    Kf = K.reshape(-1, 3, 3).to(like)
    n = max(Kf.shape[0], d.shape[0])
    intrinsics = torch.stack([Kf[:, 0, 0], Kf[:, 1, 1], Kf[:, 0, 2], Kf[:, 1, 2]], -1)
    return torch.cat([intrinsics.expand(n, 4), d[:, :12].expand(n, 12)], -1).contiguous()


def undistort_image(image: torch.Tensor, K: torch.Tensor, dist: torch.Tensor) -> torch.Tensor:
    """Remove the lens distortion ``dist`` (*,4|5|8|12|14) of camera ``K`` (*,3,3) from ``image`` (*,C,H,W)."""
    if image.dim() < 3:
        raise ValueError(f"Image shape is invalid. Got: {image.shape}.")
    if K.shape[-2:] != (3, 3):
        raise ValueError(f"K matrix shape is invalid. Got {K.shape}.")
    if dist.shape[-1] not in (4, 5, 8, 12, 14):
        raise ValueError(f"Invalid number of distortion coefficients. Got {dist.shape[-1]}.")
    if not image.is_floating_point():
        raise ValueError(f"Invalid input image data type. Input should be float. Got {image.dtype}.")
    lead = image.shape[:-3]
    if lead != K.shape[:-2] or lead != dist.shape[:-1]:
        # (1,C,H,W) with an unbatched K (3,3) and dist (n,) is accepted (undistort.py:174-181)
        if not (lead == (1,) and K.shape[:-2] == () and dist.shape[:-1] == ()):
            raise ValueError("Input shape is invalid. Input batch dimensions should match. "
                             f"Got {image.shape[:-3]}, {K.shape[:-2]}, {dist.shape[:-1]}.")
    channels, rows, cols = image.shape[-3:]
    B = image.numel() // (channels * rows * cols)
    lens = _fused_request(image, K, dist, B)
    if lens is not None:
        try:
            return _ops.undistort_fused(image.reshape(B, channels, rows, cols), lens).view_as(image)
        except _lib.Unsupported:
            pass
    # pixel grid (x, y) of the output, (rows*cols, 2), in the image's dtype (grid.py:65-79 with normalized=False)
    xs = torch.linspace(0, cols - 1, cols, device=image.device, dtype=image.dtype)
    ys = torch.linspace(0, rows - 1, rows, device=image.device, dtype=image.dtype)
    gy, gx = torch.meshgrid(ys, xs, indexing="ij")
    pts = torch.stack([gx, gy], -1).reshape(-1, 2)
    seen_at = distort_points(pts, K, dist)
    map_x = seen_at[..., 0].reshape(B, rows, cols)
    map_y = seen_at[..., 1].reshape(B, rows, cols)
    out = remap(image.reshape(B, channels, rows, cols), map_x, map_y, align_corners=True)
    return out.view_as(image)


def undistort_image_from_uint8(image: torch.Tensor, K: torch.Tensor, dist: torch.Tensor, normalize=True) -> torch.Tensor:
    """``undistort_image(image_to_tensor(image).float() / 255, K, dist)`` for a decoder's uint8 ``image`` (B,H,W,C) or
    (H,W,C) -> fp32 (B,C,H,W) (SURVEY.md 8f row 4: the wire format and the maps fused).  One kernel
    (kb200_undistort_u8hwc_forward: bytes staged and converted once per window, lens model per pixel, no maps) when no
    gradient is asked for, the tilt coefficients are zero, C is 1 or 3 and W % 4 == 0; otherwise the image is converted
    and ``undistort_image`` runs (differentiable w.r.t. ``K`` and ``dist``).  ``normalize`` as in
    ``warp_perspective_from_uint8``: True / "device" (times 1/255, torch's CUDA ``x / 255.0``), "exact" (divided), False."""
    from ..transform.ingest import _batched_hwc, _normalize_code

    image = _batched_hwc(image)
    if K.shape[-2:] != (3, 3):
        raise ValueError(f"K matrix shape is invalid. Got {K.shape}.")
    if dist.shape[-1] not in (4, 5, 8, 12, 14):
        raise ValueError(f"Invalid number of distortion coefficients. Got {dist.shape[-1]}.")
    norm = _normalize_code(normalize)
    B = image.shape[0]
    needs_grad = torch.is_grad_enabled() and (K.requires_grad or dist.requires_grad)
    if image.is_cuda and not needs_grad:
        lens = pack_lens(K, dist, torch.empty(0, device=image.device, dtype=torch.float32))
        if lens is not None and lens.shape[0] in (1, B):  # one camera for the whole batch, or one per image
            try:
                return _ops.undistort_u8hwc(image, lens.expand(B, 16), norm)
            except _lib.Unsupported:
                pass
    x = image.permute(0, 3, 1, 2).float()
    if norm == 1:
        x = x / 255.0  # on a CUDA device: times the fp32 reciprocal (the form the kernel reproduces)
    elif norm == 2:
        x = torch.div(x, torch.tensor(255.0, device=x.device))  # a tensor divisor keeps the true division on every backend
    Kb = K if K.dim() == 3 else K.expand(B, 3, 3)
    db = dist if dist.dim() == 2 else dist.expand(B, dist.shape[-1])
    return undistort_image(x.contiguous(), Kb, db)
