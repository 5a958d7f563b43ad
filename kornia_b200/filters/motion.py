"""Drop-in ``get_motion_kernel2d``, ``motion_blur`` and ``MotionBlur`` (reference: kornia/filters/kernels_geometry.py:30-109,
kornia/filters/motion.py).

The kernel is the reference's op sequence -- a line of taps whose weights ramp with ``direction``, rotated by ``angle``
with :func:`~kornia_b200.geometry.transform.rotate` (``align_corners=True``), then divided by its sum -- and the image
goes through :func:`~kornia_b200.filters.filter2d`.  Motion kernels are mostly zeros; for K from 9 to 31 filter2d runs
a kernel that skips the zero taps and stays bit-identical to the dense sum.

Device: the reference builds the kernel on the CPU when ``angle`` and ``direction`` are Python numbers.  This package has
no CPU path, so they become tensors on the image's device in :func:`motion_blur` (and on the current CUDA device in
:func:`get_motion_kernel2d` called on its own); tensor arguments move there too.  CPU and CUDA nearest rotation can
round a tie differently, so a kernel built here can differ from the reference's CPU kernel by a tap at such a tie.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F
from torch import nn

from ..core.check import check, check_shape
from ..core.exceptions import BaseError
from ..geometry.transform import rotate
from .filter import filter2d
from .kernels import _check_kernel_size, _unpack_2d_ks

__all__ = ["get_motion_kernel2d", "motion_blur", "MotionBlur"]


def _device_dtype(angle, direction):
    """kornia/core/utils.py:_extract_device_dtype over (angle, direction): the tensors' device (None without tensors) and
    dtype (the default dtype without tensors)."""
    dev, dtype = None, None
    for t in (angle, direction):
        if not isinstance(t, torch.Tensor):
            continue
        if dev is None:
            dev, dtype = t.device, t.dtype
        elif dev != t.device or dtype != t.dtype:
            raise BaseError(f"Passed values are not in the same device and dtype. Got ({dev}, {dtype}) and ({t.device}, {t.dtype}).")
    return dev, (dtype if dtype is not None else torch.get_default_dtype())


def _batch(v, device, dtype) -> torch.Tensor:
    if isinstance(v, torch.Tensor):
        return v.to(device)
    return torch.tensor([v], device=device, dtype=dtype)


def _motion_kernel2d(kernel_size: int, angle, direction, mode: str, device: Optional[torch.device]) -> torch.Tensor:
    dev, dtype = _device_dtype(angle, direction)
    kernel_tuple = _unpack_2d_ks(kernel_size)
    _check_kernel_size(kernel_size, 2)
    # the reference's checks, in its order, before anything touches a device
    if isinstance(angle, torch.Tensor):
        angle = angle[None] if angle.dim() == 0 else angle
        check_shape(angle, ["B"])
    if isinstance(direction, torch.Tensor):
        direction = direction[None] if direction.dim() == 0 else direction
        check_shape(direction, ["B"])
    na = angle.size(0) if isinstance(angle, torch.Tensor) else 1
    nd = direction.size(0) if isinstance(direction, torch.Tensor) else 1
    if nd != na:
        show = lambda v: v if isinstance(v, torch.Tensor) else torch.tensor([v], dtype=dtype)  # noqa: E731
        check(False, f"direction and angle must have the same length. Got {show(direction)} and {show(angle)}.")

    if device is None:  # no CPU path: the arguments' CUDA device, else the current one
        device = dev if dev is not None and dev.type == "cuda" else torch.device("cuda", torch.cuda.current_device())
    angle, direction = _batch(angle, device, dtype), _batch(direction, device, dtype)

    # direction from [-1, 1] to [0, 1]; the line's taps ramp from `direction` to 1 - `direction`
    direction = (torch.clamp(direction, -1.0, 1.0) + 1.0) / 2.0
    k = torch.stack([(direction + ((1 - 2 * direction) / (kernel_size - 1)) * i) for i in range(kernel_size)], -1)
    kernel = F.pad(k[:, None], [0, 0, kernel_size // 2, kernel_size // 2, 0, 0])
    expected_shape = torch.Size([direction.size(0), *kernel_tuple])
    check(kernel.shape == expected_shape, f"Kernel shape should be {expected_shape}. Gotcha {kernel.shape}")
    kernel = kernel[:, None, ...]
    kernel = rotate(kernel, angle, mode=mode, align_corners=True)  # counter-clockwise
    kernel = kernel[:, 0]
    return kernel / kernel.sum(dim=(1, 2), keepdim=True)


def get_motion_kernel2d(kernel_size: int, angle: torch.Tensor | float, direction: torch.Tensor | float = 0.0,
                        mode: str = "nearest") -> torch.Tensor:
    """(B, K, K) motion-blur kernel: a horizontal line of ``kernel_size`` taps, weighted from the back (``direction``
    -1) through uniform (0) to the front (1), rotated counter-clockwise by ``angle`` degrees with ``mode``
    ('nearest' or 'bilinear') interpolation and normalised to sum 1.  ``angle`` / ``direction``: numbers or (B,)
    tensors.  The kernel is built on the arguments' CUDA device, or on the current CUDA device (module docstring)."""
    return _motion_kernel2d(kernel_size, angle, direction, mode, None)


def motion_blur(input: torch.Tensor, kernel_size: int, angle: float | torch.Tensor, direction: float | torch.Tensor,
                border_type: str = "constant", mode: str = "nearest") -> torch.Tensor:
    """Blur every channel of ``input`` (B,C,H,W) with the motion kernel of :func:`get_motion_kernel2d` -- one kernel for
    the batch when ``angle`` and ``direction`` are numbers, one per sample when they are (B,) tensors.  ``border_type``:
    'constant' | 'reflect' | 'replicate' | 'circular'.  The kernel is built on the image's device."""
    kernel = _motion_kernel2d(kernel_size, angle, direction, mode, input.device if isinstance(input, torch.Tensor) else None)
    return filter2d(input, kernel, border_type)


class MotionBlur(nn.Module):
    """Module form of :func:`motion_blur` (same constructor as the reference's)."""

    def __init__(self, kernel_size: int, angle: float, direction: float, border_type: str = "constant", mode: str = "nearest") -> None:
        super().__init__()
        self.kernel_size = kernel_size
        self.angle = angle
        self.direction = direction
        self.border_type = border_type
        self.mode = mode

    def __repr__(self) -> str:
        return (f"{self.__class__.__name__} (kernel_size={self.kernel_size}, "
                f"angle={self.angle}, direction={self.direction}, border_type={self.border_type})")

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return motion_blur(x, self.kernel_size, self.angle, self.direction, self.border_type)
