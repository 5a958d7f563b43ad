"""ORACLE for motion blur (test infrastructure, not product code): the reference's get_motion_kernel2d / motion_blur
(kornia/filters/kernels_geometry.py:30-109, kornia/filters/motion.py) restated with the same ATen calls, on top of the
rotate / filter2d restatements of oracle/kornia_restated.py.  It runs on whatever device its arguments live on: on the CPU
it reproduces the recorded goldens (tests/golden/motion.*.npz), on CUDA it is the same-device reference composition the
CUDA kernels are compared with."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle import kornia_restated as R


def get_motion_kernel2d(kernel_size, angle, direction=0.0, mode="nearest", device=None):
    """kernels_geometry.py:61-109: numbers become (1,) tensors on ``device`` (the reference: the default device, the CPU)."""
    dev, dtype = None, torch.get_default_dtype()
    for t in (angle, direction):
        if isinstance(t, torch.Tensor):
            dev, dtype = t.device, t.dtype
            break
    dev = device if device is not None else (dev if dev is not None else torch.device("cpu"))
    angle = angle if isinstance(angle, torch.Tensor) else torch.tensor([angle], device=dev, dtype=dtype)
    angle = angle[None] if angle.dim() == 0 else angle
    direction = direction if isinstance(direction, torch.Tensor) else torch.tensor([direction], device=dev, dtype=dtype)
    direction = direction[None] if direction.dim() == 0 else direction
    direction = (torch.clamp(direction, -1.0, 1.0) + 1.0) / 2.0
    k = torch.stack([(direction + ((1 - 2 * direction) / (kernel_size - 1)) * i) for i in range(kernel_size)], -1)
    kernel = F.pad(k[:, None], [0, 0, kernel_size // 2, kernel_size // 2, 0, 0])[:, None, ...]
    kernel = R.rotate(kernel, angle, mode=mode, align_corners=True)[:, 0]
    return kernel / kernel.sum(dim=(1, 2), keepdim=True)


def motion_blur(input, kernel_size, angle, direction, border_type="constant", mode="nearest", device=None):
    """motion.py: filter2d with the motion kernel (``device``: where number arguments build it)."""
    return R.filter2d(input, get_motion_kernel2d(kernel_size, angle, direction, mode, device), border_type)
