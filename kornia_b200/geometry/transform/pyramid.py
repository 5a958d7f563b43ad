"""Drop-in ``pyrdown`` / ``pyrup`` / ``build_pyramid`` / ``build_laplacian_pyramid`` (reference:
kornia/geometry/transform/pyramid.py:32-47,409-457,460-502,505-560,572-665; SURVEY.md 8f row 3).

The blur is the 5x5 binomial stencil through :func:`kornia_b200.filters.filter2d` -- the tiled TMA
kernel of csrc/filter2d_tiled.cuh (border folded into the tile load, no ``F.pad`` copy).  The 2x
resampling step is ``torch.nn.functional.interpolate``, the third-party call the reference itself makes
at pyramid.py:450-455,496-498 (the reference's own ``TODO: use kornia.geometry.resize``): 5 B/element of
traffic next to the blur's 8.  At an exact factor of two (``align_corners=False``, no gradient) the resampling is a 2x2
average and runs in the blur kernel's epilogue (kb200_pyrdown_forward): bit-identical to the composition;
``config.set("fused_pyrdown", 0)`` selects the composition.  ``ScalePyramid`` (the SIFT octave builder) is a feature-
detection caller and stays out of scope."""
from __future__ import annotations

import torch
import torch.nn.functional as F
from torch import nn

from ... import _lib, _ops, config
from ...core.check import check, check_shape
from ...filters.filter import filter2d

__all__ = ["pyrdown", "pyrup", "build_pyramid", "build_laplacian_pyramid", "PyrDown", "PyrUp"]

_BINOMIAL = (1.0, 4.0, 6.0, 4.0, 1.0)


def _binomial5x5() -> torch.Tensor:
    """(1,5,5) outer product of (1,4,6,4,1), scaled by 1/256 (pyramid.py:32-47); fp32 on the CPU like the
    reference's -- ``filter2d`` moves it to the image's device and dtype (filter.py:124-126)."""
    row = torch.tensor(_BINOMIAL)
    return (row[:, None] * row[None, :])[None] / 256.0


def _fused_request(input: torch.Tensor, border_type: str, align_corners: bool, factor: float):
    """(taps, border code) when the one-pass kernel (kb200_pyrdown_forward: the 2x2 average that the bilinear
    resampling reduces to at an exact factor of two runs in the blur's epilogue) may serve the call, else None.
    Switch ``fused_pyrdown`` of kornia_b200.config (on by default)."""
    if not config.enabled("fused_pyrdown") or torch.compiler.is_compiling():
        return None
    if not (input.is_cuda and input.dtype == torch.float32) or (torch.is_grad_enabled() and input.requires_grad):
        return None
    height, width = input.shape[-2:]
    if factor != 2.0 or align_corners or height % 2 or width % 4 or height < 4:
        return None
    code = _lib.BORDERS.get(str(border_type).lower())
    if code is None or code == _lib.CIRCULAR:
        return None
    return _binomial5x5().to(device=input.device, dtype=input.dtype), code


def pyrdown(input: torch.Tensor, border_type: str = "reflect", align_corners: bool = False, factor: float = 2.0) -> torch.Tensor:
    """Blur with the 5x5 binomial kernel, then resample bilinearly onto (int(H / factor), int(W // factor))."""
    check_shape(input, ["B", "C", "H", "W"])
    height, width = input.shape[-2:]
    fused = _fused_request(input, border_type, align_corners, factor)
    if fused is not None:
        try:
            return _ops.pyrdown_fused(input, *fused)
        except _lib.Unsupported:
            pass
    blurred = filter2d(input, _binomial5x5(), border_type)
    size = (int(float(height) / factor), int(float(width) // factor))  # the reference's mixed / and // (pyramid.py:452)
    return F.interpolate(blurred, size=size, mode="bilinear", align_corners=align_corners)


def pyrup(input: torch.Tensor, border_type: str = "reflect", align_corners: bool = False) -> torch.Tensor:
    """Resample bilinearly onto (2H, 2W), then blur with the 5x5 binomial kernel."""
    check_shape(input, ["B", "C", "H", "W"])
    height, width = input.shape[-2:]
    up = F.interpolate(input, size=(height * 2, width * 2), mode="bilinear", align_corners=align_corners)
    return filter2d(up, _binomial5x5(), border_type)


def _check_levels(max_level) -> None:
    # the reference's test is `isinstance(int) or max_level < 0` (pyramid.py:546-549): every int passes, a float raises
    check(isinstance(max_level, int) or max_level < 0, f"Invalid max_level, it must be a positive integer. Got: {max_level}")


def build_pyramid(input: torch.Tensor, max_level: int, border_type: str = "reflect", align_corners: bool = False) -> list[torch.Tensor]:
    """[input, pyrdown(input), pyrdown(pyrdown(input)), ...]: ``max_level`` entries (at least one)."""
    check_shape(input, ["B", "C", "H", "W"])
    _check_levels(max_level)
    levels = [input]
    for _ in range(max_level - 1):
        levels.append(pyrdown(levels[-1], border_type, align_corners))
    return levels


def _is_pow2(n: int) -> bool:
    return n > 0 and n & (n - 1) == 0


def _next_pow2(n: int) -> int:
    return 1 << (n - 1).bit_length()


def build_laplacian_pyramid(input: torch.Tensor, max_level: int, border_type: str = "reflect",
                            align_corners: bool = False) -> list[torch.Tensor]:
    """Band-pass levels g[i] - pyrup(g[i+1]) of the Gaussian pyramid g, followed by its last level.  The input is
    reflect-padded up to powers of two only when neither side already is one (pyramid.py:636-644)."""
    check_shape(input, ["B", "C", "H", "W"])
    _check_levels(max_level)
    h, w = input.shape[-2:]
    if not (_is_pow2(w) or _is_pow2(h)):
        input = F.pad(input, (0, _next_pow2(w) - w, 0, _next_pow2(h) - h), "reflect")
    gauss = build_pyramid(input, max_level, border_type, align_corners)
    bands = [gauss[i] - pyrup(gauss[i + 1], border_type, align_corners) for i in range(max_level - 1)]
    bands.append(gauss[-1])
    return bands


class PyrDown(nn.Module):
    """Module form of :func:`pyrdown` (pyramid.py:50-99)."""

    def __init__(self, border_type: str = "reflect", align_corners: bool = False, factor: float = 2.0) -> None:
        super().__init__()
        self.border_type = border_type
        self.align_corners = align_corners
        self.factor = factor

    def forward(self, input: torch.Tensor) -> torch.Tensor:
        return pyrdown(input, self.border_type, self.align_corners, self.factor)


class PyrUp(nn.Module):
    """Module form of :func:`pyrup` (pyramid.py:102-148)."""

    def __init__(self, border_type: str = "reflect", align_corners: bool = False) -> None:
        super().__init__()
        self.border_type = border_type
        self.align_corners = align_corners

    def forward(self, input: torch.Tensor) -> torch.Tensor:
        return pyrup(input, self.border_type, self.align_corners)
