"""Drop-in ``pyrdown`` / ``pyrup`` / ``build_pyramid`` / ``build_laplacian_pyramid`` (reference:
kornia/geometry/transform/pyramid.py:32-47,409-457,460-502,505-560,572-665; SURVEY.md 8f row 3).

The blur is the 5x5 binomial stencil through :func:`kornia_b200.filters.filter2d` -- the tiled TMA
kernel of csrc/filter2d_tiled.cuh (border folded into the tile load, no ``F.pad`` copy).  The 2x
resampling step is ``torch.nn.functional.interpolate``, the third-party call the reference itself makes
at pyramid.py:450-455,496-498 (the reference's own ``TODO: use kornia.geometry.resize``): 5 B/element of
traffic next to the blur's 8.  At an exact factor of two (``align_corners=False``, no gradient) the resampling is a 2x2
average and runs in the blur kernel's epilogue (kb200_pyrdown_forward): bit-identical to the composition;
``config.set("fused_pyrdown", 0)`` selects the composition.

``ScalePyramid`` (the octave builder of ScaleSpaceDetector, SIFTFeature, HesAffNetHardNet and GFTTAffNetHardNet;
pyramid.py:151-404) builds each octave of an inference-style call (fp32 CUDA, no gradient, W % 4 == 0, every tap count
<= min(H, W), an instantiated tap chain) in ONE kernel (kb200_scale_octave_forward): it reads the octave's seed once and
writes the stacked (B, C, L, H, W) levels, bit-identical to ``_composed_octave`` -- the reference's op sequence over
this library's ``filter2d_separable`` and ``gaussian_blur2d`` plus ``torch.stack``, which is also the differentiable
path and what every other octave runs.  The octave seeds stay ``F.interpolate``, the call the reference makes."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F
from torch import nn

from ... import _lib, _ops, config
from ...core.check import check, check_shape
from .._prelude import _cached
from ...filters.filter import filter2d, filter2d_separable
from ...filters.gaussian import gaussian_blur2d

__all__ = ["pyrdown", "pyrup", "build_pyramid", "build_laplacian_pyramid", "PyrDown", "PyrUp", "ScalePyramid"]

_BINOMIAL = (1.0, 4.0, 6.0, 4.0, 1.0)


def _binomial5x5() -> torch.Tensor:
    """(1,5,5) outer product of (1,4,6,4,1), scaled by 1/256 (pyramid.py:32-47); fp32 on the CPU like the
    reference's -- ``filter2d`` moves it to the image's device and dtype (filter.py:124-126)."""
    row = torch.tensor(_BINOMIAL)
    return (row[:, None] * row[None, :])[None] / 256.0


def _binomial5x5_on(device, dtype) -> torch.Tensor:
    """:func:`_binomial5x5` made once per (device, dtype) on that device (the same values: small integers over 256), so a
    ``pyrdown`` call copies nothing from the host and can be captured in a CUDA graph."""

    def build():
        row = torch.tensor(_BINOMIAL, device=device)
        return ((row[:, None] * row[None, :])[None] / 256.0).to(dtype)

    return _cached(("binomial5x5", str(device), dtype), build)


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
    return _binomial5x5_on(input.device, input.dtype), code


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
    blurred = filter2d(input, _binomial5x5_on(input.device, input.dtype), border_type)
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


# tap chains of the octave kernel (csrc/octave_vwalk.cu): (initial blur or 0 for none, level kernels...) of ScalePyramid(),
# ScalePyramid(3, 1.6, 16, extra_levels=2) and ScalePyramid(3, 1.6, 32, double_image=True), each also without the blur
_OCTAVE_CHAINS = {(13, 11, 13, 17, 21, 25), (13, 11, 13, 17, 21), (11, 11, 13, 17, 21, 25), (0, 11, 13, 17, 21, 25), (0, 11, 13, 17, 21)}


class ScalePyramid(nn.Module):
    """Gaussian scale pyramid for local feature detection (same constructor, attributes, buffers and outputs as the
    reference's).  ``forward(x)`` returns ``(pyr, sigmas, pixel_dists)``, one entry per octave: ``pyr[o]`` is
    (B, C, L, H_o, W_o) with ``L = n_levels + extra_levels`` levels, each a reflect-bordered Gaussian blur of the level
    before it; ``sigmas[o]`` and ``pixel_dists[o]`` are (B, L).  Octave o + 1 is seeded with a bilinear
    (``align_corners=True``) half-size resize of level ``-extra_levels`` of octave o, until a side would fall to
    ``min_size`` or below.  ``double_image`` starts from a 2x bilinear upsample of the input."""

    def __init__(self, n_levels: int = 3, init_sigma: float = 1.6, min_size: int = 15, double_image: bool = False,
                 extra_levels: int = 3) -> None:
        super().__init__()
        self.n_levels = n_levels
        self.extra_levels = extra_levels
        self.init_sigma = init_sigma
        self.min_size = min_size
        self.border = min_size // 2 - 1
        self.sigma_step = 2 ** (1.0 / float(self.n_levels))
        self.double_image = double_image
        self._precompute_gauss_kernels(n_levels, extra_levels, init_sigma, double_image)

    def __repr__(self) -> str:
        return (f"{self.__class__.__name__}(n_levels={self.n_levels}, init_sigma={self.init_sigma}, min_size={self.min_size}, "
                f"extra_levels={self.extra_levels}, border={self.border}, sigma_step={self.sigma_step}, double_image={self.double_image})")

    @staticmethod
    def _make_gaussian_kernel1d(sigma: float, ksize: int) -> torch.Tensor:
        """Normalized 1-D Gaussian, built in fp64 and stored in fp32 (pyramid.py:238-242)."""
        x = torch.arange(ksize, dtype=torch.float64) - ksize // 2
        kernel = torch.exp(-0.5 * x**2 / sigma**2)
        return (kernel / kernel.sum()).float()

    def _precompute_gauss_kernels(self, n_levels: int, extra_levels: int, init_sigma: float, double_image: bool) -> None:
        """Buffers ``_gk_init`` (None when the first level is not blurred) and ``_gk_0 ... _gk_{L-2}``, with the
        reference's names, so its state_dict loads."""
        cur_sigma_init = 1.0 if double_image else 0.5
        if init_sigma > cur_sigma_init:
            sigma = max(math.sqrt(init_sigma**2 - cur_sigma_init**2), 0.01)
            self.register_buffer("_gk_init", self._make_gaussian_kernel1d(sigma, self.get_kernel_size(sigma)))
        else:
            self.register_buffer("_gk_init", None)
        cur_s = init_sigma
        for lvl in range(n_levels + extra_levels - 1):
            delta = cur_s * math.sqrt(self.sigma_step**2 - 1.0)
            self.register_buffer(f"_gk_{lvl}", self._make_gaussian_kernel1d(delta, self.get_kernel_size(delta)))
            cur_s *= self.sigma_step
        self._refresh_host_taps()

    def _refresh_host_taps(self) -> None:
        # the octave kernel takes its taps as launch arguments: a host copy of the buffers, read once here rather than per call
        names = ["_gk_init"] + [f"_gk_{lvl}" for lvl in range(self.n_levels + self.extra_levels - 1)]
        self._host_taps = {n: None if getattr(self, n) is None else [float(v) for v in getattr(self, n).detach().cpu().tolist()] for n in names}

    def _load_from_state_dict(self, *args, **kwargs):
        super()._load_from_state_dict(*args, **kwargs)
        self._refresh_host_taps()

    def get_kernel_size(self, sigma: float) -> int:
        """Odd kernel size ``int(8 sigma + 1)``, rounded up to odd (pyramid.py:279-297)."""
        ksize = int(2.0 * 4.0 * sigma + 1.0)
        if ksize % 2 == 0:
            ksize += 1
        return ksize

    def _blur_fast(self, x: torch.Tensor, kernel: torch.Tensor) -> torch.Tensor:
        """The reference's F.pad + F.conv2d separable blur (pyramid.py:267-277) as one filter2d_separable call."""
        k = kernel.to(device=x.device, dtype=x.dtype)[None]
        return filter2d_separable(x, k, k, "reflect")

    def _first_blur(self, x: torch.Tensor, cur_sigma: float) -> torch.Tensor:
        sigma = max(math.sqrt(self.init_sigma**2 - cur_sigma**2), 0.01)
        ksize = self.get_kernel_size(sigma)
        min_dim = min(x.size(2), x.size(3))
        if self._gk_init is not None and ksize <= min_dim:
            return self._blur_fast(x, self._gk_init)
        ksize = min(ksize, min_dim if min_dim % 2 == 1 else min_dim - 1)
        return gaussian_blur2d(x, (ksize, ksize), (sigma, sigma))

    def _seed(self, input: torch.Tensor) -> tuple[torch.Tensor, float, float]:
        pixel_distance, cur_sigma = 1.0, 0.5
        if self.double_image:
            x = F.interpolate(input, scale_factor=2.0, mode="bilinear", align_corners=True)
            pixel_distance = 0.5
            cur_sigma *= 2.0
        else:
            x = input
        return x, cur_sigma, pixel_distance

    def get_first_level(self, input: torch.Tensor) -> tuple[torch.Tensor, float, float]:
        """``(level, sigma, pixel_distance)`` of the first level: the (2x upsampled) input, blurred up to ``init_sigma``
        when the assumed input blur (0.5, or 1.0 with ``double_image``) is below it."""
        x, cur_sigma, pixel_distance = self._seed(input)
        if self.init_sigma > cur_sigma:
            return self._first_blur(x, cur_sigma), self.init_sigma, pixel_distance
        return x, cur_sigma, pixel_distance

    def _composed_octave(self, seed: torch.Tensor, blur_first: bool, cur_sigma: float) -> list[torch.Tensor]:
        """Levels of one octave as the reference builds them (pyramid.py:324-335, 367-384), over this library's filters."""
        levels = [self._first_blur(seed, cur_sigma) if blur_first else seed]
        cur_sigma_oct = self.init_sigma
        for level_idx in range(1, self.n_levels + self.extra_levels):
            kernel = getattr(self, f"_gk_{level_idx - 1}")
            min_dim = min(levels[-1].size(2), levels[-1].size(3))
            if kernel.shape[0] <= min_dim:
                new_level = self._blur_fast(levels[-1], kernel)
            else:  # tiny level: the reference's clamped gaussian_blur2d
                delta_sigma = cur_sigma_oct * math.sqrt(self.sigma_step**2 - 1.0)
                ksize = min_dim if min_dim % 2 == 1 else min_dim - 1
                new_level = gaussian_blur2d(levels[-1], (ksize, ksize), (delta_sigma, delta_sigma))
            cur_sigma_oct *= self.sigma_step
            levels.append(new_level)
        return levels

    def _fused_octave(self, seed: torch.Tensor, blur_first: bool):
        """The octave as one kernel, (B, C, L, H, W), or None when the octave takes the composition."""
        if seed.dtype != torch.float32 or not seed.is_cuda or seed.numel() == 0 or (torch.is_grad_enabled() and seed.requires_grad):
            return None
        L = self.n_levels + self.extra_levels
        names = (["_gk_init"] if blur_first else []) + [f"_gk_{lvl}" for lvl in range(L - 1)]
        taps = [self._host_taps.get(n) for n in names]
        if any(t is None for t in taps):
            return None
        ksizes = ([len(taps[0])] if blur_first else [0]) + [len(t) for t in taps[int(blur_first):]]
        H, W = seed.shape[-2:]
        if W % 4 or max(ksizes) > min(H, W) or tuple(ksizes) not in _OCTAVE_CHAINS:
            return None
        try:
            return _ops.ops.scale_octave_fwd(seed, [v for t in taps for v in t], ksizes)
        except _lib.Unsupported:
            return None

    def forward(self, x: torch.Tensor) -> tuple[list[torch.Tensor], list[torch.Tensor], list[torch.Tensor]]:
        """``(pyr, sigmas, pixel_dists)`` of ``x`` (B, C, H, W); see the class docstring."""
        return self._pyramid(x, True)

    def _composed_pyramid(self, x: torch.Tensor) -> tuple[list[torch.Tensor], list[torch.Tensor], list[torch.Tensor]]:
        """``forward`` with every octave composed: the reference's op sequence, what the octave kernel must equal."""
        return self._pyramid(x, False)

    def _pyramid(self, x: torch.Tensor, fused: bool):
        bs = x.size(0)
        L = self.n_levels + self.extra_levels
        seed, cur_sigma, pixel_distance = self._seed(x)
        assumed = cur_sigma
        blur_first = self.init_sigma > cur_sigma
        if blur_first:
            cur_sigma = self.init_sigma
        sigmas = [torch.full((bs, L), cur_sigma, device=x.device, dtype=x.dtype)]
        pixel_dists = [torch.full((bs, L), pixel_distance, device=x.device, dtype=x.dtype)]
        pyr = []
        while True:
            octave = self._fused_octave(seed, blur_first) if fused else None
            if octave is None:
                levels = self._composed_octave(seed, blur_first, assumed)
                seed_level = levels[-self.extra_levels]
                octave = torch.stack(levels, 2)
            else:
                seed_level = octave[:, :, -self.extra_levels]
            pyr.append(octave)
            cur_sigma_oct = self.init_sigma
            for level_idx in range(1, L):
                cur_sigma_oct *= self.sigma_step
                sigmas[-1][:, level_idx] = cur_sigma_oct
                pixel_dists[-1][:, level_idx] = pixel_distance
            H, W = seed_level.shape[2], seed_level.shape[3]
            if min(H // 2, W // 2) <= self.min_size:
                break
            seed = F.interpolate(seed_level, size=(H // 2, W // 2), mode="bilinear", align_corners=True)
            blur_first = False
            pixel_distance *= 2.0
            sigmas.append(torch.full((bs, L), self.init_sigma, device=x.device, dtype=x.dtype))
            pixel_dists.append(torch.full((bs, L), pixel_distance, device=x.device, dtype=x.dtype))
        return pyr, sigmas, pixel_dists
