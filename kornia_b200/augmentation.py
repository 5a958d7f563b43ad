"""The augmentation callers of the hot path (SURVEY.md section 8f row 1), as classes with the reference's constructors:

    RandomPerspective   kornia/augmentation/_2d/geometric/perspective.py:34-134   -> get_perspective_transform + warp_perspective
    RandomAffine        kornia/augmentation/_2d/geometric/affine.py:33-166        -> get_affine_matrix2d + warp_affine
    RandomGaussianBlur  kornia/augmentation/_2d/intensity/gaussian_blur.py:30-122 -> gaussian_blur2d with per-sample sigmas
    RandomMotionBlur    kornia/augmentation/_2d/intensity/motion_blur.py          -> motion_blur with per-sample angles / directions

What is kept from the reference's framework (kornia/augmentation/base.py:159-330, _2d/base.py:55-140) is the contract those
classes expose: ``forward(input, params=None)`` accepting (H,W), (C,H,W) or (B,C,H,W); the parameter dictionaries (same keys,
shapes and -- on the default CPU generator -- the same random stream: gate first, then the generator's draws in the
reference's order, so a ``torch.manual_seed`` reproduces the reference's parameters bit for bit); ``p`` / ``p_batch`` /
``same_on_batch`` / ``keepdim``; ``._params`` and ``.transform_matrix`` after the call; every sample is transformed and the
gate blends with ``torch.where`` (base.py:282-300).  Not rebuilt: containers (AugmentationSequential), masks / boxes /
keypoints, ``inverse``, ONNX export -- the control plane around the path, out of scope.

What changes is the execution: sampling happens on the input's device (``.to(device)`` moves the generator like the
reference's), the corner points go to the homography in ONE launch (kb200_perspective_from_points) and on to the fused warp
kernel -- no (B,8,8) solve, no meshgrid, no sampling grid; the blur taps of per-sample sigmas feed the one-pass separable
kernel."""
from __future__ import annotations

import math
from typing import Any, Dict, Optional, Tuple, Union

import torch
from torch import nn
from torch.distributions import Uniform

from .filters import gaussian_blur2d, motion_blur
from .geometry._prelude import affine_to_homography
from .geometry.transform import get_perspective_transform, get_rotation_matrix2d, warp_affine, warp_perspective

__all__ = ["RandomPerspective", "RandomAffine", "RandomGaussianBlur", "RandomMotionBlur", "get_affine_matrix2d", "get_shear_matrix2d"]

_RESAMPLE = {0: "nearest", 1: "bilinear", 2: "bicubic", "nearest": "nearest", "bilinear": "bilinear", "bicubic": "bicubic"}
_PADDING = {0: "zeros", 1: "border", 2: "reflection", 3: "fill", "zeros": "zeros", "border": "border", "reflection": "reflection", "fill": "fill"}


def _name(table, value, what: str) -> str:
    key = getattr(value, "name", value)  # the reference's Resample / SamplePadding enums carry .name
    key = key.lower() if isinstance(key, str) else key
    if key not in table:
        raise NotImplementedError(f"Invalid {what}: {value}")
    return table[key]


def _rsample(shape, dist: Uniform, same_on_batch: bool) -> torch.Tensor:
    """kornia/augmentation/utils/helpers.py:289-306 (_adapted_rsampling): one draw shared by the batch when same_on_batch."""
    shape = torch.Size(shape)
    if same_on_batch:
        r = dist.rsample(torch.Size((1, *shape[1:])))
        return r.repeat(shape[0], *[1] * (len(r.shape) - 1))
    return dist.rsample(shape)


def _range(value, name: str, center: float = 0.0, bounds=(-float("inf"), float("inf")), singular: bool = False) -> torch.Tensor:
    """(lo, hi) tensor from a scalar (center +- value) or a pair, as kornia/augmentation/utils/param_validation.py:_range_bound."""
    t = torch.as_tensor(value, dtype=torch.float32) if not isinstance(value, torch.Tensor) else value.float()
    if t.dim() == 0:
        if t < 0:
            raise ValueError(f"If {name} is a single number, it must be non negative. Got {t}.")
        t = torch.stack([center - t, center + t]) if not singular else torch.stack([t, t])
    if t.shape != torch.Size([2]):
        raise TypeError(f"{name} must be a scalar or a pair. Got {value}.")
    if not (bounds[0] <= t[0] <= t[1] <= bounds[1]) and not singular:
        raise ValueError(f"{name} out of bounds {bounds}: {value}")
    return t


# ------------------------------------------------------------------------------------------ matrix builders
def get_shear_matrix2d(center: torch.Tensor, sx: Optional[torch.Tensor] = None, sy: Optional[torch.Tensor] = None) -> torch.Tensor:
    """(B,3,3) shear about ``center`` by the angles ``sx`` / ``sy`` in radians (imgwarp.py:817-869)."""
    sx = torch.zeros(center.size(0), device=center.device, dtype=center.dtype) if sx is None else sx
    sy = torch.zeros(center.size(0), device=center.device, dtype=center.dtype) if sy is None else sy
    x, y = center[:, 0], center[:, 1]
    sx_tan, sy_tan = torch.tan(sx), torch.tan(sy)
    ones = torch.ones_like(sx)
    mat = torch.stack([ones, -sx_tan, sx_tan * y, -sy_tan, ones + sx_tan * sy_tan, sy_tan * (x - sx_tan * y)], dim=-1).view(-1, 2, 3)
    return affine_to_homography(mat)


def get_affine_matrix2d(translations: torch.Tensor, center: torch.Tensor, scale: torch.Tensor, angle: torch.Tensor,
                        sx: Optional[torch.Tensor] = None, sy: Optional[torch.Tensor] = None) -> torch.Tensor:
    """(B,3,3) = [R(-angle) S about center, + translation] @ shear (imgwarp.py:746-787)."""
    transform = get_rotation_matrix2d(center, -angle, scale)
    transform = transform.clone()
    transform[..., 2] += translations
    transform_h = affine_to_homography(transform)
    if sx is not None or sy is not None:
        transform_h = transform_h @ get_shear_matrix2d(center, sx, sy)
    return transform_h


# ------------------------------------------------------------------------------------------ the shared contract
class _RandomAugmentation2D(nn.Module):
    """forward / parameter / gate plumbing of kornia/augmentation/base.py (see the module docstring for what is kept)."""

    geometric = False

    def __init__(self, p: float = 0.5, p_batch: float = 1.0, same_on_batch: bool = False, keepdim: bool = False) -> None:
        super().__init__()
        self.p, self.p_batch, self.same_on_batch, self.keepdim = p, p_batch, same_on_batch, keepdim
        self._params: Dict[str, torch.Tensor] = {}
        self._transform_matrix: Optional[torch.Tensor] = None
        self.flags: Dict[str, Any] = {}
        self.device, self.dtype = torch.device("cpu"), torch.get_default_dtype()

    # -- random stream: device / dtype follow .to() like base.py:101-119
    def set_rng_device_and_dtype(self, device: torch.device, dtype: torch.dtype) -> None:
        self.device, self.dtype = torch.device(device), dtype
        self._samplers = None

    def to(self, *args: Any, **kwargs: Any):
        device, dtype, _, _ = torch._C._nn._parse_to(*args, **kwargs)
        self.set_rng_device_and_dtype(device if device is not None else self.device, dtype if dtype is not None else self.dtype)
        return super().to(*args, **kwargs)

    def _uniform(self, lo, hi, key: Optional[str] = None) -> Uniform:
        """Uniform(lo, hi) on the generator device; ``key`` caches the sampler (and its two scalar tensors) across calls --
        building them is ~10 host-side tensor ops per call otherwise.  set_rng_device_and_dtype / .to() drop the cache."""
        cache = getattr(self, "_samplers", None)
        if cache is None:
            cache = self._samplers = {}
        if key is not None and key in cache:
            return cache[key]
        dist = Uniform(torch.as_tensor(lo, device=self.device, dtype=self.dtype), torch.as_tensor(hi, device=self.device, dtype=self.dtype),
                       validate_args=False)
        if key is not None:
            cache[key] = dist
        return dist

    def _gate(self, batch: int) -> torch.Tensor:
        """base.py:165-196: batch gate, then element gate; the draws (torch.rand on the generator device) in that order."""
        if self.p_batch == 1:
            batch_prob = torch.ones(1, device=self.device, dtype=self.dtype)
        elif self.p_batch == 0:
            batch_prob = torch.zeros(1, device=self.device, dtype=self.dtype)
        else:
            batch_prob = (torch.rand(1, device=self.device) < self.p_batch).to(self.dtype)
        if self.p == 1:
            elem = torch.ones(batch, device=self.device, dtype=self.dtype)
        elif self.p == 0:
            elem = torch.zeros(batch, device=self.device, dtype=self.dtype)
        elif self.same_on_batch:
            elem = (torch.rand(1, device=self.device) < self.p).to(self.dtype).expand(batch)
        else:
            elem = (torch.rand(batch, device=self.device) < self.p).to(self.dtype)
        return batch_prob * elem

    def generate_parameters(self, batch_shape: Tuple[int, ...]) -> Dict[str, torch.Tensor]:
        raise NotImplementedError

    def forward_parameters(self, batch_shape: Tuple[int, ...]) -> Dict[str, torch.Tensor]:
        batch_prob = self._gate(batch_shape[0])
        params = self.generate_parameters(tuple(batch_shape))
        params["batch_prob"] = batch_prob
        params["forward_input_shape"] = torch.tensor(batch_shape, dtype=torch.long)
        return params

    # -- what the subclasses implement
    def compute_transformation(self, input: torch.Tensor, params: Dict[str, torch.Tensor], flags: Dict[str, Any]) -> torch.Tensor:
        return torch.eye(3, device=input.device, dtype=input.dtype).expand(input.shape[0], 3, 3)

    def apply_transform(self, input: torch.Tensor, params: Dict[str, torch.Tensor], flags: Dict[str, Any],
                        transform: Optional[torch.Tensor] = None) -> torch.Tensor:
        raise NotImplementedError

    @property
    def transform_matrix(self) -> Optional[torch.Tensor]:
        return self._transform_matrix

    def forward(self, input: torch.Tensor, params: Optional[Dict[str, torch.Tensor]] = None, **kwargs: Any) -> torch.Tensor:
        if not isinstance(input, torch.Tensor):
            raise TypeError(f"Input type is not a torch.Tensor. Got {type(input)}")
        if not input.is_floating_point():
            raise TypeError(f"Expected input of a floating dtype. Got {input.dtype}")
        ori_shape = input.shape
        if input.dim() not in (2, 3, 4):
            raise ValueError(f"Input size must have a shape of either (H, W), (C, H, W) or (*, C, H, W). Got {input.shape}")
        x = input.reshape((1,) * (4 - input.dim()) + tuple(input.shape))
        if params is None:
            params = self.forward_parameters(tuple(x.shape))
        if "batch_prob" not in params:
            params["batch_prob"] = torch.tensor([True] * x.shape[0])
        self._params = params
        flags = {**self.flags, **{k: v for k, v in kwargs.items() if k in self.flags}}
        always = self.p == 1.0 and self.p_batch == 1.0
        to_apply = torch.atleast_1d(params["batch_prob"] > 0.5).to(x.device)
        transform = None
        if self.geometric:
            transform = self.compute_transformation(x, params, flags)
            if not always:
                eye = torch.eye(3, device=x.device, dtype=x.dtype).expand(x.shape[0], 3, 3)
                self._transform_matrix = torch.where(to_apply.view(-1, 1, 1), transform, eye)
            else:
                self._transform_matrix = transform
        out = self.apply_transform(x, params, flags, transform=transform)
        if not always:  # every sample is transformed; the gate selects (base.py:282-300)
            out = torch.where(to_apply.view(-1, 1, 1, 1), out, x)
        if self.keepdim:
            while out.dim() > len(ori_shape):
                if out.shape[0] != 1:
                    raise AssertionError(f"Dimension 0 of the output is expected to be 1, got {out.shape[0]}")
                out = out.squeeze(0)
        return out


# ------------------------------------------------------------------------------------------ the three classes
class RandomPerspective(_RandomAugmentation2D):
    """Random perspective: each image corner moves by up to ``distortion_scale`` / 2 of the image size (``sampling_method``
    'basic': inwards; 'area_preserving': any direction), the four point pairs give the homography, the image is warped.
    Constructor of kornia/augmentation/_2d/geometric/perspective.py:76-89."""

    geometric = True

    def __init__(self, distortion_scale: Union[torch.Tensor, float] = 0.5, resample: Union[str, int] = "BILINEAR", same_on_batch: bool = False,
                 align_corners: bool = False, p: float = 0.5, keepdim: bool = False, sampling_method: str = "basic") -> None:
        super().__init__(p=p, same_on_batch=same_on_batch, keepdim=keepdim)
        if sampling_method not in ("basic", "area_preserving"):
            raise NotImplementedError(f"Sampling method {sampling_method} not yet implemented.")
        self.distortion_scale, self.sampling_method = distortion_scale, sampling_method
        self.flags = {"align_corners": align_corners, "resample": _name(_RESAMPLE, resample, "resample")}

    def generate_parameters(self, batch_shape):
        """random_generator/_2d/perspective.py:74-110: rand in [0,1) of shape (B,4,2), scaled by (w, h) * scale / 2."""
        B, height, width = batch_shape[0], batch_shape[-2], batch_shape[-1]
        dev, dt = self.device, self.dtype
        scale = torch.as_tensor(self.distortion_scale, device=dev, dtype=dt)
        if not (scale.dim() == 0 and 0 <= scale <= 1):
            raise AssertionError(f"'distortion_scale' must be a scalar within [0, 1]. Got {scale}.")
        start = torch.tensor([[[0.0, 0], [width - 1, 0], [width - 1, height - 1], [0, height - 1]]], device=dev, dtype=dt).expand(B, -1, -1)
        factor = torch.stack([scale * width / 2, scale * height / 2], dim=0).view(-1, 1, 2)
        rand_val = _rsample(start.shape, self._uniform(0, 1, "unit"), self.same_on_batch)
        if self.sampling_method == "basic":
            offset = factor * rand_val * torch.tensor([[[1, 1], [-1, 1], [-1, -1], [1, -1]]], device=dev, dtype=dt)
        else:
            offset = 2 * factor * (rand_val - 0.5)
        return {"start_points": start, "end_points": start + offset}

    def compute_transformation(self, input, params, flags):
        return get_perspective_transform(params["start_points"].to(input), params["end_points"].to(input))

    def apply_transform(self, input, params, flags, transform=None):
        _, _, height, width = input.shape
        return warp_perspective(input, transform, (height, width), mode=flags["resample"], align_corners=flags["align_corners"])


class RandomAffine(_RandomAugmentation2D):
    """Random rotation / translation / scale / shear about the image centre.  Constructor of
    kornia/augmentation/_2d/geometric/affine.py:80-107."""

    geometric = True

    def __init__(self, degrees, translate=None, scale=None, shear=None, resample: Union[str, int] = "BILINEAR", same_on_batch: bool = False,
                 align_corners: bool = False, padding_mode: Union[str, int] = "ZEROS", p: float = 0.5, keepdim: bool = False,
                 fill_value: Optional[Union[torch.Tensor, float]] = None) -> None:
        super().__init__(p=p, same_on_batch=same_on_batch, keepdim=keepdim)
        self.degrees, self.translate, self.scale, self.shear = degrees, translate, scale, shear
        if fill_value is not None and not isinstance(fill_value, torch.Tensor):
            fill_value = torch.as_tensor(fill_value)
        self.flags = {"resample": _name(_RESAMPLE, resample, "resample"), "padding_mode": _name(_PADDING, padding_mode, "padding_mode"),
                      "align_corners": align_corners, "fill_value": fill_value}

    def _ranges(self):
        deg = _range(self.degrees, "degrees", 0.0, (-360, 360))
        tr = None if self.translate is None else torch.as_tensor(self.translate, dtype=torch.float32)
        sc = None if self.scale is None else torch.as_tensor(self.scale, dtype=torch.float32)
        if sc is not None and sc.numel() not in (2, 4):
            raise ValueError(f"'scale' expected to be either 2 or 4 elements. Got {self.scale}")
        sh = None
        if self.shear is not None:
            s = torch.as_tensor(self.shear, dtype=torch.float32)
            if s.shape == torch.Size([2, 2]):
                sh = s
            else:
                sh = torch.stack([_range(s if s.dim() == 0 else s[:2], "shear-x", 0.0, (-360, 360)),
                                  torch.zeros(2) if s.dim() == 0 or len(s) == 2 else _range(s[2:], "shear-y", 0.0, (-360, 360))])
        return deg, tr, sc, sh

    def generate_parameters(self, batch_shape):
        """random_generator/_2d/affine.py:160-222: angle, scale (x, then y), translate x, translate y, shear x, shear y."""
        B, height, width = batch_shape[0], batch_shape[-2], batch_shape[-1]
        dev, dt, same = self.device, self.dtype, self.same_on_batch
        if getattr(self, "_range_cache", None) is None:
            self._range_cache = self._ranges()
        deg, tr, sc, sh = self._range_cache
        angle = _rsample((B,), self._uniform(deg[0], deg[1], "angle"), same)
        if sc is not None:
            scale = _rsample((B,), self._uniform(sc[0], sc[1], "scale_x"), same).unsqueeze(1).repeat(1, 2)
            if sc.numel() == 4:
                scale[:, 1] = _rsample((B,), self._uniform(sc[2], sc[3], "scale_y"), same)
        else:
            scale = torch.ones((B, 2), device=dev, dtype=dt)
        if tr is not None:
            translations = torch.stack([_rsample((B,), self._uniform(-tr[0], tr[0], "tx"), same) * width,
                                        _rsample((B,), self._uniform(-tr[1], tr[1], "ty"), same) * height], dim=-1)
        else:
            translations = torch.zeros((B, 2), device=dev, dtype=dt)
        center = (torch.tensor([width, height], device=dev, dtype=dt).view(1, 2) / 2.0 - 0.5).expand(B, -1)
        if sh is not None:
            sx = _rsample((B,), self._uniform(sh[0][0], sh[0][1], "shear_x"), same)
            sy = _rsample((B,), self._uniform(sh[1][0], sh[1][1], "shear_y"), same)
        else:
            sx = torch.zeros(B, device=dev, dtype=dt)
            sy = torch.zeros(B, device=dev, dtype=dt)
        return {"translations": translations, "center": center, "scale": scale, "angle": angle, "shear_x": sx, "shear_y": sy}

    def compute_transformation(self, input, params, flags):
        k = math.pi / 180.0  # affine.py:113-118
        get = lambda name: torch.as_tensor(params[name], device=input.device, dtype=input.dtype)  # noqa: E731
        return get_affine_matrix2d(get("translations"), get("center"), get("scale"), get("angle"), get("shear_x") * k, get("shear_y") * k)

    def apply_transform(self, input, params, flags, transform=None):
        _, _, height, width = input.shape
        return warp_affine(input, transform[:, :2, :], (height, width), flags["resample"], align_corners=flags["align_corners"],
                           padding_mode=flags["padding_mode"], fill_value=flags["fill_value"])


class RandomGaussianBlur(_RandomAugmentation2D):
    """Gaussian blur with a standard deviation drawn per sample from ``sigma`` = (min, max).  Constructor of
    kornia/augmentation/_2d/intensity/gaussian_blur.py:62-80."""

    def __init__(self, kernel_size: Union[Tuple[int, int], int], sigma: Union[Tuple[float, float], torch.Tensor], border_type: str = "reflect",
                 separable: bool = True, same_on_batch: bool = False, p: float = 0.5, keepdim: bool = False) -> None:
        super().__init__(p=p, same_on_batch=same_on_batch, p_batch=1.0, keepdim=keepdim)
        if sigma[1] < sigma[0]:
            raise TypeError(f"sigma_max should be higher than sigma_min: {sigma} passed.")
        self.sigma = sigma
        self.flags = {"kernel_size": kernel_size, "separable": separable, "border_type": getattr(border_type, "name", border_type).lower()}

    def generate_parameters(self, batch_shape):
        s = self.sigma if isinstance(self.sigma, torch.Tensor) else torch.tensor(self.sigma)
        return {"sigma": _rsample((batch_shape[0],), self._uniform(s[0], s[1], "sigma"), self.same_on_batch)}

    def apply_transform(self, input, params, flags, transform=None):
        sigma = params["sigma"].to(input).unsqueeze(-1).expand(-1, 2)
        if self.same_on_batch:
            sigma = sigma[:1]
        return gaussian_blur2d(input, kernel_size=flags["kernel_size"], sigma=sigma, border_type=flags["border_type"], separable=flags["separable"])


_BORDER = {0: "constant", 1: "reflect", 2: "replicate", 3: "circular", "constant": "constant", "reflect": "reflect", "replicate": "replicate",
           "circular": "circular"}


class RandomMotionBlur(_RandomAugmentation2D):
    """Motion blur with an angle and a direction drawn per sample and one kernel size for the batch.  Constructor of
    kornia/augmentation/_2d/intensity/motion_blur.py: ``kernel_size`` an odd int or a (min, max) range, ``angle`` in
    degrees and ``direction`` in [-1, 1] as a number (the range -x .. x) or a pair."""

    def __init__(self, kernel_size: Union[int, Tuple[int, int]], angle: Union[torch.Tensor, float, Tuple[float, float]],
                 direction: Union[torch.Tensor, float, Tuple[float, float]], border_type: Union[int, str] = "CONSTANT",
                 resample: Union[str, int] = "NEAREST", same_on_batch: bool = False, p: float = 0.5, keepdim: bool = False) -> None:
        super().__init__(p=p, same_on_batch=same_on_batch, keepdim=keepdim)
        self.kernel_size, self.angle, self.direction = kernel_size, angle, direction
        # the reference validates when its generator builds the samplers, in the constructor: angle, direction, kernel size
        _range(angle, "angle", 0.0, (-360, 360))
        _range(direction, "direction", 0.0, (-1, 1))
        self._ksize_range()
        self.flags = {"border_type": _name(_BORDER, border_type, "border_type"), "resample": _name(_RESAMPLE, resample, "resample")}

    def _ksize_range(self) -> Tuple[int, int]:
        """random_generator/_2d/motion_blur.py make_samplers: the half sizes k // 2 the sampler draws between."""
        k = self.kernel_size
        if isinstance(k, int):
            if not (k >= 3 and k % 2 == 1):
                raise AssertionError(f"`kernel_size` must be odd and greater than 3. Got {k}.")
            return k // 2, k // 2
        if isinstance(k, tuple):
            if len(k) != 2:
                raise AssertionError(f"`kernel_size` must be (2,) if it is a tuple. Got {k}.")
            return k[0] // 2, k[1] // 2
        raise TypeError(f"Unsupported type: {type(k)}")

    def generate_parameters(self, batch_shape):
        """MotionBlurGenerator.forward (angle, direction, then kernel size: a CPU draw, since the reference's sampler is
        built from Python numbers), then RandomMotionBlur.generate_parameters' ``idx``.  The factors land where the
        reference puts them: on the device and dtype of tensor ``angle`` / ``direction``, else on the CPU in the default
        dtype."""
        B, same = batch_shape[0], self.same_on_batch
        angle = _range(self.angle, "angle", 0.0, (-360, 360))
        direction = _range(self.direction, "direction", 0.0, (-1, 1))
        lo, hi = self._ksize_range()
        angle_factor = _rsample((B,), self._uniform(angle[0], angle[1]), same)
        direction_factor = _rsample((B,), self._uniform(direction[0], direction[1]), same)
        ksize_sampler = Uniform(torch.as_tensor(float(lo)), torch.as_tensor(float(hi)), validate_args=False)
        ksize_factor = _rsample((B,), ksize_sampler, same).int() * 2 + 1
        dev, dt = torch.empty(0).device, torch.get_default_dtype()
        for t in (self.angle, self.direction):
            if isinstance(t, torch.Tensor):
                dev, dt = t.device, t.dtype
                break
        idx = torch.tensor([0]) if B == 0 else torch.randint(B, (1,))
        return {"ksize_factor": ksize_factor.to(device=dev, dtype=torch.int32), "angle_factor": angle_factor.to(device=dev, dtype=dt),
                "direction_factor": direction_factor.to(device=dev, dtype=dt), "idx": idx}

    def apply_transform(self, input, params, flags, transform=None):
        if isinstance(self.kernel_size, int):
            kernel_size = self.kernel_size
        else:  # one size for the batch: the one the drawn index picks
            kernel_size = int(params["ksize_factor"].tolist()[int(params["idx"][0])])
        return motion_blur(input, kernel_size=kernel_size, angle=params["angle_factor"], direction=params["direction_factor"],
                           border_type=flags["border_type"], mode=flags["resample"])
