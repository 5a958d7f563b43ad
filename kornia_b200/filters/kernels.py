"""Kernel-tap generators of the filter family (reference: kornia/filters/kernels.py:29-47,68-74,
77-120,288-333,357-398,470-528,552-585,661-715,778-838).  Tiny (B,k) tensors: kept in torch so the
taps are bit-identical to the reference's and gradients w.r.t. ``sigma`` come from autograd."""
from __future__ import annotations

import math
from typing import Optional, Union

import torch

from ..core.check import check, check_is_tensor, check_shape


def _check_kernel_size(kernel_size, min_value: int = 0, allow_even: bool = False) -> None:
    sizes = (kernel_size,) if isinstance(kernel_size, int) else kernel_size
    kind = "even or odd" if allow_even else "odd"
    for s in sizes:
        check(isinstance(s, int) and ((s % 2 == 1) or allow_even) and s > min_value,
              f"Kernel size must be an {kind} integer bigger than {min_value}. Gotcha {s} on {sizes}")


def _unpack_2d_ks(kernel_size) -> tuple[int, int]:
    if isinstance(kernel_size, int):
        return kernel_size, kernel_size
    check(len(kernel_size) == 2, "2D Kernel size should have a length of 2.")
    return int(kernel_size[0]), int(kernel_size[1])


def normalize_kernel2d(kernel: torch.Tensor) -> torch.Tensor:
    """Divide every (..., kh, kw) kernel by the sum of the absolute values of its taps."""
    check_shape(kernel, ["*", "H", "W"])
    return kernel / kernel.abs().sum(dim=-1).sum(dim=-1)[..., None, None]


def gaussian(window_size: int, sigma, *, mean=None, device=None, dtype=None) -> torch.Tensor:
    """(B, window_size) samples of exp(-(x - mean)^2 / (2 sigma^2)), each row normalised to sum 1.
    ``sigma`` is a float or a (B,1) tensor; even windows are shifted by half a tap."""
    if isinstance(sigma, float):
        sigma = torch.tensor([[sigma]], device=device, dtype=dtype)
    check_is_tensor(sigma)
    check_shape(sigma, ["B", "1"])
    mean = float(window_size // 2) if mean is None else mean
    if isinstance(mean, float):
        mean = torch.tensor([[mean]], device=sigma.device, dtype=sigma.dtype)
    check_is_tensor(mean)
    check_shape(mean, ["B", "1"])
    x = (torch.arange(window_size, device=sigma.device, dtype=sigma.dtype) - mean).expand(sigma.shape[0], -1)
    if window_size % 2 == 0:
        x = x + 0.5
    g = torch.exp(-x.pow(2.0) / (2 * sigma.pow(2.0)))
    return g / g.sum(-1, keepdim=True)


def get_gaussian_kernel1d(kernel_size: int, sigma: Union[float, torch.Tensor], force_even: bool = False, *,
                          device: Optional[torch.device] = None, dtype: Optional[torch.dtype] = None) -> torch.Tensor:
    _check_kernel_size(kernel_size, allow_even=force_even)
    return gaussian(kernel_size, sigma, device=device, dtype=dtype)


def get_gaussian_kernel2d(kernel_size, sigma, force_even: bool = False, *, device=None, dtype=None) -> torch.Tensor:
    """(B, ky, kx) outer product of the two 1-D kernels; ``sigma`` is (sigma_y, sigma_x) or (B,2)."""
    if isinstance(sigma, tuple):
        sigma = torch.tensor([sigma], device=device, dtype=dtype)
    check_is_tensor(sigma)
    check_shape(sigma, ["B", "2"])
    ky, kx = _unpack_2d_ks(kernel_size)
    col = get_gaussian_kernel1d(ky, sigma[:, 0, None], force_even, device=device, dtype=dtype)[..., None]
    row = get_gaussian_kernel1d(kx, sigma[:, 1, None], force_even, device=device, dtype=dtype)[..., None]
    return col * row.view(-1, 1, kx)


# ---------------------------------------------------------------- discrete Gaussian (modified Bessel functions)
# Polynomial approximations of I0 and I1 (Abramowitz & Stegun 9.8.1-9.8.4), for |x| < 3.75 in (x / 3.75)^2 and beyond
# in 3.75 / |x|, highest power first.
_I0_SMALL = (0.0045813, 0.0360768, 0.2659732, 1.2067492, 3.0899424, 3.5156229, 1.0)
_I0_LARGE = (0.00392377, -0.01647633, 0.02635537, -0.02057706, 0.00916281, -0.00157565, 0.00225319, 0.01328592, 0.39894228)
_I1_SMALL = (0.00032411, 0.00301532, 0.02658733, 0.15084934, 0.51498869, 0.87890594, 0.5)
_I1_LARGE = (-0.00420059, 0.01787654, -0.02895312, 0.02282967, -0.01031555, 0.00163801, -0.00362018, -0.03988024, 0.39894228)


def _horner(coeffs, y: torch.Tensor) -> torch.Tensor:
    acc = torch.full_like(y, coeffs[0])
    for c in coeffs[1:]:
        acc = c + y * acc
    return acc


def _bessel_i0(x: torch.Tensor) -> torch.Tensor:
    ax = x.abs()
    small = _horner(_I0_SMALL, (x / 3.75) * (x / 3.75))
    large = (ax.exp() / ax.sqrt()) * _horner(_I0_LARGE, 3.75 / ax)
    return torch.where(ax < 3.75, small, large)


def _bessel_i1(x: torch.Tensor) -> torch.Tensor:
    ax = x.abs()
    small = ax * _horner(_I1_SMALL, (x / 3.75) * (x / 3.75))
    large = _horner(_I1_LARGE, 3.75 / ax) * ax.exp() / ax.sqrt()
    return torch.where(ax < 3.75, small, torch.where(x < 0, -large, large))


def _bessel_in(n: int, x: torch.Tensor) -> torch.Tensor:
    """I_n(x), n >= 2, by Miller's downward recurrence I_{j-1} = I_{j+1} + (2 j / x) I_j normalised with I_0."""
    zero = torch.isclose(x, torch.zeros((), device=x.device, dtype=x.dtype))
    tox = 2.0 / torch.where(zero, torch.ones_like(x), x.abs())
    ans, bip, bi = torch.zeros_like(x), torch.zeros_like(x), torch.ones_like(x)
    for j in range(2 * (n + int(math.sqrt(40.0 * n))), 0, -1):
        bip, bi = bi, bip + j * tox * bi
        scale = torch.where(bi.abs() > 1.0e10, 1e-10, 1.0).to(x.dtype)
        ans, bi, bip = ans * scale, bi * scale, bip * scale
        if j == n:
            ans = bip
    out = ans * _bessel_i0(x) / bi
    if n % 2 == 1:
        out = torch.where(x < 0.0, -out, out)
    return torch.where(zero, torch.zeros_like(x), out)


def gaussian_discrete(window_size: int, sigma, *, device=None, dtype=None) -> torch.Tensor:
    """(B, window_size) discrete Gaussian T(n, t) = exp(-t) I_n(t), t = sigma^2, for n = -(window_size // 2) ...
    window_size // 2, each row normalised to sum 1.  ``sigma`` is a float or a (B, 1) tensor."""
    if isinstance(sigma, float):
        sigma = torch.tensor([[sigma]], device=device, dtype=dtype)
    check_is_tensor(sigma)
    check_shape(sigma, ["B", "1"])
    t = sigma * sigma
    half = int(window_size // 2)
    orders = [_bessel_i0(t), _bessel_i1(t)] + [_bessel_in(n, t) for n in range(2, half + 1)]
    out = torch.cat(orders[:0:-1] + orders, -1) * t.exp()
    return out / out.sum(-1, keepdim=True)


def get_gaussian_discrete_kernel1d(kernel_size: int, sigma: Union[float, torch.Tensor], force_even: bool = False, *,
                                   device: Optional[torch.device] = None, dtype: Optional[torch.dtype] = None) -> torch.Tensor:
    """(B, kernel_size) discrete Gaussian taps (modified Bessel functions) with the reference's name and validation; the
    angular smoothing of ``PatchDominantGradientOrientation`` is ``get_gaussian_discrete_kernel1d(5, 1.6)``."""
    _check_kernel_size(kernel_size, allow_even=force_even)
    return gaussian_discrete(kernel_size, sigma, device=device, dtype=dtype)


# ---------------------------------------------------------------- box / laplacian / derivative taps
def get_box_kernel1d(kernel_size: int, *, device=None, dtype=None) -> torch.Tensor:
    """(1, k) taps, all 1/k (an expanded scalar, as in the reference: kernels.py:299-315)."""
    return torch.tensor(1.0 / kernel_size, device=device, dtype=dtype).expand(1, kernel_size)


def get_box_kernel2d(kernel_size, *, device=None, dtype=None) -> torch.Tensor:
    """(1, ky, kx) taps, all 1/(ky*kx) (kernels.py:318-333)."""
    ky, kx = _unpack_2d_ks(kernel_size)
    return torch.tensor(1.0 / (kx * ky), device=device, dtype=dtype).expand(1, ky, kx)


def laplacian_1d(window_size: int, *, device=None, dtype: torch.dtype = torch.float32) -> torch.Tensor:
    """Ones with the middle tap set to 1 - window_size (kernels.py:288-296)."""
    taps = torch.ones(window_size, device=device, dtype=dtype)
    taps[window_size // 2] = 1 - window_size
    return taps


def get_laplacian_kernel1d(kernel_size: int, *, device=None, dtype: torch.dtype = torch.float32) -> torch.Tensor:
    _check_kernel_size(kernel_size)
    return laplacian_1d(kernel_size, device=device, dtype=dtype)


def get_laplacian_kernel2d(kernel_size, *, device=None, dtype: torch.dtype = torch.float32) -> torch.Tensor:
    """(ky, kx) ones whose centre tap makes the kernel sum to zero (kernels.py:808-838)."""
    ky, kx = _unpack_2d_ks(kernel_size)
    _check_kernel_size((ky, kx))
    taps = torch.ones((ky, kx), device=device, dtype=dtype)
    taps[ky // 2, kx // 2] = 1 - taps.sum()
    return taps


_SOBEL_X = [[-1.0, 0.0, 1.0], [-2.0, 0.0, 2.0], [-1.0, 0.0, 1.0]]
_DIFF_X = [[-0.0, 0.0, 0.0], [-1.0, 0.0, 1.0], [-0.0, 0.0, 0.0]]
_SOBEL_XX = [[-1.0, 0.0, 2.0, 0.0, -1.0], [-4.0, 0.0, 8.0, 0.0, -4.0], [-6.0, 0.0, 12.0, 0.0, -6.0],
             [-4.0, 0.0, 8.0, 0.0, -4.0], [-1.0, 0.0, 2.0, 0.0, -1.0]]
_SOBEL_XY = [[-1.0, -2.0, 0.0, 2.0, 1.0], [-2.0, -4.0, 0.0, 4.0, 2.0], [0.0, 0.0, 0.0, 0.0, 0.0],
             [2.0, 4.0, 0.0, -4.0, -2.0], [1.0, 2.0, 0.0, -2.0, -1.0]]
_DIFF_XX = [[0.0, 0.0, 0.0], [1.0, -2.0, 1.0], [0.0, 0.0, 0.0]]
_DIFF_XY = [[-1.0, 0.0, 1.0], [0.0, 0.0, 0.0], [1.0, 0.0, -1.0]]


def _first_order(taps_x, device, dtype) -> torch.Tensor:
    kx = torch.tensor(taps_x, device=device, dtype=dtype)
    return torch.stack([kx, kx.transpose(0, 1)])


def _second_order(taps_xx, taps_xy, device, dtype) -> torch.Tensor:
    gxx = torch.tensor(taps_xx, device=device, dtype=dtype)
    return torch.stack([gxx, torch.tensor(taps_xy, device=device, dtype=dtype), gxx.transpose(0, 1)])


def get_sobel_kernel2d(*, device=None, dtype=None) -> torch.Tensor:
    """(2,3,3): d/dx Sobel taps and their transpose (kernels.py:470-474)."""
    return _first_order(_SOBEL_X, device, dtype)


def get_diff_kernel2d(*, device=None, dtype=None) -> torch.Tensor:
    """(2,3,3): central differences (kernels.py:477-481)."""
    return _first_order(_DIFF_X, device, dtype)


def get_sobel_kernel2d_2nd_order(*, device=None, dtype=None) -> torch.Tensor:
    """(3,5,5): gxx, gxy, gyy (kernels.py:484-491)."""
    return _second_order(_SOBEL_XX, _SOBEL_XY, device, dtype)


def get_diff_kernel2d_2nd_order(*, device=None, dtype=None) -> torch.Tensor:
    """(3,3,3): gxx, gxy, gyy (kernels.py:494-501)."""
    return _second_order(_DIFF_XX, _DIFF_XY, device, dtype)


def get_spatial_gradient_kernel2d(mode: str, order: int, *, device=None, dtype=None) -> torch.Tensor:
    """Derivative taps for ``mode`` in {'sobel','diff'} and ``order`` in {1,2} (kernels.py:504-528)."""
    check(mode.lower() in {"sobel", "diff"}, f"Mode should be `sobel` or `diff`. Got {mode}")
    check(order in {1, 2}, f"Order should be 1 or 2. Got {order}")
    table = {("sobel", 1): get_sobel_kernel2d, ("sobel", 2): get_sobel_kernel2d_2nd_order,
             ("diff", 1): get_diff_kernel2d, ("diff", 2): get_diff_kernel2d_2nd_order}
    make = table.get((mode, order))
    if make is None:
        raise NotImplementedError(f"Not implemented for order {order} on mode {mode}")
    return make(device=device, dtype=dtype)
