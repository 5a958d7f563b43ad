"""Drop-in ``harris_response``, ``gftt_response``, ``hessian_response`` and their modules (reference:
kornia/feature/responses.py:39-282,378-467).

The reference computes the structure tensor with ``spatial_gradient``, three products and three
``gaussian_blur2d((7, 7), (1.0, 1.0))`` calls, then 7 (Harris) or ~17 (Shi-Tomasi) elementwise kernels; the Hessian
response is ``spatial_gradient(order=2)`` and three more.  Inference-style calls (fp32 CUDA input, no gradient, rows a
multiple of 4 floats) run as ONE CUDA kernel that reads the image once and writes the response, bit-identical to
``_composed_*``: the reference's op sequence over this library's ``spatial_gradient`` and ``gaussian_blur2d``, which
is also the differentiable path and what every other call runs."""
from __future__ import annotations

from typing import Optional, Union

import torch
from torch import nn

from .. import _lib, _ops
from ..core.check import check_shape
from ..filters.gaussian import _constant_taps, gaussian_blur2d
from ..filters.sobel import _host_taps, spatial_gradient

__all__ = ["harris_response", "gftt_response", "hessian_response", "CornerHarris", "CornerGFTT", "BlobHessian"]


def _check_sigmas(input: torch.Tensor, sigmas) -> None:
    if sigmas is not None:
        if not isinstance(sigmas, torch.Tensor):
            raise TypeError(f"sigmas type is not a torch.Tensor. Got {type(sigmas)}")
        if (not len(sigmas.shape) == 1) or (sigmas.size(0) != input.size(0)):
            raise ValueError(f"Invalid sigmas shape, we expect B == input.size(0). Got: {sigmas.shape}")


def _structure_tensor(input, grads_mode):
    """responses.py:107-118: the blurred products and det / trace of M."""
    gradients = spatial_gradient(input, grads_mode)
    dx = gradients[:, :, 0]
    dy = gradients[:, :, 1]
    dx2 = gaussian_blur2d(dx**2, (7, 7), (1.0, 1.0))
    dy2 = gaussian_blur2d(dy**2, (7, 7), (1.0, 1.0))
    dxy = gaussian_blur2d(dx * dy, (7, 7), (1.0, 1.0))
    det_m = dx2 * dy2 - dxy * dxy
    trace_m = dx2 + dy2
    return det_m, trace_m


def _scaled(scores, sigmas):
    if sigmas is not None:
        scores = scores * sigmas.pow(4).view(-1, 1, 1, 1)
    return scores


def _composed_harris(input, k, grads_mode, sigmas):
    det_m, trace_m = _structure_tensor(input, grads_mode)
    return _scaled(det_m - k * (trace_m**2), sigmas)


def _composed_gftt(input, grads_mode, sigmas):
    det_m, trace_m = _structure_tensor(input, grads_mode)
    e1 = 0.5 * (trace_m + torch.sqrt((trace_m**2 - 4 * det_m).abs()))
    e2 = 0.5 * (trace_m - torch.sqrt((trace_m**2 - 4 * det_m).abs()))
    return _scaled(torch.min(e1, e2), sigmas)


def _composed_hessian(input, grads_mode, sigmas):
    gradients = spatial_gradient(input, grads_mode, 2)
    dxx = gradients[:, :, 0]
    dxy = gradients[:, :, 1]
    dyy = gradients[:, :, 2]
    return _scaled(dxx * dyy - dxy**2, sigmas)


def _fused(input, kind, grads_mode, sigmas, k=0.0):
    """The one-kernel response, or None when the call takes the composition: a gradient is needed, the input is not fp32
    CUDA with W % 4 == 0, or an operand would change the result's dtype through type promotion (``sigmas`` other than a
    (B,) fp32 tensor on the input's device, ``k`` other than a number or a 0-d floating tensor)."""
    if not isinstance(input, torch.Tensor) or input.dim() != 4:
        return None
    if not torch.compiler.is_compiling():
        _ops._require_cuda(input, "input")
    B, C, H, W = input.shape
    if sigmas is not None and not isinstance(sigmas, torch.Tensor):  # gftt_response: the composition raises what the reference raises
        return None
    # every tensor operand, wherever it lives, before k is turned into a kernel argument: a gradient takes the composition
    needs_grad = torch.is_grad_enabled() and any(isinstance(t, torch.Tensor) and t.requires_grad for t in (input, k, sigmas))
    if (input.dtype != torch.float32 or not input.is_cuda or needs_grad or W % 4 != 0 or input.numel() == 0
            or (kind != _ops.HESSIAN and min(H, W) <= 3)):
        return None
    k_tensor = None
    if isinstance(k, torch.Tensor):
        if k.dim() != 0 or not k.is_floating_point():
            return None
        if k.device == input.device:
            k_tensor = k if k.dtype == torch.float32 else k.float()  # torch's mul rounds its operand to fp32 the same way
            k = 0.0
        elif k.device.type == "cpu":
            k = float(k)  # a CPU scalar: torch reads it on the host as well
        else:
            return None
    elif isinstance(k, bool) or not isinstance(k, (int, float)):
        return None
    if sigmas is not None and not (sigmas.dtype == torch.float32 and sigmas.device == input.device and tuple(sigmas.shape) == (B,)):
        return None
    taps, _, stencil_k = _host_taps(grads_mode, 2 if kind == _ops.HESSIAN else 1, True, input.dtype)
    blur = None if kind == _ops.HESSIAN else _constant_taps((7, 7), (1.0, 1.0), True, input.device, input.dtype)[0]
    s4 = None if sigmas is None else sigmas.pow(4)
    try:
        return _ops.ops.feature_response_fwd(input, list(taps), stencil_k, blur, float(k), k_tensor, s4, kind)
    except _lib.Unsupported:
        return None


def harris_response(
    input: torch.Tensor,
    k: Union[torch.Tensor, float] = 0.04,
    grads_mode: str = "sobel",
    sigmas: Optional[torch.Tensor] = None,
) -> torch.Tensor:
    """Harris cornerness ``det(M) - k trace(M)^2`` of every channel of ``input`` (B,C,H,W), where M is the structure
    tensor of ``grads_mode`` ('sobel' or 'diff') derivatives blurred by a 7x7 Gaussian of sigma 1; the response of
    sample b is multiplied by ``sigmas[b]**4`` when ``sigmas`` (B,) is given."""
    check_shape(input, ["B", "C", "H", "W"])
    _check_sigmas(input, sigmas)
    out = _fused(input, _ops.HARRIS, grads_mode, sigmas, k)
    return out if out is not None else _composed_harris(input, k, grads_mode, sigmas)


def gftt_response(input: torch.Tensor, grads_mode: str = "sobel", sigmas: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Shi-Tomasi cornerness ``min(eig(M))`` of every channel of ``input`` (B,C,H,W), M as in :func:`harris_response`.
    ``sigmas`` is not validated, as in the reference."""
    check_shape(input, ["B", "C", "H", "W"])
    out = _fused(input, _ops.GFTT, grads_mode, sigmas)
    return out if out is not None else _composed_gftt(input, grads_mode, sigmas)


def hessian_response(input: torch.Tensor, grads_mode: str = "sobel", sigmas: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Determinant of the Hessian ``dxx dyy - dxy^2`` of every channel of ``input`` (B,C,H,W), from the second-order
    ``grads_mode`` stencils; times ``sigmas[b]**4`` when ``sigmas`` (B,) is given."""
    check_shape(input, ["B", "C", "H", "W"])
    _check_sigmas(input, sigmas)
    out = _fused(input, _ops.HESSIAN, grads_mode, sigmas)
    return out if out is not None else _composed_hessian(input, grads_mode, sigmas)


class CornerHarris(nn.Module):
    """Module form of :func:`harris_response` (same constructor as the reference's; ``k`` is a buffer)."""

    k: torch.Tensor

    def __init__(self, k: Union[float, torch.Tensor], grads_mode: str = "sobel") -> None:
        super().__init__()
        if isinstance(k, float):
            self.register_buffer("k", torch.tensor(k))
        else:
            self.register_buffer("k", k)
        self.grads_mode: str = grads_mode

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}(k={self.k}, grads_mode={self.grads_mode})"

    def forward(self, input: torch.Tensor, sigmas: Optional[torch.Tensor] = None) -> torch.Tensor:
        return harris_response(input, self.k, self.grads_mode, sigmas)


class CornerGFTT(nn.Module):
    """Module form of :func:`gftt_response` (same constructor as the reference's)."""

    def __init__(self, grads_mode: str = "sobel") -> None:
        super().__init__()
        self.grads_mode: str = grads_mode

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}(grads_mode={self.grads_mode})"

    def forward(self, input: torch.Tensor, sigmas: Optional[torch.Tensor] = None) -> torch.Tensor:
        return gftt_response(input, self.grads_mode, sigmas)


class BlobHessian(nn.Module):
    """Module form of :func:`hessian_response` (same constructor as the reference's)."""

    def __init__(self, grads_mode: str = "sobel") -> None:
        super().__init__()
        self.grads_mode: str = grads_mode

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}(grads_mode={self.grads_mode})"

    def forward(self, input: torch.Tensor, sigmas: Optional[torch.Tensor] = None) -> torch.Tensor:
        return hessian_response(input, self.grads_mode, sigmas)
