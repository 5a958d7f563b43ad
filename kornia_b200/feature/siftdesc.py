"""Drop-in ``SIFTDescriptor``, ``sift_describe``, ``get_sift_pooling_kernel`` and ``get_sift_bin_ksize_stride_pad``
(reference: kornia/feature/siftdesc.py).

The reference describes an (N, 1, P, P) patch stack with about 100 ATen kernels, each reading or writing a full
N x P x P plane: the 'diff' gradient, about 20 elementwise passes, then per angular bin two one-hot masks, casts,
products, an add and a strided ``nn.Conv2d`` pooling, and finally three ``F.normalize`` calls, a clamp and a sqrt.

An fp32 CUDA call whose configuration is in the kernel's envelope (patch_size <= 64, num_ang_bins * num_spatial_bins^2
<= 1024), whose patches have column stride 1 and that needs no gradient runs as ONE CUDA kernel (csrc/siftdesc.cuh)
that reads each patch once and writes its descriptor.  "Needs no gradient" means grad mode is off, or neither the input,
``gk`` nor ``pk.weight`` requires grad.  ``pk.weight`` is a trainable parameter, as in the reference, so a
default-constructed module called in grad mode runs the composition; ``torch.inference_mode()``, ``torch.no_grad()`` or
``descriptor.requires_grad_(False)`` selects the kernel.  The kernel reads the module's current ``gk`` and
``pk.weight``, so an edited or loaded state is honoured.

Every other call runs ``_composed_sift``: the reference's op sequence over this library's ``spatial_gradient``, with the
pooling taken as strided windows and a product with ``pk.weight`` (not a convolution cuDNN runs in TF32 by default), so
the gradients with respect to the input and ``pk.weight`` are the reference's.  It is also the differentiable path."""
from __future__ import annotations

import math
from typing import Tuple

import torch
import torch.nn.functional as F
from torch import nn

from .. import _ops
from ..core.check import check_shape
from ..filters.kernels import get_gaussian_kernel2d
from ..filters.sobel import spatial_gradient

__all__ = ["SIFTDescriptor", "sift_describe", "get_sift_pooling_kernel", "get_sift_bin_ksize_stride_pad"]

# kornia's pi is a 0-d fp32 tensor: 2 * pi is the fp32-rounded value even in fp64 evaluations
pi = torch.tensor(3.14159265358979323846)

MAX_PATCH_SIZE = 64  # the fused kernels' envelope (csrc/siftdesc.cuh)
MAX_DESCRIPTOR_SIZE = 1024


def get_sift_pooling_kernel(ksize: int = 25) -> torch.Tensor:
    """(ksize, ksize) bilinear pooling weights of one spatial bin: the outer product of a triangle over the window,
    divided by (ksize / 2)^2."""
    half = float(ksize) / 2.0
    tri = half - (torch.arange(ksize).float() + 0.5 - half).abs()
    return torch.outer(tri, tri) / (half**2)


def get_sift_bin_ksize_stride_pad(patch_size: int, num_spatial_bins: int) -> Tuple[int, int, int]:
    """(ksize, stride, pad) of the spatial-bin pooling; raises ``ValueError`` when it does not give ``num_spatial_bins``
    bins per side."""
    ksize: int = 2 * int(patch_size / (num_spatial_bins + 1))
    stride: int = patch_size // num_spatial_bins
    pad: int = ksize // 4
    if (patch_size + 2 * pad - (ksize - 1) - 1) // stride + 1 != num_spatial_bins:
        raise ValueError(
            f"Patch size {patch_size} is incompatible with             requested number of spatial bins"
            f" {num_spatial_bins}             for SIFT descriptor. Usually it happens when patch size is too small     "
            "       for num_spatial_bins specified"
        )
    return ksize, stride, pad


def _pool(planes: torch.Tensor, weight: torch.Tensor, stride: int, pad: int) -> torch.Tensor:
    """The strided, zero-padded K x K correlation of every (N, A, P, P) plane with ``weight`` (1, 1, K, K), taken
    exactly: (N, A, S, S).  The windows are strided views of the padded planes and one fp32 matrix-vector product sums
    them (``F.unfold`` would launch one im2col kernel per plane).  The product reads a copy of the windows, N·A·S²·K²
    floats (1.05 GB at N = 8000 for SIFTDescriptor(41), against 0.43 GB for the reference's eight per-bin planes), which
    grad mode keeps for the backward."""
    K = weight.shape[-1]
    win = F.pad(planes, (pad, pad, pad, pad)).unfold(2, K, stride).unfold(3, K, stride)  # (N, A, S, S, K, K)
    return torch.matmul(win.reshape(win.shape[:4] + (K * K,)), weight.reshape(K * K))


class SIFTDescriptor(nn.Module):
    r"""SIFT descriptors of (B, 1, patch_size, patch_size) patches: (B, num_ang_bins * num_spatial_bins ** 2).

    Args:
        patch_size: input patch size in pixels.
        num_ang_bins: number of angular bins.
        num_spatial_bins: number of spatial bins per side.
        rootsift: if ``True``, RootSIFT (Arandjelović et al., 2012) is computed.
        clipval: clipping value to reduce single-bin dominance.

    An fp32 CUDA call that needs no gradient runs one fused kernel (see the module docstring); a default module in grad
    mode has a trainable ``pk.weight`` and runs the differentiable composition.
    """

    def __repr__(self) -> str:
        return (
            f"{self.__class__.__name__}("
            f"num_ang_bins={self.num_ang_bins}, "
            f"num_spatial_bins={self.num_spatial_bins}, "
            f"patch_size={self.patch_size}, "
            f"rootsift={self.rootsift}, "
            f"clipval={self.clipval})"
        )

    def __init__(
        self,
        patch_size: int = 41,
        num_ang_bins: int = 8,
        num_spatial_bins: int = 4,
        rootsift: bool = True,
        clipval: float = 0.2,
    ) -> None:
        super().__init__()
        self.eps = 1e-10
        self.num_ang_bins = num_ang_bins
        self.num_spatial_bins = num_spatial_bins
        self.clipval = clipval
        self.rootsift = rootsift
        self.patch_size = patch_size
        sigma: float = float(patch_size) / math.sqrt(2.0)
        self.gk = get_gaussian_kernel2d((patch_size, patch_size), (sigma, sigma), True)
        (self.bin_ksize, self.bin_stride, self.pad) = get_sift_bin_ksize_stride_pad(patch_size, num_spatial_bins)
        nw = get_sift_pooling_kernel(ksize=self.bin_ksize).float()
        self.pk = nn.Conv2d(1, 1, kernel_size=(nw.size(0), nw.size(1)), stride=(self.bin_stride, self.bin_stride),
                            padding=(self.pad, self.pad), bias=False)
        self.pk.weight.data.copy_(nw.reshape(1, 1, nw.size(0), nw.size(1)))
        self._gk_device = None  # (host snapshot of gk, its fp32 copy on a device): gk is a plain attribute kept where it is

    def get_pooling_kernel(self) -> torch.Tensor:
        """The spatial pooling kernel (``pk.weight``), detached."""
        return self.pk.weight.detach()

    def get_weighting_kernel(self) -> torch.Tensor:
        """The Gaussian weighting kernel (``gk``), detached."""
        return self.gk.detach()

    def _fused_ok(self, input: torch.Tensor) -> bool:
        w = self.pk.weight
        needs_grad = torch.is_grad_enabled() and (input.requires_grad or w.requires_grad or self.gk.requires_grad)
        # N = 0 runs the composition, which raises the reference's error for an empty stack
        return (input.shape[0] > 0 and input.dtype == torch.float32 and input.is_cuda and not needs_grad and self.patch_size <= MAX_PATCH_SIZE
                and self.num_ang_bins * self.num_spatial_bins**2 <= MAX_DESCRIPTOR_SIZE and (input.shape[-1] == 1 or input.stride(-1) == 1)
                and w.shape[-1] == w.shape[-2] == self.bin_ksize and tuple(self.gk.shape[-2:]) == (self.patch_size, self.patch_size))

    def _gk_on(self, device: torch.device) -> torch.Tensor:
        """``gk`` as a contiguous fp32 tensor on ``device``.  A ``gk`` already there is used as is; a host ``gk`` (where the
        reference keeps it) is copied once and copied again only when its values differ from the snapshot the copy was
        made from.  Comparing values rather than version counters also covers inference tensors, which have none (a
        module built under ``torch.inference_mode()``)."""
        gk = self.gk
        if gk.device == device and gk.dtype == torch.float32:
            return gk.detach().contiguous()
        if torch.compiler.is_compiling():
            return gk.to(device=device, dtype=torch.float32)
        hit = self._gk_device
        if hit is None or hit[1].device != device or hit[0].shape != gk.shape or not torch.equal(hit[0], gk.detach()):
            hit = self._gk_device = (gk.detach().clone(), gk.detach().to(device=device, dtype=torch.float32).contiguous())
        return hit[1]

    def forward(self, input: torch.Tensor) -> torch.Tensor:
        check_shape(input, ["B", "1", f"{self.patch_size}", f"{self.patch_size}"])
        self.pk = self.pk.to(input.dtype).to(input.device)
        if self._fused_ok(input):
            return _ops.ops.sift_describe_fwd(input, self._gk_on(input.device), self.pk.weight, self.num_ang_bins, self.num_spatial_bins,
                                              self.bin_stride, self.pad, bool(self.rootsift), float(self.clipval), float(self.eps))
        return _composed_sift(self, input)


def _composed_sift(m: SIFTDescriptor, input: torch.Tensor) -> torch.Tensor:
    """siftdesc.py forward: the reference's op sequence, with the pooling taken exactly."""
    B: int = input.shape[0]
    grads = spatial_gradient(input, "diff")
    gx = grads[:, :, 0]
    gy = grads[:, :, 1]
    mag = torch.sqrt(gx * gx + gy * gy + m.eps)
    ori = torch.atan2(gy, gx + m.eps) + 2.0 * pi
    mag = mag * m.gk.expand_as(mag).type_as(mag).to(mag.device)
    o_big = float(m.num_ang_bins) * ori / (2.0 * pi)
    bo0_big_ = torch.floor(o_big)
    wo1_big_ = o_big - bo0_big_
    bo0_big = bo0_big_ % m.num_ang_bins
    bo1_big = (bo0_big + 1) % m.num_ang_bins
    wo0_big = (1.0 - wo1_big_) * mag
    wo1_big = wo1_big_ * mag
    planes = torch.cat([(bo0_big == i).to(input.dtype) * wo0_big + (bo1_big == i).to(input.dtype) * wo1_big
                        for i in range(m.num_ang_bins)], 1)
    ang_bins = _pool(planes, m.pk.weight, m.bin_stride, m.pad).view(B, -1)
    ang_bins = F.normalize(ang_bins, p=2)
    ang_bins = torch.clamp(ang_bins, 0.0, float(m.clipval))
    ang_bins = F.normalize(ang_bins, p=2)
    if m.rootsift:
        ang_bins = torch.sqrt(F.normalize(ang_bins, p=1) + m.eps)
    return ang_bins


def sift_describe(
    input: torch.Tensor,
    patch_size: int = 41,
    num_ang_bins: int = 8,
    num_spatial_bins: int = 4,
    rootsift: bool = True,
    clipval: float = 0.2,
) -> torch.Tensor:
    r"""SIFT descriptors of ``input`` with a fresh :class:`SIFTDescriptor`; see there for details."""
    return SIFTDescriptor(patch_size, num_ang_bins, num_spatial_bins, rootsift, clipval)(input)
