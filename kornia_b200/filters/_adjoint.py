"""Input gradient of the one-pass separable filter without the four generic passes the autograd composition costs.
Pure host logic over two primitives that are passed in, so that the band arithmetic can be
checked on CPU with the primitives swapped for torch ops (tests/test_filter_adjoint_host_logic.py):

  forward_constant(g, kx, ky)     'same' separable correlation of g with zero ('constant') border   -- the fast kernel
  exact_adjoint(g, kx, ky)        exact adjoint of (border pad, separable correlation) applied to g  -- the generic path

For a 'constant' border the adjoint of correlation with taps k IS correlation with the flipped taps (zero outside).
For 'reflect' / 'replicate' the padded cells fold back onto the image, which only changes the outputs within
h = (K-1)/2 cells of an edge -- and those depend on the upstream gradient within 2h cells of that edge only.  So the
image-sized work runs through the fast kernel once, and four bands of h+1 rows / columns are recomputed exactly on
(3h+2)-wide crops of the upstream gradient: cost proportional to the perimeter."""
from __future__ import annotations

from typing import Callable

import torch

CONSTANT = 0  # _lib.CONSTANT


def separable_adjoint(gout: torch.Tensor, kx: torch.Tensor, ky: torch.Tensor, border: int,
                      forward_constant: Callable[[torch.Tensor, torch.Tensor, torch.Tensor], torch.Tensor],
                      exact_adjoint: Callable[[torch.Tensor, torch.Tensor, torch.Tensor], torch.Tensor]) -> torch.Tensor:
    """d/dx of ``filter2d_separable(x, kx, ky, border, padding='same')`` contracted with ``gout`` (B,C,H,W); kx (Bk,kw),
    ky (Bk,kh), odd kw == kh.  Falls back to ``exact_adjoint`` on images too small for the band argument."""
    kw, kh = kx.shape[-1], ky.shape[-1]
    h = (max(kw, kh) - 1) // 2
    H, W = gout.shape[-2:]
    crop = 3 * h + 2
    if H <= crop or W <= crop:
        return exact_adjoint(gout, kx, ky)
    gx = forward_constant(gout, kx.flip(-1), ky.flip(-1))
    if border == CONSTANT or h == 0:
        return gx
    band = h + 1
    # rows first (full width: the horizontal border is the true one), then columns (full height: corners come out exact too)
    gx[..., :band, :] = exact_adjoint(gout[..., :crop, :].contiguous(), kx, ky)[..., :band, :]
    gx[..., H - band:, :] = exact_adjoint(gout[..., H - crop:, :].contiguous(), kx, ky)[..., crop - band:, :]
    gx[..., :, :band] = exact_adjoint(gout[..., :, :crop].contiguous(), kx, ky)[..., :, :band]
    gx[..., :, W - band:] = exact_adjoint(gout[..., :, W - crop:].contiguous(), kx, ky)[..., :, crop - band:]
    return gx
