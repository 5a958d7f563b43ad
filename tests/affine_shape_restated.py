"""Plain-torch restatement of kornia/feature/affine_shape.py PatchAffineShapeEstimator.forward and
LAFAffineShapeEstimator.forward (no kornia_b200 code), organised differently from the reference: the LAF arithmetic works
on the four entries of each 2 x 2 linear part as separate tensors, the moments are single means over both axes, the
rotation is written out entry by entry, and the 2 x 2 inverse is ``torch.linalg.inv``.  The patches come from
tests/patches_restated.py, the gradients from tests/sift_restated.py."""
import math

import torch

import patches_restated as PR
import sift_restated as SR

PI = SR.PI


def weighting(P):
    return SR.gaussian2d(P, float(P) / math.sqrt(2.0))


def patch_shape(x, w, eps):
    """(B, 1, 3) normalised second-moment shapes of (B, 1, P, P) patches ``x`` under the P x P weighting ``w``."""
    g = SR.gradient(x, SR.SOBEL) * w
    gx, gy = g[:, :, 0], g[:, :, 1]
    m = torch.stack([(gx * gx).mean(dim=(-2, -1)), (gx * gy).mean(dim=(-2, -1)), (gy * gy).mean(dim=(-2, -1))], -1)  # (B, 1, 3)
    bad = ((m < eps).sum(-1, keepdim=True) >= 2).to(m.dtype)
    m = m * (1.0 - bad) + torch.tensor([1.0, 0.0, 1.0], dtype=m.dtype) * bad
    return m / m.max(-1, keepdim=True).values


def _entries(laf):
    return laf[..., 0, 0], laf[..., 0, 1], laf[..., 1, 0], laf[..., 1, 1]


def _scale(a, b, c, d):
    return (a * d - c * b + 1e-10).abs().sqrt()


def _laf(a, b, c, d, centre):
    return torch.cat([torch.stack([torch.stack([a, b], -1), torch.stack([c, d], -1)], -2), centre], -1)


def upright(laf):
    a, b, c, d = _entries(laf)
    s = _scale(a, b, c, d)
    n = (b * b + a * a).sqrt() + 1e-9
    return _laf(s * (n / s), s * torch.zeros_like(s), s * ((d * b + c * a) / (n * s)), s * (s / n), laf[..., :, 2:3])


def _deg(t):
    return 180.0 * t / PI


def laf_shape(img, laf, PS, eps, preserve):
    """(B, N, 2, 3) LAFs with the affine shape estimated on ``img``."""
    B, N = laf.shape[:2]
    patches = PR.extract(img, upright(laf), PS, True, True).view(-1, 1, PS, PS)
    e = patch_shape(patches, weighting(PS), eps).view(B, N, 3)
    a11, a22 = e[..., 0].abs().sqrt(), e[..., 2].abs().sqrt()
    a21 = e[..., 1] / (a11 + a22).clamp(1e-9)
    low = torch.stack([torch.stack([a11, torch.zeros_like(a11)], -1), torch.stack([a21, a22], -1)], -2)
    inv = torch.linalg.inv(low)
    a, b, c, d = _entries(inv)
    coef = _scale(*_entries(laf)) / _scale(a, b, c, d)
    a, b, c, d = coef * a, coef * b, coef * c, coef * d
    if preserve:
        ang = _deg(torch.atan2(laf[..., 0, 1], laf[..., 0, 0])) - _deg(torch.atan2(b, a))
        rad = ang * PI / 180.0
        co, si = torch.cos(rad), torch.sin(rad)
        a, b, c, d = a * co - b * si, a * si + b * co, c * co - d * si, c * si + d * co
    return _laf(a, b, c, d, laf[..., :, 2:3])
