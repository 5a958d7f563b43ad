"""Plain-torch restatement of kornia/feature/siftdesc.py SIFTDescriptor.forward and kornia/feature/orientation.py
PatchDominantGradientOrientation.forward (no kornia_b200 code): the reference's op sequence, with the 3 x 3 gradients as
the sum of every tap (zero taps included, so a non-finite texel makes 0 * x = NaN in its neighbours' gradients, as the
reference's convolution does) over a replicate border, and the pooling and the circular smoothing as CPU convolutions."""
import math

import torch
import torch.nn.functional as F

PI = torch.tensor(3.14159265358979323846)  # kornia's pi: a 0-d fp32 tensor

DIFF = ([[0.0, 0.0, 0.0], [-0.5, 0.0, 0.5], [0.0, 0.0, 0.0]], [[0.0, -0.5, 0.0], [0.0, 0.0, 0.0], [0.0, 0.5, 0.0]])
SOBEL = ([[-0.125, 0.0, 0.125], [-0.25, 0.0, 0.25], [-0.125, 0.0, 0.125]], [[-0.125, -0.25, -0.125], [0.0, 0.0, 0.0], [0.125, 0.25, 0.125]])


def gradient(x, stencil):
    """(B, 1, 2, P, P): every tap of the normalised 3 x 3 stencil over a replicate border."""
    P = x.shape[-1]
    xp = F.pad(x, (1, 1, 1, 1), mode="replicate")
    out = []
    for taps in stencil:
        acc = torch.zeros_like(x)
        for r in range(3):
            for c in range(3):
                acc = acc + taps[r][c] * xp[..., r:r + P, c:c + P]
        out.append(acc)
    return torch.stack(out, 2)


def gaussian2d(P, sigma, dtype=torch.float32):
    x = torch.arange(P, dtype=dtype) - P // 2
    if P % 2 == 0:
        x = x + 0.5
    g = torch.exp(-x.pow(2.0) / (2 * sigma**2))
    g = g / g.sum()
    return (g[:, None] * g[None, :])[None]


def _bins(mag, ori_big, n, dtype):
    b0_ = torch.floor(ori_big)
    w1_ = ori_big - b0_
    b0 = b0_ % n
    b1 = (b0 + 1) % n
    w0 = (1.0 - w1_) * mag
    w1 = w1_ * mag
    return [(b0 == i).to(dtype) * w0 + (b1 == i).to(dtype) * w1 for i in range(n)]


def sift(x, gk, pk, n_ang, n_sp, stride, pad, rootsift, clipval, eps=1e-10):
    B = x.shape[0]
    g = gradient(x, DIFF)
    gx, gy = g[:, :, 0], g[:, :, 1]
    mag = torch.sqrt(gx * gx + gy * gy + eps)
    ori = torch.atan2(gy, gx + eps) + 2.0 * PI
    mag = mag * gk.expand_as(mag).to(mag.dtype)
    o_big = float(n_ang) * ori / (2.0 * PI)
    planes = _bins(mag, o_big, n_ang, x.dtype)
    w = pk.to(x.dtype)
    out = torch.cat([F.conv2d(p, w, stride=stride, padding=pad) for p in planes], 1).view(B, -1)
    out = F.normalize(out, p=2)
    out = torch.clamp(out, 0.0, float(clipval))
    out = F.normalize(out, p=2)
    if rootsift:
        out = torch.sqrt(F.normalize(out, p=1) + eps)
    return out


def orientation(x, weighting, smooth, n, eps=1e-8, return_hist=False):
    g = gradient(x, SOBEL)
    gx, gy = g[:, :, 0], g[:, :, 1]
    mag = torch.sqrt(gx * gx + gy * gy + eps) * weighting.to(x.dtype)
    ori = torch.atan2(gy, gx + eps) + 2.0 * PI
    o_big = float(n) * (ori + 1.0 * PI) / (2.0 * PI)
    hist = torch.cat([p.mean((-2, -1), keepdim=True) for p in _bins(mag, o_big, n, x.dtype)], 1).view(-1, 1, n)
    hist = F.conv1d(F.pad(hist, (2, 2), mode="circular"), smooth.to(x.dtype).view(1, 1, 5)).view(-1, n)
    values, idx = hist.max(1)
    left = torch.gather(hist, 1, ((n + idx - 1) % n).reshape(-1, 1)).reshape(-1)
    right = torch.gather(hist, 1, ((idx + 1) % n).reshape(-1, 1)).reshape(-1)
    c_subpix = 0.5 * (left - right) / (left + right - 2.0 * values)
    angle = -((2.0 * PI * (idx.to(x.dtype) + c_subpix) / float(n)) - PI)
    return (angle, hist) if return_hist else angle


def sift_params(P, S):
    ksize = 2 * int(P / (S + 1))
    return ksize, P // S, ksize // 4


def sift_pooling_kernel(ksize):
    half = ksize / 2.0
    tri = half - (torch.arange(ksize).float() + 0.5 - half).abs()
    return (torch.outer(tri, tri) / half**2).view(1, 1, ksize, ksize)


def sift_gk(P):
    return gaussian2d(P, float(P) / math.sqrt(2.0))
