"""ORACLE for the feature responses (test infrastructure, not product code): the reference's harris_response /
gftt_response / hessian_response (kornia/feature/responses.py:39-282) restated with the same ATen calls, on top of the
spatial_gradient / gaussian_blur2d restatements of oracle/kornia_restated.py.  It runs on whatever device its arguments
live on; on CUDA it is the reference composition tools/bench_responses.py times the fused kernels against."""
from __future__ import annotations

import torch

from oracle import kornia_restated as R


def _scaled(scores, sigmas):
    if sigmas is not None:
        scores = scores * sigmas.pow(4).view(-1, 1, 1, 1)
    return scores


def _structure(input, grads_mode):
    gradients = R.spatial_gradient(input, grads_mode)
    dx, dy = gradients[:, :, 0], gradients[:, :, 1]
    dx2 = R.gaussian_blur2d(dx**2, (7, 7), (1.0, 1.0))
    dy2 = R.gaussian_blur2d(dy**2, (7, 7), (1.0, 1.0))
    dxy = R.gaussian_blur2d(dx * dy, (7, 7), (1.0, 1.0))
    return dx2 * dy2 - dxy * dxy, dx2 + dy2


def harris_response(input, k=0.04, grads_mode="sobel", sigmas=None):
    det_m, trace_m = _structure(input, grads_mode)
    return _scaled(det_m - k * (trace_m**2), sigmas)


def gftt_response(input, grads_mode="sobel", sigmas=None):
    det_m, trace_m = _structure(input, grads_mode)
    e1 = 0.5 * (trace_m + torch.sqrt((trace_m**2 - 4 * det_m).abs()))
    e2 = 0.5 * (trace_m - torch.sqrt((trace_m**2 - 4 * det_m).abs()))
    return _scaled(torch.min(e1, e2), sigmas)


def hessian_response(input, grads_mode="sobel", sigmas=None):
    gradients = R.spatial_gradient(input, grads_mode, 2)
    dxx, dxy, dyy = gradients[:, :, 0], gradients[:, :, 1], gradients[:, :, 2]
    return _scaled(dxx * dyy - dxy**2, sigmas)
