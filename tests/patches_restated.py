"""Plain-torch restatement of the reference's extract_patches_from_pyramid / extract_patches_simple (kornia/feature/laf.py),
organised differently from the reference: every level is sampled once for all B * N patches (each patch reads its own
image), and each patch keeps the level its scale picked.  The arithmetic is the reference's op for op, so it reproduces the
goldens; ``pyrdown`` is the oracle's."""
import torch
import torch.nn.functional as F

from oracle.kornia_restated import pyrdown


def _coef(h, w, dtype, inverse):
    m = float(min(h - 1, w - 1))
    c = torch.ones(1, 1, 2, 3, dtype=dtype)
    c = c / m if inverse else c * m
    c[0, 0, 0, 2] = 1.0 / float(w - 1) if inverse else float(w - 1)
    c[0, 0, 1, 2] = 1.0 / float(h - 1) if inverse else float(h - 1)
    return c


def _sample(level, nlaf, PS):
    """(B * N, C, PS, PS) patches of every LAF on ``level`` (batch b of the LAFs reads image b)."""
    B, N = nlaf.shape[:2]
    _, C, h, w = level.shape
    theta = (_coef(h, w, nlaf.dtype, False).to(nlaf.device) * nlaf).reshape(B * N, 2, 3)
    grid = F.affine_grid(theta, [B * N, C, PS, PS], align_corners=False)
    gx = 2.0 * grid[..., 0] / float(w - 1) - 1.0
    gy = 2.0 * grid[..., 1] / float(h - 1) - 1.0
    src = level[:B].repeat_interleave(N, 0)
    return F.grid_sample(src, torch.stack([gx, gy], -1), padding_mode="border", align_corners=False)


def extract(img, laf, PS, normalize, pyramid):
    B, N = laf.shape[:2]
    _, C, h, w = img.shape
    nlaf = _coef(h, w, laf.dtype, True).to(laf.device) * laf if normalize else laf
    if not pyramid:
        return _sample(img, nlaf, PS).view(B, N, C, PS, PS)
    d = _coef(h, w, laf.dtype, False).to(laf.device) * nlaf
    scale = 2.0 * (d[..., 0, 0] * d[..., 1, 1] - d[..., 1, 0] * d[..., 0, 1] + 1e-10).abs().sqrt() / float(PS)
    top = min(h, w) // PS
    idx = scale.log2().clamp(min=0.0, max=max(0, top - 1)).long().view(B * N, 1, 1, 1)
    out = torch.zeros(B * N, C, PS, PS, dtype=laf.dtype)
    level = img
    for lv in range(max(1, top)):
        if lv > 0:
            level = pyrdown(level)
            if min(level.shape[-2:]) < PS:
                break
        out = torch.where(idx == lv, _sample(level, nlaf, PS).to(laf.dtype), out)
    return out.view(B, N, C, PS, PS)
