"""Golden vectors for non-maximum suppression: nms2d, nms3d and nms3d_minmax of the UNMODIFIED reference run on CPU fp32.
Needs a checkout of the reference (make_golden.import_reference):

    python tests/golden/make_golden_nms.py    ->  tests/golden/nms.npz (shards nms.<k>.npz)

Inputs: quantised texels (ties and plateaus are common), a smooth image, and special texels (NaN, +-Inf, -0, subnormals)
with negative isolated peaks.  nms2d runs at K = 3, 5, 7, 9 and 15 with both ``mask_only`` values, also on images with
H or W below K, a 1 x 1 image and odd widths; nms3d at (3, 3, 3) with both values; nms3d_minmax.  Even and non-square
2-D sizes and a (5, 5, 5) 3-D size record the reference's error type and message instead of outputs.
"""
from __future__ import annotations

import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import Bag, import_reference, smooth_image  # noqa: E402


def quantised(shape, gen):
    return torch.round(torch.rand(shape, generator=gen) * 6) / 4 - 0.5


def specials(shape, gen):
    x = torch.rand(shape, generator=gen) * 2 - 1
    flat = x.view(-1)
    vals = torch.tensor([float("nan"), float("inf"), float("-inf"), -0.0, 1e-40, -1e-41, 2e-45, 0.0])
    idx = torch.randperm(flat.numel(), generator=gen)[: max(8, flat.numel() // 40)]
    flat[idx] = vals[torch.arange(idx.numel()) % vals.numel()]
    return x


def negative_peaks(shape, gen):
    """A negative plateau with isolated negative peaks and subnormal bumps: the explicit forms keep the peaks, the general
    form (0 joins the neighbour set) does not."""
    x = torch.full(shape, -1.0)
    flat = x.view(-1)
    idx = torch.randperm(flat.numel(), generator=gen)[: max(2, flat.numel() // 60)]
    flat[idx] = -0.25
    flat[idx[::3]] = 1e-40
    return x


def main():
    import_reference()
    from kornia.geometry.subpix import nms2d, nms3d, nms3d_minmax

    torch.set_num_threads(1)
    gen = torch.Generator().manual_seed(2026)
    bag = Bag()
    images = {
        "quant": quantised((2, 3, 24, 29), gen),
        "smooth": smooth_image(1, 2, 26, 31, gen),
        "special": specials((1, 2, 20, 23), gen),
        "negpeaks": negative_peaks((1, 1, 22, 25), gen),
        "short": quantised((1, 2, 5, 40), gen),     # H below 7, 9 and 15
        "narrow": specials((1, 1, 33, 6), gen),     # W below 7, 9 and 15
        "one": torch.tensor([[[[0.5]]]]),
        "two": quantised((1, 1, 2, 3), gen),
    }
    for k in (3, 5, 7, 9, 15):
        for img in images:
            for mask_only in (True, False):
                out = nms2d(images[img], (k, k), mask_only)
                bag.add(f"nms2d_k{k}_{img}_{'mask' if mask_only else 'values'}", "nms2d", {"input": images[img]},
                        {"kernel_size": [k, k], "mask_only": mask_only}, {"out": out})
    vols = {
        "quant": quantised((2, 2, 5, 17, 21), gen),
        "special": specials((1, 2, 4, 15, 19), gen),
        "tiny": quantised((1, 1, 2, 5, 5), gen),
        "one": torch.tensor([[[[[0.5]]]]]),
        "three": quantised((1, 1, 3, 3, 3), gen),
    }
    for v in vols:
        for mask_only in (True, False):
            bag.add(f"nms3d_{v}_{'mask' if mask_only else 'values'}", "nms3d", {"input": vols[v]},
                    {"kernel_size": [3, 3, 3], "mask_only": mask_only}, {"out": nms3d(vols[v], (3, 3, 3), mask_only)})
        mx, mn = nms3d_minmax(vols[v])
        bag.add(f"nms3d_minmax_{v}", "nms3d_minmax", {"input": vols[v]}, {}, {"max": mx, "min": mn})
    x = quantised((2, 3, 16, 24), gen)
    for ks in ((4, 4), (3, 5), (5, 3), (6, 6)):
        try:
            nms2d(x, ks, True)
            raise SystemExit(f"expected the reference to raise for {ks}")
        except RuntimeError as e:
            bag.add(f"nms2d_error_{ks[0]}x{ks[1]}", "nms2d", {"input": x},
                    {"kernel_size": list(ks), "mask_only": True, "error": type(e).__name__, "message": str(e)}, {})
    v = quantised((1, 2, 5, 16, 24), gen)
    for ks in ((5, 5, 5), (1, 3, 3)):
        try:
            nms3d(v, ks, True)
            raise SystemExit(f"expected the reference to raise for {ks}")
        except RuntimeError as e:
            bag.add(f"nms3d_error_{'x'.join(map(str, ks))}", "nms3d", {"input": v},
                    {"kernel_size": list(ks), "mask_only": True, "error": type(e).__name__, "message": str(e)}, {})
    bag.save(os.path.join(HERE, "nms.npz"))


if __name__ == "__main__":
    main()
