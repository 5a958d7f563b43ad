"""Golden vectors for ScalePyramid: every octave of the UNMODIFIED reference run on CPU fp32.  Needs a checkout of the
reference (make_golden.import_reference):

    python tests/golden/make_golden_scale_pyramid.py    ->  tests/golden/scale_pyramid.npz (shards scale_pyramid.<k>.npz)

Configurations: the default, extra_levels=2, double_image with min_size=32, n_levels=1 with init_sigma=0.25 (no initial
blur), n_levels=4 (a tap chain the octave kernel does not instantiate), a 31 x 31 image (levels that take the reference's
gaussian_blur2d fallback) and an odd width.  Every case records each octave's levels (``pyr<o>``), ``sigmas`` and
``pixel_dists`` (``sig<o>``, ``pd<o>``) and the gradient of sum over octaves of (level * cot) with respect to the input.
"""
from __future__ import annotations

import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import Bag, import_reference, smooth_image  # noqa: E402

CASES = [
    ("default", (1, 2, 40, 48), {}),
    ("extra2", (2, 1, 36, 44), {"n_levels": 3, "init_sigma": 1.6, "min_size": 15, "extra_levels": 2}),
    ("double", (1, 1, 24, 32), {"n_levels": 3, "init_sigma": 1.6, "min_size": 32, "double_image": True}),
    ("noblur", (1, 1, 32, 40), {"n_levels": 1, "init_sigma": 0.25}),
    ("levels4", (1, 1, 40, 44), {"n_levels": 4}),
    ("tiny31", (1, 1, 31, 31), {}),
    ("oddwidth", (1, 1, 36, 45), {}),
]


def main():
    import_reference()
    from kornia.geometry.transform import ScalePyramid

    torch.set_num_threads(1)
    gen = torch.Generator().manual_seed(1717)
    bag = Bag()
    for name, shape, kw in CASES:
        x = smooth_image(*shape, gen) + 0.05 * torch.rand(shape, generator=gen)
        xi = x.clone().requires_grad_(True)
        pyr, sigmas, pds = ScalePyramid(**kw)(xi)
        cots = [torch.rand(p.shape, generator=gen) for p in pyr]
        (g,) = torch.autograd.grad(sum((p * c).sum() for p, c in zip(pyr, cots)), [xi])
        ins = {"input": x}
        outs = {"grad_input": g}
        for o, (p, s, d, c) in enumerate(zip(pyr, sigmas, pds, cots)):
            ins[f"cot{o}"] = c
            outs[f"pyr{o}"] = p.detach()
            outs[f"sig{o}"] = s
            outs[f"pd{o}"] = d
        bag.add(name, "ScalePyramid", ins, kw, outs)
    bag.save(os.path.join(HERE, "scale_pyramid.npz"))


if __name__ == "__main__":
    main()
