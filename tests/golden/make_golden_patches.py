"""Golden vectors for extract_patches_from_pyramid and extract_patches_simple from the UNMODIFIED reference on CPU fp32.
Needs a checkout of the reference (make_golden.import_reference):

    python tests/golden/make_golden_patches.py    ->  tests/golden/patches.npz (shards patches.<k>.npz)

Inputs are smooth and uniform-noise images at C = 1 and 3: 100 x 120 (where the pyramid stops before the last level the
scales may pick, so those patches stay zero), odd sizes, and images smaller than the patch.  PS is 19, 32 and 41.  The LAFs
are rotated, sheared and anisotropic, some centred outside the image, with log-uniform scales that reach every level the
clamp allows, built or not; both ``normalize_lafs_before_extraction`` values, B = 1 and 2, and both functions.  Some cases
record the gradients of a fixed cotangent with respect to the image and the LAFs; the errors are recorded by type and
message.  The script asserts that every finite LAF has log2(scale) at least 1e-3 away from an integer, except the explicit
exact-power-of-two cases, so a one-ulp difference in the scale cannot move a patch to another level.
"""
from __future__ import annotations

import math
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import Bag, import_reference, smooth_image  # noqa: E402


def make_lafs(B, N, h, w, PS, gen, outside=0.15):
    """(B, N, 2, 3) pixel LAFs: centres in (and partly around) the image, scale 2^U * PS / 2 with U uniform over one level
    below level 0 to two above the top of the clamp, a rotation, an anisotropy and a shear."""
    top = max(0, min(h, w) // PS - 1)
    u = torch.rand(B, N, generator=gen) * (top + 3.0) - 1.0
    s = torch.pow(2.0, u) * PS / 2.0
    ang = torch.rand(B, N, generator=gen) * 2 * math.pi
    r = torch.exp(torch.randn(B, N, generator=gen) * 0.3)
    sh = torch.randn(B, N, generator=gen) * 0.2
    c, si = torch.cos(ang), torch.sin(ang)
    a00, a01 = r.sqrt(), sh
    a10, a11 = torch.zeros_like(r), 1.0 / r.sqrt()
    A = torch.stack([torch.stack([c * a00 - si * a10, c * a01 - si * a11], -1),
                     torch.stack([si * a00 + c * a10, si * a01 + c * a11], -1)], -2) * s[..., None, None]
    cx = (torch.rand(B, N, generator=gen) * (1 + 2 * outside) - outside) * (w - 1)
    cy = (torch.rand(B, N, generator=gen) * (1 + 2 * outside) - outside) * (h - 1)
    return torch.cat([A, torch.stack([cx, cy], -1)[..., None]], -1)


def level_margin_ok(kornia, img, laf, PS, normalize):
    """log2 of the reference's scale, for every finite LAF, at least 1e-3 away from an integer."""
    from kornia.feature.laf import denormalize_laf, get_laf_scale, normalize_laf

    nlaf = normalize_laf(laf, img) if normalize else laf
    lg = (2.0 * get_laf_scale(denormalize_laf(nlaf, img)) / float(PS)).log2().view(-1)
    lg = lg[lg.isfinite()]
    return bool(((lg - lg.round()).abs() >= 1e-3).all())


def main():
    kornia = import_reference()
    from kornia.feature.laf import extract_patches_from_pyramid, extract_patches_simple, normalize_laf

    fns = {"pyramid": extract_patches_from_pyramid, "simple": extract_patches_simple}
    gen = torch.Generator().manual_seed(20261018)
    bag = Bag()

    def image(kind, B, C, h, w):
        return smooth_image(B, C, h, w, gen) if kind == "smooth" else torch.rand(B, C, h, w, generator=gen)

    def lafs(B, N, img, PS, normalize):
        h, w = img.shape[-2:]
        for _ in range(100):
            laf = make_lafs(B, N, h, w, PS, gen)
            if level_margin_ok(kornia, img, laf, PS, True):
                break
        else:
            raise SystemExit("no LAF draw kept its scales away from the level boundaries")
        return laf if normalize else normalize_laf(laf, img)

    def add(name, fn, img, laf, PS, normalize, grad=False, extra=None):
        kw = {"fn": fn, "PS": PS, "normalize": normalize, **(extra or {})}
        if not extra or not extra.get("exact_pow2"):
            assert level_margin_ok(kornia, img, laf, PS, normalize), name
        if grad:
            ig, lg = img.clone().requires_grad_(True), laf.clone().requires_grad_(True)
            out = fns[fn](ig, lg, PS, normalize)
            cot = torch.randn(out.shape, generator=gen)
            gi, gl = torch.autograd.grad((out * cot).sum(), [ig, lg])
            outs = {"out": out.detach(), "cot": cot, "grad_img": gi, "grad_laf": gl}
        else:
            outs = {"out": fns[fn](img, laf, PS, normalize)}
        bag.add(name, "patches", {"img": img, "laf": laf}, kw, outs)

    # the main grid: sizes x channels x PS, both functions, both normalisations
    shapes = [("smooth", 1, 1, 100, 120), ("noise", 2, 3, 100, 120), ("noise", 1, 1, 97, 131), ("smooth", 2, 3, 61, 53),
              ("noise", 1, 1, 130, 167)]
    for kind, B, C, h, w in shapes:
        img = image(kind, B, C, h, w)
        for PS in (19, 32, 41):
            N = 10 if C == 1 else 5
            if PS == 41 and C == 3:
                N = 3
            for normalize in (True, False):
                laf = lafs(B, N, img, PS, normalize)
                for fn in ("pyramid", "simple"):
                    grad = kind == "smooth" and normalize and PS == 19
                    add(f"{fn}_{kind}_B{B}C{C}_{h}x{w}_PS{PS}_{'norm' if normalize else 'raw'}", fn, img, laf, PS, normalize, grad)
    # an image smaller than the patch, and one taller than wide below PS on its short side
    for h, w, PS in ((15, 23, 19), (40, 12, 32)):
        img = image("noise", 1, 1, h, w)
        laf = lafs(1, 6, img, PS, True)
        for fn in ("pyramid", "simple"):
            add(f"{fn}_small_{h}x{w}_PS{PS}", fn, img, laf, PS, True)
    # one pixel high (normalize=False only: normalize_laf divides by h - 1) and one pixel wide
    for h, w in ((1, 40), (37, 1)):
        img = image("noise", 1, 1, h, w)
        laf = make_lafs(1, 4, max(h, 2), max(w, 2), 19, gen) * 0.01
        for fn in ("pyramid", "simple"):
            add(f"{fn}_line_{h}x{w}", fn, img, laf, 19, False, extra={"exact_pow2": True})
    # more images than LAF sets: the extra images are ignored
    img = image("noise", 3, 1, 100, 120)
    laf = lafs(2, 6, img[:2], 32, True)
    for fn in ("pyramid", "simple"):
        add(f"{fn}_extra_images", fn, img, laf, 32, True)
    # exact powers of two: scales PS / 2 * 2^k in pixels with axis-aligned LAFs
    img = image("smooth", 1, 1, 100, 120)
    k = torch.tensor([0.0, 1.0, 2.0, 0.5])
    s = torch.pow(2.0, k) * 32 / 2.0
    laf = torch.zeros(1, 4, 2, 3)
    laf[0, :, 0, 0] = s
    laf[0, :, 1, 1] = s
    laf[0, :, 0, 2] = 60.0
    laf[0, :, 1, 2] = 50.0
    for fn in ("pyramid", "simple"):
        add(f"{fn}_exact_pow2", fn, img, laf, 32, True, extra={"exact_pow2": True})
    # non-finite LAFs: NaN and inf in the linear part and in the centre
    img = image("noise", 1, 1, 100, 120)
    laf = make_lafs(1, 6, 100, 120, 32, gen)
    laf[0, 1, 0, 0] = float("nan")
    laf[0, 2, 1, 2] = float("nan")
    laf[0, 3, 0, 1] = float("inf")
    laf[0, 4, 0, 2] = float("-inf")
    for fn in ("pyramid", "simple"):
        add(f"{fn}_nonfinite", fn, img, laf, 32, True, extra={"exact_pow2": True, "nonfinite": [1, 2, 3, 4]})
    # errors
    ok_img, ok_laf = image("noise", 1, 1, 50, 60), make_lafs(1, 3, 50, 60, 19, gen)
    errors = {
        "empty": (ok_img, torch.zeros(1, 0, 2, 3), 19, True),
        "too_few_images": (ok_img, make_lafs(2, 3, 50, 60, 19, gen), 19, True),
        "one_pixel_normalize": (torch.rand(1, 1, 1, 40, generator=gen), ok_laf, 19, True),
        "laf_shape": (ok_img, torch.zeros(1, 3, 3, 3), 19, True),
        "laf_ndim": (ok_img, torch.zeros(3, 2, 3), 19, True),
    }
    for name, (img, laf, PS, normalize) in errors.items():
        for fn in ("pyramid", "simple"):
            try:
                fns[fn](img, laf, PS, normalize)
                raise SystemExit(f"expected the reference to raise for {name}")
            except SystemExit:
                raise
            except Exception as e:  # noqa: BLE001 -- the type is what is recorded
                bag.add(f"error_{fn}_{name}", "error", {"img": img, "laf": laf},
                        {"fn": fn, "PS": PS, "normalize": normalize, "error": type(e).__name__, "message": str(e)}, {})
    bag.save(os.path.join(HERE, "patches.npz"))


if __name__ == "__main__":
    main()
