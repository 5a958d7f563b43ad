"""Golden vectors for PatchAffineShapeEstimator and LAFAffineShapeEstimator from the UNMODIFIED reference on CPU fp32.
Needs a checkout of the reference (make_golden.import_reference):

    python tests/golden/make_golden_affine_shape.py    ->  tests/golden/affine_shape.npz (shards affine_shape.<k>.npz)

LAF cases: smooth, uniform-noise, constant and vertical-stripe images (the stripes give patches with no vertical gradient
once the LAF is upright, so they take the degenerate, circular branch), PS 19 / 32 / 41, B = 1 and 2 and more images than
LAF sets, rotated / sheared / anisotropic LAFs with some centred outside the image and scales reaching levels the pyramid
does not build, both ``preserve_orientation`` values and a non-default ``eps``.  Patch cases: ``PatchAffineShapeEstimator``
on noise, smooth, flat and anti-correlated (negative b) patch stacks.  Some cases record the gradients of a fixed cotangent
with respect to the image and the LAFs; non-finite LAFs are recorded, and the errors by type and message.

The script asserts, except for the explicitly marked cases, that every upright LAF has log2(scale) at least 1e-3 away from an
integer and that every moment is at least 1e-3 (relative) away from eps, so a one-ulp difference cannot move a keypoint to
another level or flip the degenerate decision.
"""
from __future__ import annotations

import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import Bag, import_reference, smooth_image  # noqa: E402
from make_golden_patches import level_margin_ok, make_lafs  # noqa: E402


def moments(det, patches):
    """The raw (a, b, c) of PatchAffineShapeEstimator before the degenerate test, as the reference computes them."""
    grads = det.gradient(patches) * det.weighting.to(patches.dtype)
    gx, gy = grads[:, :, 0], grads[:, :, 1]
    return torch.cat([gx.pow(2).mean(dim=2).mean(dim=2, keepdim=True), (gx * gy).mean(dim=2).mean(dim=2, keepdim=True),
                      gy.pow(2).mean(dim=2).mean(dim=2, keepdim=True)], dim=2)


def moment_margin_ok(det, patches):
    m = moments(det, patches)
    return bool(((m - det.eps).abs() >= 1e-3 * det.eps).all())


def main():
    kornia = import_reference()
    from kornia.feature.affine_shape import LAFAffineShapeEstimator, PatchAffineShapeEstimator
    from kornia.feature.laf import extract_patches_from_pyramid, make_upright

    gen = torch.Generator().manual_seed(20261019)
    bag = Bag()

    def image(kind, B, h, w):
        if kind == "smooth":
            return smooth_image(B, 1, h, w, gen)
        if kind == "noise":
            return torch.rand(B, 1, h, w, generator=gen)
        if kind == "constant":
            return torch.full((B, 1, h, w), 0.375)
        x = torch.arange(w).float()
        return ((x // 4) % 2).view(1, 1, 1, w).expand(B, 1, h, w).contiguous()  # vertical stripes

    def margins_ok(img, laf, m):
        det = m.affine_shape_detector
        up = make_upright(laf)
        fin = laf.isfinite().view(laf.shape[0], laf.shape[1], -1).all(-1)
        if not level_margin_ok(kornia, img, up[fin].view(1, -1, 2, 3), m.patch_size, True):
            return False
        patches = extract_patches_from_pyramid(img, up, m.patch_size, True).view(-1, 1, m.patch_size, m.patch_size)
        return moment_margin_ok(det, patches[fin.view(-1)])

    def lafs(B, N, img, m):
        h, w = img.shape[-2:]
        for _ in range(200):
            laf = make_lafs(B, N, h, w, m.patch_size, gen)
            if margins_ok(img[:B], laf, m):
                return laf
        raise SystemExit("no LAF draw kept its scales and moments away from the decision boundaries")

    def add_laf(name, img, laf, m, grad=False, extra=None):
        kw = {"PS": m.patch_size, "preserve_orientation": m.preserve_orientation, "eps": m.affine_shape_detector.eps, **(extra or {})}
        if not kw.get("unchecked"):
            assert margins_ok(img[:laf.shape[0]], laf, m), name
        if grad:
            ig, lg = img.clone().requires_grad_(True), laf.clone().requires_grad_(True)
            out = m(lg, ig)
            cot = torch.randn(out.shape, generator=gen)
            gi, gl = torch.autograd.grad((out * cot).sum(), [ig, lg])
            outs = {"out": out.detach(), "cot": cot, "grad_img": gi, "grad_laf": gl}
        else:
            with torch.no_grad():
                outs = {"out": m(laf, img)}
        bag.add(name, "laf", {"img": img, "laf": laf}, kw, outs)

    # the main grid: image kinds x PS x preserve_orientation
    for kind, B, h, w in (("smooth", 1, 100, 120), ("noise", 2, 97, 131), ("constant", 1, 64, 80), ("stripes", 1, 90, 110)):
        img = image(kind, B, h, w)
        for PS in (19, 32, 41):
            for preserve in (True, False):
                m = LAFAffineShapeEstimator(PS, preserve_orientation=preserve)
                laf = lafs(B, 8 if PS < 41 else 5, img, m)
                grad = kind == "smooth" and PS == 19 and preserve
                add_laf(f"laf_{kind}_B{B}_{h}x{w}_PS{PS}_{'preserve' if preserve else 'upright'}", img, laf, m, grad)
    # more images than LAF sets; a non-default eps
    img = image("smooth", 3, 100, 120)
    m = LAFAffineShapeEstimator(32)
    add_laf("laf_extra_images", img, lafs(2, 6, img, m), m)
    m = LAFAffineShapeEstimator(19, PatchAffineShapeEstimator(19, eps=1e-5))
    img = image("smooth", 1, 100, 120)
    add_laf("laf_eps_1e-5", img, lafs(1, 8, img, m), m)
    # non-finite LAFs: NaN and inf in the linear part and in the centre
    img = image("noise", 1, 100, 120)
    m = LAFAffineShapeEstimator(32)
    laf = make_lafs(1, 6, 100, 120, 32, gen)
    laf[0, 1, 0, 0] = float("nan")
    laf[0, 2, 1, 2] = float("nan")
    laf[0, 3, 0, 1] = float("inf")
    laf[0, 4, 0, 2] = float("-inf")
    add_laf("laf_nonfinite", img, laf, m, extra={"unchecked": True, "nonfinite": [1, 2, 3, 4]})

    # PatchAffineShapeEstimator on its own
    def add_patch(name, patches, det):
        assert moment_margin_ok(det, patches), name
        with torch.no_grad():
            out = det(patches)
        bag.add(name, "patch", {"patch": patches}, {"patch_size": det.patch_size, "eps": det.eps}, {"out": out})

    for P in (19, 32):
        n = 12
        noise = torch.rand(n, 1, P, P, generator=gen)
        smooth = smooth_image(n, 1, P, P, gen)
        flat = torch.full((4, 1, P, P), 0.5)
        yy, xx = torch.meshgrid(torch.arange(P).float(), torch.arange(P).float(), indexing="ij")
        anti = (0.05 * (xx - yy)).view(1, 1, P, P) * torch.rand(4, 1, 1, 1, generator=gen) + 0.01 * torch.rand(4, 1, P, P, generator=gen)
        add_patch(f"patch_mix_P{P}", torch.cat([noise, smooth, flat, anti]), PatchAffineShapeEstimator(P))
    add_patch("patch_eps_1e-3", torch.rand(8, 1, 19, 19, generator=gen) * 0.2, PatchAffineShapeEstimator(19, eps=1e-3))

    # the LAF helpers on their own
    from kornia.feature import laf as KL

    laf = make_lafs(2, 7, 100, 120, 19, gen)
    ang = torch.rand(2, 7, 1, generator=gen) * 720.0 - 360.0
    coef = torch.rand(2, 7, 1, 1, generator=gen) + 0.5
    ells = torch.cat([torch.rand(2, 7, 2, generator=gen) * 100, torch.rand(2, 7, 1, generator=gen) + 0.1,
                      torch.rand(2, 7, 1, generator=gen) * 0.2 - 0.1, torch.rand(2, 7, 1, generator=gen) + 0.1], -1)
    bag.add("helpers", "helpers", {"laf": laf, "angle": ang, "coef": coef, "ells": ells}, {},
            {"make_upright": KL.make_upright(laf), "scale_laf": KL.scale_laf(laf, coef), "scale_laf_float": KL.scale_laf(laf, 0.75),
             "ellipse_to_laf": KL.ellipse_to_laf(ells), "get_laf_orientation": KL.get_laf_orientation(laf),
             "set_laf_orientation": KL.set_laf_orientation(laf, ang), "rotate_laf": KL.rotate_laf(laf, ang)})

    # errors
    ok_img = image("noise", 1, 50, 60)
    ok_laf = make_lafs(1, 3, 50, 60, 19, gen)
    errors = {
        "laf_no_lafs": ("laf", (torch.zeros(1, 0, 2, 3), ok_img), 19),
        "laf_three_channels": ("laf", (ok_laf, image("noise", 1, 50, 60).expand(1, 3, 50, 60).contiguous()), 19),
        "laf_shape": ("laf", (torch.zeros(1, 3, 3, 3), ok_img), 19),
        "laf_ndim": ("laf", (torch.zeros(3, 2, 3), ok_img), 19),
        "laf_too_few_images": ("laf", (make_lafs(2, 3, 50, 60, 19, gen), ok_img), 19),
        "patch_wrong_size": ("patch", (torch.rand(2, 1, 20, 20, generator=gen),), 19),
        "patch_two_channels": ("patch", (torch.rand(2, 2, 19, 19, generator=gen),), 19),
    }
    for name, (op, args, PS) in errors.items():
        mod = LAFAffineShapeEstimator(PS) if op == "laf" else PatchAffineShapeEstimator(PS)
        try:
            mod(*args)
            raise SystemExit(f"expected the reference to raise for {name}")
        except SystemExit:
            raise
        except Exception as e:  # noqa: BLE001 -- the type is what is recorded
            ins = {"laf": args[0], "img": args[1]} if op == "laf" else {"patch": args[0]}
            bag.add(f"error_{name}", "error", ins, {"op": op, "PS": PS, "error": type(e).__name__, "message": str(e)}, {})
    bag.save(os.path.join(HERE, "affine_shape.npz"))


if __name__ == "__main__":
    main()
