"""Golden vectors for sub-pixel refinement: conv_quad_interp3d, iterative_quad_interp3d and the three modules of the
UNMODIFIED reference run on CPU fp32.  Needs a checkout of the reference (make_golden.import_reference):

    python tests/golden/make_golden_subpix.py    ->  tests/golden/subpix.npz (shards subpix.<k>.npz)

Inputs: rough volumes (randn, where keypoints walk), a smooth blob response (where they almost never move), quantised
plateaus (singular Hessians), special texels (NaN, +-Inf, -0, subnormals) and tiny volumes (D, H or W < 3).  Both forms
run at n_iters 0, 1 and 5, bonus 0 and 10, max_subpixel_shift 0.6 and 0.3, dilation_radius 1 and 2 and both
allow_scale_steps, without a mask, with nms3d_minmax's max mask, with its min mask on -x and with a hand-made mask that
is True on border voxels; the iterative form also with max_candidates.  The reference's errors are recorded by type and
message.  The script asserts that the cases include multi-step walks and keypoints where the two forms disagree.
"""
from __future__ import annotations

import itertools
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import Bag, import_reference, smooth_image  # noqa: E402


def specials(shape, gen):
    x = torch.randn(shape, generator=gen)
    flat = x.view(-1)
    vals = torch.tensor([float("nan"), float("inf"), float("-inf"), -0.0, 1e-40, -1e-41, 2e-45, 0.0])
    idx = torch.randperm(flat.numel(), generator=gen)[: max(8, flat.numel() // 50)]
    flat[idx] = vals[torch.arange(idx.numel()) % vals.numel()]
    return x


def plateaus(shape, gen):
    """Quantised texels with isolated peaks: flat neighbourhoods give det = 0."""
    x = torch.round(torch.rand(shape, generator=gen) * 2) / 4
    flat = x.view(-1)
    idx = torch.randperm(flat.numel(), generator=gen)[: max(2, flat.numel() // 40)]
    flat[idx] = 2.0
    return x


def border_mask(shape, gen):
    m = torch.rand(shape, generator=gen) < 0.05
    m[..., 0, :, :] |= torch.rand(m[..., 0, :, :].shape, generator=gen) < 0.2
    m[..., :, 0, :] = True
    m[..., :, :, -1] |= torch.rand(m[..., :, :, -1].shape, generator=gen) < 0.5
    return m


def main():
    kornia = import_reference()
    from kornia.feature.responses import BlobHessian
    from kornia.geometry.subpix import (AdaptiveQuadInterp3d, ConvQuadInterp3d, IterativeQuadInterp3d, conv_quad_interp3d,
                                        iterative_quad_interp3d, nms3d_minmax)

    torch.set_num_threads(1)
    gen = torch.Generator().manual_seed(2027)
    bag = Bag()
    blob = smooth_image(1, 5, 40, 52, gen)
    resp = BlobHessian()(blob.view(5, 1, 40, 52)).view(1, 5, 1, 40, 52).permute(0, 2, 1, 3, 4).contiguous()
    vols = {
        "randn": torch.randn(1, 2, 5, 16, 20, generator=gen),
        "rough": torch.randn(1, 1, 6, 14, 18, generator=gen) * torch.linspace(0.2, 3, 18),
        "blob": resp,
        "plateau": plateaus((1, 1, 4, 17, 19), gen),
        "special": specials((1, 2, 5, 19, 23), gen),
    }
    tiny = {"d2": torch.randn(1, 1, 2, 9, 9, generator=gen), "h2": torch.randn(1, 2, 4, 2, 9, generator=gen),
            "w1": torch.randn(1, 1, 4, 7, 1, generator=gen), "three": torch.randn(1, 1, 3, 3, 3, generator=gen)}
    walks = disagree = 0
    for name, x in vols.items():
        mx, mn = nms3d_minmax(x)
        masks = {"none": (x, None), "max": (x, mx), "min": (-x, mn), "border": (x, border_mask(x.shape, gen))}
        # every mask with n_iters 0, 1 and 5, the (bonus, shift, allow_scale_steps) triples taken in turn so each occurs;
        # the smooth and degenerate volumes at n_iters 5 only
        combos = list(itertools.product(masks.items(), (0, 1, 5) if name in ("randn", "rough") else (5,)))
        params = list(itertools.product((0.0, 10.0), (0.6, 0.3), (True, False)))
        for i, ((mname, (inp, mask)), n_iters) in enumerate(combos):
            bonus, shift, allow = params[(i * 3) % len(params)] if len(combos) > 4 else (10.0, 0.6, True)
            ins = {"input": inp} if mask is None else {"input": inp, "mask": mask}
            kw = {"n_iters": n_iters, "strict_maxima_bonus": bonus, "max_subpixel_shift": shift, "allow_scale_steps": allow}
            it = iterative_quad_interp3d(inp, n_iters, bonus, shift, allow, precomputed_nms_mask=mask)
            tag = f"{name}_{mname}_n{n_iters}_b{int(bonus)}_s{shift}_{'scale' if allow else 'flat'}"
            bag.add(f"iterative_{tag}", "iterative", ins, kw, {"coords": it[0], "y": it[1]})
            for r in (1, 2):
                cv = conv_quad_interp3d(inp, n_iters, bonus, shift, mask, r, allow)
                bag.add(f"conv_r{r}_{tag}", "conv", ins, {**kw, "dilation_radius": r}, {"coords": cv[0], "y": cv[1]})
                if r == 1:
                    disagree += int((~(cv[0] == it[0]) & ~(cv[0].isnan() & it[0].isnan())).any(2).sum())
            grid = torch.stack(torch.meshgrid(*(torch.arange(n, dtype=torch.float32) for n in inp.shape[2:]), indexing="ij"))
            grid = grid[[0, 2, 1]].expand_as(it[0])
            walks += int(((it[0] - grid).abs() > 1.5).any(2).sum())
        kw = {"n_iters": 5, "strict_maxima_bonus": 10.0, "max_subpixel_shift": 0.6, "allow_scale_steps": True, "max_candidates": 7}
        it = iterative_quad_interp3d(x, max_candidates=7)
        bag.add(f"iterative_{name}_candidates7", "iterative", {"input": x}, kw, {"coords": it[0], "y": it[1]})
        for mod in (ConvQuadInterp3d(), IterativeQuadInterp3d(3, 0.0), AdaptiveQuadInterp3d("conv", dilation_radius=2),
                    AdaptiveQuadInterp3d("patch", max_candidates=5), AdaptiveQuadInterp3d()):
            out = mod(x, mx)
            bag.add(f"module_{name}_{repr(mod)}", "module", {"input": x, "mask": mx}, {"repr": repr(mod)}, {"coords": out[0], "y": out[1]})
    for name, x in tiny.items():
        mask = torch.ones(x.shape, dtype=torch.bool)
        for op, fn in (("conv", lambda t, m: conv_quad_interp3d(t, precomputed_nms_mask=m)),
                       ("iterative", lambda t, m: iterative_quad_interp3d(t, precomputed_nms_mask=m))):
            out = fn(x, mask)
            kw = {"n_iters": 5, "strict_maxima_bonus": 10.0, "max_subpixel_shift": 0.6, "allow_scale_steps": True}
            if op == "conv":
                kw["dilation_radius"] = 1
            bag.add(f"{op}_tiny_{name}", op, {"input": x, "mask": mask}, kw, {"coords": out[0], "y": out[1]})
    x = torch.randn(1, 2, 4, 9, 11, generator=gen)
    x3 = torch.randn(1, 3, 4, 9, 11, generator=gen)  # (B, L, C, H, W) read as (B, C, L, H, W): C > 1 cannot be viewed
    errors = {
        "type": (lambda: conv_quad_interp3d(x.numpy()), "conv"),
        "type_iterative": (lambda: iterative_quad_interp3d([1.0]), "iterative"),
        "ndim": (lambda: conv_quad_interp3d(x[0]), "conv"),
        "ndim_iterative": (lambda: iterative_quad_interp3d(x[:, :, 0]), "iterative"),
        "view": (lambda: conv_quad_interp3d(x3.transpose(1, 2)), "conv"),
        "mode": (lambda: AdaptiveQuadInterp3d("fast"), "module"),
    }
    for name, (fn, op) in errors.items():
        try:
            fn()
            raise SystemExit(f"expected the reference to raise for {name}")
        except (TypeError, ValueError, RuntimeError) as e:
            bag.add(f"error_{name}", op, {"input": x3 if name == "view" else x}, {"case": name, "error": type(e).__name__, "message": str(e)}, {})
    print(f"keypoints that walked more than 1.5 voxels: {walks}; conv / iterative disagreements (r = 1): {disagree}")
    assert walks > 0 and disagree > 0, (walks, disagree)
    bag.save(os.path.join(HERE, "subpix.npz"))


if __name__ == "__main__":
    main()
