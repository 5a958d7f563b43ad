"""Golden vectors for SIFTDescriptor, sift_describe, PatchDominantGradientOrientation and their kernel helpers from the
UNMODIFIED reference on CPU fp32.  Needs a checkout of the reference (make_golden.import_reference):

    python tests/golden/make_golden_sift.py    ->  tests/golden/sift.npz (shards sift.<k>.npz)

SIFT runs every configuration the reference's own tests use -- (41, 8, 4), (32, 8, 4), (15, 8, 4), (19, 5, 3) and
(6, 4, 1) -- with rootsift both ways and clipval 0.2 and 0.1; orientation runs P = 19 and 32 with 36 and 8 bins.  Inputs are
smooth, random, constant and special-texel (NaN, +-Inf, -0) patches, N = 1 and N = 0.  Finite cases also record the
gradients of a fixed cotangent with respect to the input and pk.weight / angular_smooth.weight.  The errors are recorded
by type and message, and get_sift_pooling_kernel, get_sift_bin_ksize_stride_pad and get_gaussian_discrete_kernel1d by
value.  The script asserts that every orientation case whose patches are not special texels has its top two smoothed
bins apart by more than 1e-4 relative, and builds an exact tie between two non-adjacent bins (a constant patch and
smoothing taps [1, 0, 0, 0, 1]), whose angle is that of the first of them, as torch.max returns.
"""
from __future__ import annotations

import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from make_golden import Bag, import_reference, smooth_image  # noqa: E402
import sift_restated as SR  # noqa: E402

SIFT_CONFIGS = [(41, 8, 4), (32, 8, 4), (15, 8, 4), (19, 5, 3), (6, 4, 1)]
ORI_CONFIGS = [(19, 36), (32, 36), (19, 8), (32, 8)]


def specials(N, P, gen):
    x = torch.rand(N, 1, P, P, generator=gen)
    flat = x.view(-1)
    vals = torch.tensor([float("nan"), float("inf"), float("-inf"), -0.0])
    for n in range(N):  # patch 0 stays finite; the others get one to three special texels each
        for k in range(n % 3 + (1 if n else 0)):
            flat[n * P * P + int(torch.randint(P * P, (1,), generator=gen))] = vals[(n + k) % 4]
    return x


def inputs(P, gen):
    return {
        "smooth": smooth_image(6, 1, P, P, gen),
        "random": torch.rand(6, 1, P, P, generator=gen),
        "constant": torch.full((2, 1, P, P), 0.37),
        "special": specials(6, P, gen),
        "single": torch.rand(1, 1, P, P, generator=gen),
        "empty": torch.zeros(0, 1, P, P),
    }


def margin_ok(hist):
    top = hist.topk(2, 1).values
    return ((top[:, 0] - top[:, 1]).abs() > 1e-4 * top[:, 0].abs()).all().item()


def main():
    kornia = import_reference()
    from kornia.feature.orientation import PatchDominantGradientOrientation
    from kornia.feature.siftdesc import SIFTDescriptor, get_sift_bin_ksize_stride_pad, get_sift_pooling_kernel, sift_describe
    from kornia.filters import get_gaussian_discrete_kernel1d

    gen = torch.Generator().manual_seed(20261017)
    bag = Bag()
    for P, A, S in SIFT_CONFIGS:
        for rootsift in (True, False):
            for clipval in (0.2, 0.1):
                if P == 6 and rootsift:
                    continue  # the reference tests (6, 4, 1) with rootsift=False only
                m = SIFTDescriptor(P, A, S, rootsift, clipval)
                kw = {"patch_size": P, "num_ang_bins": A, "num_spatial_bins": S, "rootsift": rootsift, "clipval": clipval, "repr": repr(m)}
                for name, x in inputs(P, gen).items():
                    kw = {k: v for k, v in kw.items() if k not in ("error", "message")}
                    if name in ("smooth", "random") and x.shape[0]:
                        xg = x.clone().requires_grad_(True)
                        m.zero_grad()
                        out = m(xg)
                        cot = torch.randn(out.shape, generator=gen)
                        (gx,) = torch.autograd.grad((out * cot).sum(), [xg], retain_graph=True)
                        (gw,) = torch.autograd.grad((out * cot).sum(), [m.pk.weight])
                        outs = {"out": out.detach(), "grad_input": gx, "grad_weight": gw, "cot": cot}
                    else:
                        try:
                            with torch.no_grad():
                                outs = {"out": m(x)}
                        except RuntimeError as e:  # N = 0: the reference's view(B, -1) of an empty tensor raises
                            kw = {**kw, "error": type(e).__name__, "message": str(e)}
                    bag.add(f"sift_{P}_{A}_{S}_{'root' if rootsift else 'l2'}_{clipval}_{name}", "sift", {"input": x}, kw, outs)
    x = torch.rand(3, 1, 41, 41, generator=gen)
    with torch.no_grad():
        bag.add("sift_describe_default", "sift_describe", {"input": x}, {}, {"out": sift_describe(x)})
    for P, A in ORI_CONFIGS:
        m = PatchDominantGradientOrientation(P, A)
        kw = {"patch_size": P, "num_angular_bins": A, "repr": repr(m)}
        for name, x in inputs(P, gen).items():
            if name in ("smooth", "random"):  # keep the patches whose top two smoothed bins are clearly apart
                x = torch.cat([p for p in x.split(1) if margin_ok(SR.orientation(p, m.weighting, m.angular_smooth.weight.detach(), A,
                                                                                  return_hist=True)[1])])
            if name not in ("special", "empty"):
                _, hist = SR.orientation(x, m.weighting, m.angular_smooth.weight.detach(), A, return_hist=True)
                assert margin_ok(hist), (P, A, name)
            if name in ("smooth", "random"):
                xg = x.clone().requires_grad_(True)
                m.zero_grad()
                out = m(xg)
                cot = torch.randn(out.shape, generator=gen)
                (gx,) = torch.autograd.grad((out * cot).sum(), [xg], retain_graph=True)
                (gw,) = torch.autograd.grad((out * cot).sum(), [m.angular_smooth.weight])
                outs = {"out": out.detach(), "grad_input": gx, "grad_weight": gw, "cot": cot}
            else:
                with torch.no_grad():
                    outs = {"out": m(x)}
            bag.add(f"orientation_{P}_{A}_{name}", "orientation", {"input": x}, kw, outs)
    # an exact tie between non-adjacent bins: a constant patch puts (almost) all of its weight in one bin b, and the
    # smoothing taps [1, 0, 0, 0, 1] copy that bin's value to bins b - 2 and b + 2 by the same single product, so the two
    # maxima are equal in any evaluation order; torch.max must take the first of them
    A = 36
    m = PatchDominantGradientOrientation(19, A)
    smooth = torch.tensor([1.0, 0.0, 0.0, 0.0, 1.0]).view(1, 1, 5)
    m.load_state_dict({"angular_smooth.weight": smooth}, strict=True)
    x = torch.full((1, 1, 19, 19), 0.37)
    with torch.no_grad():
        out = m(x)
    _, hist = SR.orientation(x, m.weighting, smooth, A, return_hist=True)
    top = (hist[0] == hist[0].max()).nonzero().view(-1).tolist()
    assert len(top) == 2 and (top[1] - top[0]) % A not in (1, A - 1), top
    first, last = top

    def angle(i):
        n1, n2 = hist[0, (i - 1) % A], hist[0, (i + 1) % A]
        c = 0.5 * (n1 - n2) / (n1 + n2 - 2.0 * hist[0, i])
        return float(-((2.0 * SR.PI * (i + c) / float(A)) - SR.PI))

    assert abs(angle(first) - float(out[0])) < 1e-6 and abs(angle(last) - float(out[0])) > 0.1, (angle(first), angle(last), out)
    bag.add("orientation_19_tie", "orientation", {"input": x, "smooth": smooth}, {"patch_size": 19, "num_angular_bins": A, "repr": repr(m),
                                                                                  "tie": True, "first_index": first, "last_index": last},
            {"out": out})
    print(f"exact tie between bins {first} and {last} of {A}")
    # helpers
    for k in (3, 4, 8, 16, 25):
        bag.add(f"pooling_kernel_{k}", "pooling_kernel", {}, {"ksize": k}, {"out": get_sift_pooling_kernel(k)})
    params = {f"{p}_{s}": list(get_sift_bin_ksize_stride_pad(p, s)) for p, s in [(41, 4), (32, 4), (15, 4), (19, 3), (6, 1), (64, 4), (32, 8)]}
    bag.add("bin_ksize_stride_pad", "bin_params", {}, {"params": params}, {})
    for ks, s in [(5, 1.6), (3, 2.5), (5, 1.5), (7, 3.0), (9, 0.5)]:
        bag.add(f"discrete_{ks}_{s}", "discrete", {}, {"kernel_size": ks, "sigma": s}, {"out": get_gaussian_discrete_kernel1d(ks, s)})
    sig = torch.tensor([[1.5], [2.4]])
    bag.add("discrete_batch", "discrete", {"sigma": sig}, {"kernel_size": 5}, {"out": get_gaussian_discrete_kernel1d(5, sig)})
    errors = {
        "incompatible": lambda: SIFTDescriptor(4, 8, 4),
        "incompatible_fn": lambda: get_sift_bin_ksize_stride_pad(10, 6),
        "sift_shape": lambda: SIFTDescriptor(32)(torch.zeros(2, 1, 41, 41)),
        "sift_ndim": lambda: SIFTDescriptor(32)(torch.zeros(1, 32, 32)),
        "orientation_shape": lambda: PatchDominantGradientOrientation(19)(torch.zeros(2, 1, 32, 32)),
        "orientation_channels": lambda: PatchDominantGradientOrientation(19)(torch.zeros(2, 3, 19, 19)),
    }
    for name, fn in errors.items():
        try:
            fn()
            raise SystemExit(f"expected the reference to raise for {name}")
        except Exception as e:  # noqa: BLE001 -- the type is what is recorded
            bag.add(f"error_{name}", "error", {}, {"case": name, "error": type(e).__name__, "message": str(e)}, {})
    bag.save(os.path.join(HERE, "sift.npz"))


if __name__ == "__main__":
    main()
