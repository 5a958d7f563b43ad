"""Shared helpers for the parity tests: dispatch a golden case onto an implementation module."""
import contextlib
import os
import sys

import torch

# The import graph of the kornia package that install() has to patch: the modules that define the hot-path functions, the
# package re-exports, and the importers of kornia 0.9 (``from ... import warp_perspective``-style and ``from kornia import
# metrics``).  Function bodies do not matter to install(); every defining module gets stand-ins of its names.
_STANDIN_KORNIA = {
    "__init__": "from . import filters, geometry, metrics, losses, augmentation",
    "geometry/transform/imgwarp": "def warp_perspective(): pass\ndef warp_affine(): pass\ndef remap(): pass\ndef get_perspective_transform(): pass",
    "filters/filter": "def filter2d(): pass\ndef filter2d_separable(): pass",
    "filters/gaussian": "def gaussian_blur2d(): pass",
    "filters/sobel": "def spatial_gradient(): pass\ndef sobel(): pass",
    "filters/unsharp": "from .gaussian import gaussian_blur2d",
    "filters/__init__": "from .filter import filter2d, filter2d_separable\nfrom .gaussian import gaussian_blur2d\n"
                        "from .sobel import sobel, spatial_gradient\nfrom . import unsharp",
    "metrics/ssim": "def ssim(): pass",
    "metrics/__init__": "from .ssim import ssim",
    "losses/ssim": "from kornia import metrics",
    "losses/__init__": "from . import ssim",
    "geometry/__init__": "from . import transform, calibration\nfrom .transform import warp_perspective, warp_affine, remap",
    "geometry/transform/__init__": "from .imgwarp import warp_perspective, warp_affine, remap, get_perspective_transform\n"
                                   "from . import affwarp, crop2d, pyramid",
    "geometry/transform/affwarp": "from kornia.filters import gaussian_blur2d\nfrom .imgwarp import warp_affine",
    "geometry/transform/crop2d": "from .imgwarp import get_perspective_transform, warp_affine, warp_perspective",
    "geometry/transform/pyramid": "from kornia.filters import filter2d, gaussian_blur2d",
    "geometry/calibration/__init__": "from . import undistort",
    "geometry/calibration/undistort": "from kornia.geometry.transform import remap",
    "augmentation/__init__": "from . import _2d",
    "augmentation/_2d/__init__": "from . import geometric, intensity",
    "augmentation/_2d/geometric/__init__": "from . import perspective",
    "augmentation/_2d/geometric/perspective": "from kornia.geometry.transform import get_perspective_transform, warp_perspective",
    "augmentation/_2d/intensity/__init__": "from . import gaussian_blur",
    "augmentation/_2d/intensity/gaussian_blur": "from kornia.filters import gaussian_blur2d",
}


@contextlib.contextmanager
def standin_kornia(tmp_dir):
    """Import a stand-in ``kornia`` package (the import graph above, written under ``tmp_dir``); removed again on exit."""
    for mod, src in _STANDIN_KORNIA.items():
        path = os.path.join(tmp_dir, "kornia", mod + ".py")
        os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, "w") as f:
            f.write(src + "\n")
    saved = {k: v for k, v in sys.modules.items() if k == "kornia" or k.startswith("kornia.")}
    for k in saved:
        del sys.modules[k]
    sys.path.insert(0, str(tmp_dir))
    try:
        import kornia

        yield kornia
    finally:
        sys.path.remove(str(tmp_dir))
        for k in [k for k in sys.modules if k == "kornia" or k.startswith("kornia.")]:
            del sys.modules[k]
        sys.modules.update(saved)


def _tup(v):
    return tuple(v) if isinstance(v, list) else v


def run_case(impl, op, kwargs, ins, device=None, dtype=None):
    """Call ``impl.<op>`` (oracle or product: same signatures) on a golden case; returns the output.
    For ``*_grad`` ops returns dict(out=..., grad_<name>=...)."""
    kw = dict(kwargs)
    t = {}
    for k, v in ins.items():
        if dtype is not None and v.is_floating_point():
            v = v.to(dtype)
        t[k] = v.to(device) if device is not None else v
    base = op[:-5] if op.endswith("_grad") else op
    cot = t.pop("cot", None)

    def call(tt):
        if base in ("warp_perspective", "warp_affine"):
            return getattr(impl, base)(tt["src"], tt["M"], _tup(kw["dsize"]), mode=kw["mode"], padding_mode=kw["padding_mode"],
                                       align_corners=kw["align_corners"], fill_value=tt.get("fill_value"))
        if base == "remap":
            return impl.remap(tt["image"], tt["map_x"], tt["map_y"], **kw)
        if base == "filter2d":
            return impl.filter2d(tt["input"], tt["kernel"], **kw)
        if base == "filter2d_separable":
            return impl.filter2d_separable(tt["input"], tt["kernel_x"], tt["kernel_y"], **kw)
        if base == "gaussian_blur2d":
            sigma = tt["sigma"] if "sigma" in tt else _tup(kw["sigma"])
            return impl.gaussian_blur2d(tt["input"], _tup(kw["kernel_size"]), sigma, kw["border_type"], kw["separable"])
        raise KeyError(op)

    if not op.endswith("_grad"):
        return call(t)
    wrt = [k for k in t if k != "fill_value"]
    leaves = dict(t)
    for k in wrt:
        leaves[k] = t[k].clone().requires_grad_(True)
    out = call(leaves)
    grads = torch.autograd.grad((out * cot).sum(), [leaves[k] for k in wrt], allow_unused=True)
    res = {"out": out.detach()}
    for k, g in zip(wrt, grads):
        res[f"grad_{k}"] = g if g is not None else torch.zeros_like(t[k])
    return res


def rel_l2(a, b):
    a = a.double().flatten()
    b = b.double().flatten()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def run_family_case(impl, op, kwargs, ins, device=None, dtype=None):
    """Golden cases of tests/golden/family.npz: every tensor is passed by keyword (the names are the
    reference's parameter names), lists in ``kwargs`` become tuples.  ``*_grad`` ops return
    dict(out=..., grad_<name>=...) for sum(out * cot)."""
    kw = {k: _tup(v) for k, v in kwargs.items()}
    t = {}
    for k, v in ins.items():
        if dtype is not None and v.is_floating_point():
            v = v.to(dtype)
        t[k] = v.to(device) if device is not None else v
    fn = getattr(impl, op[:-5] if op.endswith("_grad") else op)
    if not op.endswith("_grad"):
        return fn(**t, **kw)
    return t, fn, kw


def family_grads(impl, op, kwargs, ins, outs, device=None, dtype=None):
    t, fn, kw = run_family_case(impl, op, kwargs, ins, device, dtype)
    wrt = [k[5:] for k in outs if k.startswith("grad_")]
    leaves = {k: (v.clone().requires_grad_(True) if k in wrt else v) for k, v in t.items()}
    out = fn(**leaves, **kw)
    cot = outs["cot"].to(out)
    grads = torch.autograd.grad((out * cot).sum(), [leaves[k] for k in wrt])
    res = {"out": out.detach()}
    res.update({f"grad_{k}": g for k, g in zip(wrt, grads)})
    return res
