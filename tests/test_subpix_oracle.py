"""Sub-pixel refinement on the host (no GPU): the plain-torch restatement (tests/subpix_restated.py) and the library's
composition both reproduce the reference's goldens bit for bit (NaN equals NaN, -0 and +0 differ), errors included; the
public signatures, defaults, reprs, empty state_dicts, MODES and validation match the reference's; install() rebinds the
five names on a stand-in package, and a ScaleSpaceDetector stand-in built afterwards holds the library's refiner and
passes its isinstance check."""
import importlib
import inspect
import sys

import pytest
import torch

import helpers
import subpix_restated as SR
from conftest import golden

K = importlib.import_module("kornia_b200")
Q = importlib.import_module("kornia_b200.geometry.subpix.quad_interp")
G = golden("subpix")


def _same(a, b):
    assert a.shape == b.shape and a.dtype == b.dtype, (a.shape, b.shape, a.dtype, b.dtype)
    return bool(((a.view(torch.int32) == b.view(torch.int32)) | (a.isnan() & b.isnan())).all())


def _module(text):
    return eval(text, {name: getattr(Q, name) for name in Q.__all__})  # the repr is the constructor call


def _library(op, kw, ins):
    x, mask = ins["input"], ins.get("mask")
    if op == "module":
        return _module(kw["repr"])(x, mask)
    if op == "conv":
        return Q.conv_quad_interp3d(x, kw["n_iters"], kw["strict_maxima_bonus"], kw["max_subpixel_shift"], mask, kw["dilation_radius"],
                                    kw["allow_scale_steps"])
    return Q.iterative_quad_interp3d(x, kw["n_iters"], kw["strict_maxima_bonus"], kw["max_subpixel_shift"], kw["allow_scale_steps"], mask,
                                     kw.get("max_candidates"))


def _restated(op, kw, ins):
    x, mask = ins["input"], ins.get("mask")
    if op == "module":
        m = _module(kw["repr"])
        conv = isinstance(m, Q.ConvQuadInterp3d) or (isinstance(m, Q.AdaptiveQuadInterp3d) and m.mode == "conv")
        return SR.refine(x, m.n_iters, m.strict_maxima_bonus, m.max_subpixel_shift, mask, m.dilation_radius if conv else None,
                         m.allow_scale_steps, None if conv else m.max_candidates)
    return SR.refine(x, kw["n_iters"], kw["strict_maxima_bonus"], kw["max_subpixel_shift"], mask, kw.get("dilation_radius"),
                     kw["allow_scale_steps"], kw.get("max_candidates"))


ERRORS = {
    "type": lambda x: Q.conv_quad_interp3d(x.numpy()),
    "type_iterative": lambda x: Q.iterative_quad_interp3d([1.0]),
    "ndim": lambda x: Q.conv_quad_interp3d(x[0]),
    "ndim_iterative": lambda x: Q.iterative_quad_interp3d(x[:, :, 0]),
    "view": lambda x: Q.conv_quad_interp3d(x.transpose(1, 2)),
    "mode": lambda x: Q.AdaptiveQuadInterp3d("fast"),
}


@pytest.mark.parametrize("impl", ["restated", "composed"])
@pytest.mark.parametrize("name", G.names())
def test_reproduces_the_goldens(name, impl):
    op, kw, ins, outs = G.case(name)
    if "error" in kw:
        if impl == "restated":
            pytest.skip("errors are the library's to reproduce")
        with pytest.raises((TypeError, ValueError, RuntimeError)) as e:
            ERRORS[kw["case"]](ins["input"])
        assert type(e.value).__name__ == kw["error"] and str(e.value) == kw["message"]
        return
    coords, y = (_restated if impl == "restated" else _library)(op, kw, ins)
    assert _same(coords, outs["coords"]) and _same(y, outs["y"])


def test_goldens_cover_the_cases_the_issue_names():
    names = G.names()
    kws = [G.case(n)[1] for n in names]
    assert {k.get("n_iters") for k in kws} >= {0, 1, 5} and {k.get("dilation_radius") for k in kws} >= {1, 2}
    assert {k.get("strict_maxima_bonus") for k in kws} >= {0.0, 10.0} and {k.get("max_subpixel_shift") for k in kws} >= {0.6, 0.3}
    assert {k.get("allow_scale_steps") for k in kws} >= {True, False}
    for part in ("_none_", "_max_", "_min_", "_border_", "candidates7", "tiny_d2", "tiny_h2", "tiny_w1", "special_", "plateau_", "blob_"):
        assert any(part in n for n in names), part
    assert {f"error_{c}" for c in ERRORS} <= set(names)


def _sig(fn):
    params = inspect.signature(fn).parameters.values()
    return "(" + ", ".join(p.name if p.default is inspect._empty else f"{p.name}={p.default!r}" for p in params) + ")"


def test_signatures_reprs_state_dicts_match_reference():
    assert _sig(Q.conv_quad_interp3d) == ("(input, n_iters=5, strict_maxima_bonus=10.0, max_subpixel_shift=0.6, precomputed_nms_mask=None, "
                                          "dilation_radius=1, allow_scale_steps=True)")
    assert _sig(Q.iterative_quad_interp3d) == ("(input, n_iters=5, strict_maxima_bonus=10.0, max_subpixel_shift=0.6, allow_scale_steps=True, "
                                               "precomputed_nms_mask=None, max_candidates=None)")
    assert _sig(Q.ConvQuadInterp3d.__init__) == "(self, n_iters=5, strict_maxima_bonus=10.0, max_subpixel_shift=0.6, dilation_radius=1, allow_scale_steps=True)"
    assert _sig(Q.IterativeQuadInterp3d.__init__) == ("(self, n_iters=5, strict_maxima_bonus=10.0, max_subpixel_shift=0.6, allow_scale_steps=True, "
                                                      "max_candidates=None)")
    assert _sig(Q.AdaptiveQuadInterp3d.__init__) == ("(self, mode='auto', n_iters=5, strict_maxima_bonus=10.0, max_subpixel_shift=0.6, "
                                                     "dilation_radius=1, allow_scale_steps=True, max_candidates=None)")
    for cls in (Q.ConvQuadInterp3d, Q.IterativeQuadInterp3d, Q.AdaptiveQuadInterp3d):
        assert _sig(cls.forward) == "(self, x, precomputed_nms_mask=None)"
        assert list(cls().state_dict()) == []
    assert repr(Q.ConvQuadInterp3d()) == "ConvQuadInterp3d(n_iters=5, strict_maxima_bonus=10.0, max_subpixel_shift=0.6, dilation_radius=1, allow_scale_steps=True)"
    assert repr(Q.IterativeQuadInterp3d(3, 0.0)) == ("IterativeQuadInterp3d(n_iters=3, strict_maxima_bonus=0.0, max_subpixel_shift=0.6, "
                                                     "allow_scale_steps=True, max_candidates=None)")
    assert repr(Q.AdaptiveQuadInterp3d("patch", max_candidates=5)) == (
        "AdaptiveQuadInterp3d(mode='patch', n_iters=5, strict_maxima_bonus=10.0, max_subpixel_shift=0.6, dilation_radius=1, "
        "allow_scale_steps=True, max_candidates=5)")
    assert Q.AdaptiveQuadInterp3d.MODES == ("patch", "conv", "auto")
    with pytest.raises(ValueError, match=r"mode must be one of \('patch', 'conv', 'auto'\), got 'fast'"):
        Q.AdaptiveQuadInterp3d("fast")
    for name in Q.__all__:
        assert getattr(K.geometry, name) is getattr(Q, name) and getattr(K.geometry.subpix, name) is getattr(Q, name)
        assert name in K.geometry.__all__ and name in K.geometry.subpix.__all__


def test_composition_is_differentiable_on_the_cpu():
    x = torch.randn(1, 1, 4, 9, 10, dtype=torch.float64, requires_grad=True)
    for f in (lambda t: Q.conv_quad_interp3d(t, 3, 1.0, 0.3), lambda t: Q.iterative_quad_interp3d(t, 3, 1.0, 0.3)):
        coords, y = f(x)
        assert coords.requires_grad and y.requires_grad
        assert torch.autograd.gradcheck(lambda t: f(t)[1], (x,), eps=1e-6, atol=1e-6)


_QUAD_MODULES = {
    "geometry/__init__": "from . import transform, calibration, subpix\nfrom .transform import warp_perspective, warp_affine, remap\n"
                         "from .subpix import *",
    "geometry/subpix/__init__": "from .nms import nms3d\nfrom .spatial_soft_argmax import conv_quad_interp3d, iterative_quad_interp3d, "
                                "ConvQuadInterp3d, IterativeQuadInterp3d, AdaptiveQuadInterp3d",
    "geometry/subpix/nms": "def nms3d(): pass",
    "geometry/subpix/spatial_soft_argmax": "from .nms import nms3d\ndef conv_quad_interp3d(): pass\ndef iterative_quad_interp3d(): pass\n"
                                           "class _Refiner:\n    def __init__(self, *args, **kwargs): pass\n"
                                           "class ConvQuadInterp3d(_Refiner): pass\nclass IterativeQuadInterp3d(_Refiner): pass\n"
                                           "class AdaptiveQuadInterp3d(_Refiner): pass",
    "__init__": "from . import filters, geometry, metrics, losses, augmentation, feature",
    "feature/__init__": "from . import scale_space_detector, integrated",
    # the reference detector: its default refiner and its isinstance check, by the names it imports
    "feature/scale_space_detector": (
        "from kornia.geometry.subpix import AdaptiveQuadInterp3d, ConvQuadInterp3d, IterativeQuadInterp3d\n"
        "class ScaleSpaceDetector:\n"
        "    def __init__(self, subpix_module=None):\n"
        "        if subpix_module is None:\n"
        "            subpix_module = AdaptiveQuadInterp3d(strict_maxima_bonus=0.0, allow_scale_steps=True)\n"
        "        self._is_iterative_subpix = isinstance(subpix_module, (ConvQuadInterp3d, AdaptiveQuadInterp3d, IterativeQuadInterp3d))\n"
        "        self.subpix = subpix_module\n"),
    "feature/integrated": "from kornia.geometry.subpix import ConvQuadInterp3d\ndef sift_refiner():\n    return ConvQuadInterp3d(strict_maxima_bonus=0.0)",
}
_IMPORTERS = {
    "kornia.geometry.subpix.spatial_soft_argmax": Q.__all__,
    "kornia.geometry.subpix": Q.__all__,
    "kornia.geometry": Q.__all__,
    "kornia.feature.scale_space_detector": ["AdaptiveQuadInterp3d", "ConvQuadInterp3d", "IterativeQuadInterp3d"],
    "kornia.feature.integrated": ["ConvQuadInterp3d"],
}


def test_install_rebinds_the_refiners_everywhere(tmp_path, monkeypatch):
    monkeypatch.setattr(helpers, "_STANDIN_KORNIA", {**helpers._STANDIN_KORNIA, **_QUAD_MODULES})
    with helpers.standin_kornia(tmp_path) as kornia:
        origs = {(m, n): getattr(sys.modules[m], n) for m, names in _IMPORTERS.items() for n in names}
        ssd = sys.modules["kornia.feature.scale_space_detector"]
        before = ssd.ScaleSpaceDetector()  # built before install(): keeps the reference refiner it holds
        try:
            K.install(kornia)
            for (m, n), orig in origs.items():
                assert getattr(sys.modules[m], n) is getattr(Q, n), (m, n)
            det = ssd.ScaleSpaceDetector()
            assert type(det.subpix) is Q.AdaptiveQuadInterp3d and det._is_iterative_subpix
            assert det.subpix.strict_maxima_bonus == 0.0 and det.subpix.mode == "auto"
            assert type(sys.modules["kornia.feature.integrated"].sift_refiner()) is Q.ConvQuadInterp3d
            assert type(before.subpix) is origs[("kornia.feature.scale_space_detector", "AdaptiveQuadInterp3d")]
        finally:
            K.uninstall()
        for (m, n), orig in origs.items():
            assert getattr(sys.modules[m], n) is orig, (m, n)
