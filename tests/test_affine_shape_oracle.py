"""PatchAffineShapeEstimator and LAFAffineShapeEstimator on the host (no GPU): the plain-torch restatement
(tests/affine_shape_restated.py) and the library's compositions, with ``spatial_gradient`` and ``pyrdown`` swapped for the
restated ones, reproduce the reference's goldens -- the degenerate (constant, stripe, unbuilt-level) shapes, negative b,
a non-default eps, extra images, non-finite LAFs and the gradients with respect to the image and the LAFs included; the
LAF helpers reproduce theirs; the signatures, reprs, errors, the operators' fake kernels and their checks match; install()
rebinds both classes on a stand-in package with the reference's feature/ layout, and uninstall() restores them."""
import importlib
import inspect
import sys

import pytest
import torch
from torch import nn

import affine_shape_restated as AR
import helpers
import sift_restated as SR
from conftest import golden
from oracle import kornia_restated as R

K = importlib.import_module("kornia_b200")
F = importlib.import_module("kornia_b200.feature")
AS = importlib.import_module("kornia_b200.feature.affine_shape")
LAF = importlib.import_module("kornia_b200.feature.laf")
G = golden("affine_shape")


class _HostGradient(nn.Module):
    def forward(self, x):
        return SR.gradient(x, SR.SOBEL)


@pytest.fixture
def host(monkeypatch):
    """The library's pyrdown and spatial_gradient run CUDA kernels: on the host the compositions run over the restated ones."""
    monkeypatch.setattr(LAF, "pyrdown", R.pyrdown)
    monkeypatch.setattr(AS, "SpatialGradient", lambda *a: _HostGradient())


def close(got, want, atol=1e-5):
    assert got.shape == want.shape and got.dtype == want.dtype, (got.shape, want.shape, got.dtype, want.dtype)
    assert torch.equal(got.isnan(), want.isnan())
    ok = ~want.isnan()
    torch.testing.assert_close(got[ok], want[ok], rtol=0, atol=atol * max(1.0, float(want[ok].abs().max()) if ok.any() else 1.0))


LAF_CASES = G.names("laf")
PATCH_CASES = G.names("patch")
ERRORS = G.names("error")


def _laf_module(kw):
    return F.LAFAffineShapeEstimator(kw["PS"], F.PatchAffineShapeEstimator(kw["PS"], eps=kw["eps"]), kw["preserve_orientation"])


def test_the_goldens_cover_what_they_promise():
    kws = [G.case(n)[1] for n in LAF_CASES]
    assert {k["PS"] for k in kws} == {19, 32, 41} and {k["preserve_orientation"] for k in kws} == {True, False}
    assert {k["eps"] for k in kws} > {1e-10} and any("grad_img" in G.case(n)[3] for n in LAF_CASES)
    # constant and stripe images take the circular branch: the output is the scale times a rotation
    for name in ("laf_constant_B1_64x80_PS32_upright", "laf_stripes_B1_90x110_PS19_upright"):
        _, _, ins, outs = G.case(name)
        o, s = outs["out"], LAF.get_laf_scale(ins["laf"])
        torch.testing.assert_close(o[..., :2, :2], s * torch.eye(2).expand_as(o[..., :2, :2]), rtol=1e-5, atol=1e-5)
    # negative b among the patch cases
    _, _, ins, outs = G.case("patch_mix_P19")
    assert (outs["out"][..., 1] < 0).any() and (outs["out"] == torch.tensor([1.0, 0.0, 1.0])).all(-1).any()
    assert G.case("laf_nonfinite")[3]["out"].isnan().any() and len(ERRORS) == 7


@pytest.mark.parametrize("name", LAF_CASES)
def test_restatement_reproduces_the_golden(name):
    _, kw, ins, outs = G.case(name)
    close(AR.laf_shape(ins["img"], ins["laf"], kw["PS"], kw["eps"], kw["preserve_orientation"]), outs["out"])


@pytest.mark.parametrize("name", PATCH_CASES)
def test_patch_restatement_reproduces_the_golden(name):
    _, kw, ins, outs = G.case(name)
    close(AR.patch_shape(ins["patch"], AR.weighting(kw["patch_size"]), kw["eps"]), outs["out"])


@pytest.mark.parametrize("name", LAF_CASES)
def test_library_composition_reproduces_the_golden(name, host):
    _, kw, ins, outs = G.case(name)
    m = _laf_module(kw)
    if "grad_img" in outs:
        img, laf = ins["img"].clone().requires_grad_(True), ins["laf"].clone().requires_grad_(True)
        out = m(laf, img)
        gi, gl = torch.autograd.grad((out * outs["cot"]).sum(), [img, laf])
        close(out.detach(), outs["out"])
        close(gi, outs["grad_img"], 1e-4)
        close(gl, outs["grad_laf"], 1e-4)
    else:
        close(m(ins["laf"], ins["img"]), outs["out"])


@pytest.mark.parametrize("name", PATCH_CASES)
def test_library_patch_composition_reproduces_the_golden(name, host):
    _, kw, ins, outs = G.case(name)
    close(F.PatchAffineShapeEstimator(kw["patch_size"], kw["eps"])(ins["patch"]), outs["out"])


def test_the_laf_helpers_reproduce_the_golden():
    _, _, ins, outs = G.case("helpers")
    laf, ang = ins["laf"], ins["angle"]
    close(F.make_upright(laf), outs["make_upright"])
    close(F.scale_laf(laf, ins["coef"]), outs["scale_laf"])
    close(F.scale_laf(laf, 0.75), outs["scale_laf_float"])
    close(F.ellipse_to_laf(ins["ells"]), outs["ellipse_to_laf"])
    close(F.get_laf_orientation(laf), outs["get_laf_orientation"], 1e-5)
    close(F.set_laf_orientation(laf, ang), outs["set_laf_orientation"])
    close(F.rotate_laf(laf, ang), outs["rotate_laf"])
    with pytest.raises(TypeError):
        F.scale_laf(laf, 2)


@pytest.mark.parametrize("name", ERRORS)
def test_the_public_modules_raise_the_references_errors(name, host):
    _, kw, ins, _ = G.case(name)
    if kw["op"] == "laf":
        call = lambda: F.LAFAffineShapeEstimator(kw["PS"])(ins["laf"], ins["img"])  # noqa: E731
    else:
        call = lambda: F.PatchAffineShapeEstimator(kw["PS"])(ins["patch"])  # noqa: E731
    with pytest.raises(Exception) as e:
        call()
    want = kw["error"]
    assert type(e.value).__name__ == want or (want == "ShapeError" and "Shape" in type(e.value).__name__), (type(e.value), want)
    if want != "ShapeError":
        assert str(e.value) == kw["message"]


def test_signatures_reprs_and_defaults_match_the_reference():
    p = inspect.signature(F.PatchAffineShapeEstimator).parameters
    assert list(p) == ["patch_size", "eps"] and p["patch_size"].default == 19 and p["eps"].default == 1e-10
    p = inspect.signature(F.LAFAffineShapeEstimator).parameters
    assert list(p) == ["patch_size", "affine_shape_detector", "preserve_orientation"]
    assert p["patch_size"].default == 32 and p["affine_shape_detector"].default is None and p["preserve_orientation"].default is True
    m = F.LAFAffineShapeEstimator()
    assert repr(m) == ("LAFAffineShapeEstimator(patch_size=32, affine_shape_detector=PatchAffineShapeEstimator(patch_size=32, eps=1e-10), "
                       "preserve_orientation=True)")
    assert type(m.affine_shape_detector) is F.PatchAffineShapeEstimator and m.affine_shape_detector.patch_size == 32
    assert m.affine_shape_detector.weighting.shape == (1, 32, 32) and m.state_dict() == {}
    assert list(inspect.signature(F.make_upright).parameters) == ["laf", "eps"]
    assert list(inspect.signature(F.ellipse_to_laf).parameters) == ["ells"]
    for fn in (F.set_laf_orientation, F.rotate_laf):
        assert list(inspect.signature(fn).parameters) == ["LAF", "angles_degrees"]


def test_the_kernel_is_taken_only_by_the_default_detector():
    class Custom(F.PatchAffineShapeEstimator):
        pass

    laf, img = torch.zeros(1, 2, 2, 3), torch.zeros(1, 1, 40, 50)
    # CPU tensors never take the kernel; the detector tests come first and do not depend on the device
    assert not F.LAFAffineShapeEstimator(19, Custom(19))._fused_ok(laf, img)
    assert not F.LAFAffineShapeEstimator(19, F.PatchAffineShapeEstimator(32))._fused_ok(laf, img)
    assert not F.LAFAffineShapeEstimator(65)._fused_ok(laf, img)


def test_the_operator_fake_kernels_and_their_checks():
    ops = torch.ops.kornia_b200
    m = lambda *shape, **kw: torch.empty(*shape, device="meta", **kw)  # noqa: E731
    assert ops.patch_affine_shape_fwd(m(7, 1, 19, 19), m(1, 19, 19), 1e-10).shape == (7, 1, 3)
    levels = [m(2, 1, 100, 120), m(2, 1, 50, 60)]
    assert ops.laf_affine_shape_fwd(levels, m(2, 7, 2, 3), m(1, 32, 32), 32, 1e-10, True).shape == (2, 7, 2, 3)
    for x, w in ((m(7, 2, 19, 19), m(19, 19)), (m(7, 1, 19, 19), m(18, 18)), (m(7, 1, 19, 19), m(19, 19, dtype=torch.float64))):
        with pytest.raises(RuntimeError):
            ops.patch_affine_shape_fwd(x, w, 1e-10)
    bad = [([m(2, 3, 100, 120)], m(2, 7, 2, 3), m(32, 32)),                        # three channels
           ([m(2, 1, 100, 120), m(2, 1, 51, 60)], m(2, 7, 2, 3), m(32, 32)),     # not a halving
           ([m(1, 1, 100, 120)], m(2, 7, 2, 3), m(32, 32)),                      # fewer images than LAF sets
           ([m(2, 1, 100, 120)], m(2, 7, 3, 3), m(32, 32)),                      # LAF shape
           ([m(2, 1, 100, 120)], m(2, 7, 2, 3), m(19, 19)),                      # weighting size
           ([m(2, 1, 100, 120)], m(2, 7, 2, 3), m(32, 32, dtype=torch.float64)),  # weighting dtype
           ([], m(2, 7, 2, 3), m(32, 32))]
    for lv, laf, w in bad:
        with pytest.raises(RuntimeError):
            ops.laf_affine_shape_fwd(lv, laf, w, 32, 1e-10, True)
    ops_mod = importlib.import_module("kornia_b200._ops")
    assert {"patch_affine_shape_fwd", "laf_affine_shape_fwd"} <= set(ops_mod.OPERATORS)


_AFFINE_MODULES = {
    "__init__": "from . import filters, geometry, metrics, losses, augmentation, feature",
    "feature/__init__": "from .affine_shape import PatchAffineShapeEstimator, LAFAffineShapeEstimator\nfrom . import scale_space_detector",
    "feature/affine_shape": "class PatchAffineShapeEstimator: pass\nclass LAFAffineShapeEstimator: pass",
    "feature/scale_space_detector": "from .affine_shape import LAFAffineShapeEstimator\n",
}


def test_install_rebinds_both_classes_and_uninstall_restores_them(tmp_path, monkeypatch):
    monkeypatch.setattr(helpers, "_STANDIN_KORNIA", {**helpers._STANDIN_KORNIA, **_AFFINE_MODULES})
    with helpers.standin_kornia(tmp_path) as kornia:
        aff = sys.modules["kornia.feature.affine_shape"]
        ssd = sys.modules["kornia.feature.scale_space_detector"]
        orig_p, orig_l = aff.PatchAffineShapeEstimator, aff.LAFAffineShapeEstimator
        try:
            K.install(kornia)
            assert aff.PatchAffineShapeEstimator is F.PatchAffineShapeEstimator and aff.LAFAffineShapeEstimator is F.LAFAffineShapeEstimator
            assert kornia.feature.LAFAffineShapeEstimator is F.LAFAffineShapeEstimator and ssd.LAFAffineShapeEstimator is F.LAFAffineShapeEstimator
            assert kornia.feature.PatchAffineShapeEstimator is F.PatchAffineShapeEstimator
        finally:
            K.uninstall()
        assert aff.PatchAffineShapeEstimator is orig_p and aff.LAFAffineShapeEstimator is orig_l
        assert kornia.feature.LAFAffineShapeEstimator is orig_l and ssd.LAFAffineShapeEstimator is orig_l
