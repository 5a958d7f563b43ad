"""extract_patches_from_pyramid / extract_patches_simple on the host (no GPU): the plain-torch restatement
(tests/patches_restated.py) and the library's compositions, with ``pyrdown`` swapped for the oracle's, reproduce the
reference's goldens -- every level choice, the zero patches of levels the pyramid never built, the extra-image and
one-pixel cases, gradients with respect to the image and the LAFs included; the signatures, the errors, the operator's
fake kernel and its checks match; install() rebinds both names wherever the reference imports them."""
import importlib
import inspect
import sys

import pytest
import torch

import helpers
import patches_restated as PR
from conftest import golden
from oracle import kornia_restated as R

K = importlib.import_module("kornia_b200")
F = importlib.import_module("kornia_b200.feature")
LAF = importlib.import_module("kornia_b200.feature.laf")
G = golden("patches")


@pytest.fixture
def host_pyrdown(monkeypatch):
    """The library's pyrdown runs CUDA kernels: on the host its composition runs over the oracle's."""
    monkeypatch.setattr(LAF, "pyrdown", R.pyrdown)


def _library(fn):
    return {"pyramid": LAF._composed_extract_pyramid, "simple": LAF._composed_extract_simple}[fn]


def close(got, want, atol=1e-5):
    assert got.shape == want.shape and got.dtype == want.dtype, (got.shape, want.shape, got.dtype, want.dtype)
    assert torch.equal(got.isnan(), want.isnan())
    ok = ~want.isnan()
    torch.testing.assert_close(got[ok], want[ok], rtol=0, atol=atol)


CASES = G.names("patches")
ERRORS = G.names("error")


def test_the_goldens_cover_what_they_promise():
    kws = [G.case(n)[1] for n in CASES]
    assert {k["PS"] for k in kws} == {19, 32, 41} and {k["fn"] for k in kws} == {"pyramid", "simple"}
    assert {k["normalize"] for k in kws} == {True, False}
    assert any("grad_img" in G.case(n)[3] for n in CASES)
    # 100 x 120 at PS = 32: the pyramid stops after level 1, so level-2 patches come back as zeros
    op, kw, ins, outs = G.case("pyramid_noise_B2C3_100x120_PS32_norm")
    assert (outs["out"].flatten(2).abs().amax(-1) == 0).any()
    assert {k["message"] for k in (G.case(n)[1] for n in ERRORS)}


@pytest.mark.parametrize("name", CASES)
def test_restatement_reproduces_the_golden(name):
    _, kw, ins, outs = G.case(name)
    got = PR.extract(ins["img"], ins["laf"], kw["PS"], kw["normalize"], kw["fn"] == "pyramid")
    close(got, outs["out"])


@pytest.mark.parametrize("name", CASES)
def test_library_composition_reproduces_the_golden(name, host_pyrdown):
    _, kw, ins, outs = G.case(name)
    fn = _library(kw["fn"])
    if "grad_img" in outs:
        img, laf = ins["img"].clone().requires_grad_(True), ins["laf"].clone().requires_grad_(True)
        out = fn(img, laf, kw["PS"], kw["normalize"])
        gi, gl = torch.autograd.grad((out * outs["cot"]).sum(), [img, laf])
        close(out.detach(), outs["out"])
        close(gi, outs["grad_img"], 1e-4)
        close(gl, outs["grad_laf"], 1e-3 * max(1.0, float(outs["grad_laf"].abs().max())))
    else:
        close(fn(ins["img"], ins["laf"], kw["PS"], kw["normalize"]), outs["out"])


@pytest.mark.parametrize("name", ERRORS)
def test_the_public_functions_raise_the_references_errors(name, host_pyrdown):
    _, kw, ins, _ = G.case(name)
    fn = {"pyramid": F.extract_patches_from_pyramid, "simple": F.extract_patches_simple}[kw["fn"]]
    with pytest.raises(Exception) as e:
        fn(ins["img"], ins["laf"], kw["PS"], kw["normalize"])
    want = kw["error"]
    assert type(e.value).__name__ == want or (want == "ShapeError" and "Shape" in type(e.value).__name__), (type(e.value), want)
    if want != "ShapeError":
        assert str(e.value) == kw["message"]


def test_signatures_match_the_reference():
    for fn in (F.extract_patches_from_pyramid, F.extract_patches_simple):
        ps = inspect.signature(fn).parameters
        assert list(ps) == ["img", "laf", "PS", "normalize_lafs_before_extraction"]
        assert ps["PS"].default == 32 and ps["normalize_lafs_before_extraction"].default is True
    assert list(inspect.signature(F.generate_patch_grid_from_normalized_LAF).parameters) == ["img", "LAF", "PS"]
    for fn in (F.normalize_laf, F.denormalize_laf):
        assert list(inspect.signature(fn).parameters) == ["LAF", "images"]


def test_output_dtypes_follow_the_reference(host_pyrdown):
    img, laf = torch.rand(1, 1, 40, 50, dtype=torch.float64), torch.tensor([[[[8.0, 0, 20], [0, 8, 20]]]], dtype=torch.float64)
    assert F.extract_patches_simple(img, laf, 8).dtype == torch.float64  # a cat of grid_sample outputs: img.dtype
    assert F.extract_patches_from_pyramid(img, laf, 8).dtype == torch.float64  # allocated from nlaf


def test_built_levels_follow_the_reference_loop():
    for h, w, PS in [(100, 120, 32), (1080, 1920, 41), (1080, 1920, 19), (480, 640, 32), (15, 23, 19), (64, 64, 32), (63, 200, 32),
                     (2, 2, 1), (1, 40, 19)]:
        n, level, top = 1, (h, w), max(1, min(h, w) // PS)
        for _ in range(top - 1):
            level = (level[0] // 2, level[1] // 2)
            if min(level) < PS:
                break
            n += 1
        assert LAF._built_levels(h, w, PS) == n, (h, w, PS)
    assert LAF._built_levels(100, 120, 32) == 2 and LAF._built_levels(1080, 1920, 41) == 5 and LAF._built_levels(1080, 1920, 19) == 6


def test_the_operator_fake_kernel_and_its_checks():
    ops = torch.ops.kornia_b200
    m = lambda *shape, **kw: torch.empty(*shape, device="meta", **kw)  # noqa: E731
    levels = [m(2, 3, 100, 120), m(2, 3, 50, 60)]
    assert ops.extract_patches_fwd(levels, m(2, 7, 2, 3), 32, True, True).shape == (2, 7, 3, 32, 32)
    assert ops.extract_patches_fwd(levels[:1], m(1, 5, 2, 3), 19, False, False).shape == (1, 5, 3, 19, 19)
    bad = [([m(2, 3, 100, 120), m(2, 3, 51, 60)], m(2, 7, 2, 3), 32, True),     # not a halving
           ([m(2, 3, 100, 120), m(2, 1, 50, 60)], m(2, 7, 2, 3), 32, True),     # channels differ
           ([m(2, 3, 100, 120), m(1, 3, 50, 60)], m(2, 7, 2, 3), 32, True),     # batch differs
           ([m(1, 3, 100, 120)], m(2, 7, 2, 3), 32, True),                      # fewer images than LAF sets
           ([m(2, 3, 100, 120)], m(2, 7, 3, 3), 32, True),                      # LAF shape
           ([m(2, 3, 100, 120)], m(2, 7, 2, 3, dtype=torch.float64), 32, True),  # LAF dtype
           ([m(2, 3, 100, 120)], m(2, 7, 2, 3), 0, True),                       # PS
           (levels, m(2, 7, 2, 3), 32, False),                                  # several levels without level selection
           ([], m(2, 7, 2, 3), 32, True)]
    for lv, laf, PS, select in bad:
        with pytest.raises(RuntimeError):
            ops.extract_patches_fwd(lv, laf, PS, True, select)
    assert "extract_patches_fwd" in importlib.import_module("kornia_b200._ops").OPERATORS


_LAF_MODULES = {
    "__init__": "from . import filters, geometry, metrics, losses, augmentation, feature",
    "feature/__init__": "from .laf import extract_patches_from_pyramid, extract_patches_simple\nfrom . import integrated, orientation, affine_shape",
    "feature/laf": "def extract_patches_from_pyramid(): pass\ndef extract_patches_simple(): pass",
    "feature/integrated": "from .laf import extract_patches_from_pyramid\n",
    "feature/orientation": "from .laf import extract_patches_from_pyramid\n",
    "feature/affine_shape": "from .laf import extract_patches_from_pyramid\n",
}


def test_install_rebinds_the_extraction_wherever_it_is_imported(tmp_path, monkeypatch):
    monkeypatch.setattr(helpers, "_STANDIN_KORNIA", {**helpers._STANDIN_KORNIA, **_LAF_MODULES})
    with helpers.standin_kornia(tmp_path) as kornia:
        mods = [sys.modules[f"kornia.feature.{m}"] for m in ("laf", "integrated", "orientation", "affine_shape")]
        orig = mods[0].extract_patches_from_pyramid
        try:
            K.install(kornia)
            for mod in mods + [kornia.feature]:
                assert mod.extract_patches_from_pyramid is F.extract_patches_from_pyramid, mod
            assert mods[0].extract_patches_simple is F.extract_patches_simple and kornia.feature.extract_patches_simple is F.extract_patches_simple
        finally:
            K.uninstall()
        assert all(mod.extract_patches_from_pyramid is orig for mod in mods)
