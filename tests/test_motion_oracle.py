"""Motion blur on the host (no GPU): the restated reference against the goldens of the imported reference
(tests/golden/make_golden_motion.py), the public signatures and error behaviour, RandomMotionBlur's parameter stream, and
install() on stand-in packages with and without the motion modules."""
import importlib
import inspect

import pytest
import torch

import helpers
import motion_restated as MR
from conftest import golden

K = importlib.import_module("kornia_b200")
A = importlib.import_module("kornia_b200.augmentation")
G = golden("motion")


def _case(name):
    return G.case(name)


@pytest.mark.parametrize("name", G.names("get_motion_kernel2d"))
def test_oracle_reproduces_the_kernels(name):
    _, kw, ins, outs = _case(name)
    angle = ins.get("angle", kw.get("angle"))
    direction = ins.get("direction", kw.get("direction"))
    got = MR.get_motion_kernel2d(kw["kernel_size"], angle, direction, kw["mode"])
    assert torch.equal(got, outs["kernel"]), (got - outs["kernel"]).abs().max()


@pytest.mark.parametrize("name", G.names("motion_blur"))
def test_oracle_reproduces_motion_blur_and_its_gradients(name):
    _, kw, ins, outs = _case(name)
    x = ins["input"].clone().requires_grad_(True)
    batched = "angle" in ins
    angle = ins["angle"].clone().requires_grad_(True) if batched else kw["angle"]
    direction = ins["direction"].clone().requires_grad_(True) if batched else kw["direction"]
    kernel = MR.get_motion_kernel2d(kw["kernel_size"], angle, direction, kw["mode"])
    assert torch.equal(kernel.detach(), outs["kernel"])
    out = MR.motion_blur(x, kw["kernel_size"], angle, direction, kw["border_type"], kw["mode"])
    torch.testing.assert_close(out.detach(), outs["out"], rtol=1e-6, atol=1e-6)
    if batched:
        grads = torch.autograd.grad((out * outs["cot"]).sum(), [x, angle, direction], allow_unused=True)
        for g, key in zip(grads, ("grad_input", "grad_angle", "grad_direction")):
            g = torch.zeros_like(outs[key]) if g is None else g
            torch.testing.assert_close(g, outs[key], rtol=1e-5, atol=1e-5)


def test_signatures_match_reference():
    # kornia/filters/kernels_geometry.py:30-32, kornia/filters/motion.py (motion_blur, MotionBlur.__init__),
    # kornia/augmentation/_2d/intensity/motion_blur.py (RandomMotionBlur.__init__)
    KF = K.filters
    want = {
        KF.get_motion_kernel2d: "(kernel_size, angle, direction=0.0, mode='nearest')",
        KF.motion_blur: "(input, kernel_size, angle, direction, border_type='constant', mode='nearest')",
        KF.MotionBlur.__init__: "(self, kernel_size, angle, direction, border_type='constant', mode='nearest')",
        A.RandomMotionBlur.__init__: "(self, kernel_size, angle, direction, border_type='CONSTANT', resample='NEAREST', same_on_batch=False, "
                                     "p=0.5, keepdim=False)",
    }
    for fn, sig in want.items():
        params = inspect.signature(fn).parameters.values()
        got = "(" + ", ".join(p.name if p.default is inspect._empty else f"{p.name}={p.default!r}" for p in params) + ")"
        assert got == sig, fn.__qualname__
    for name in ("motion_blur", "MotionBlur", "get_motion_kernel2d"):
        assert name in KF.__all__ and getattr(KF, name) is getattr(importlib.import_module("kornia_b200.filters.motion"), name)
    assert "RandomMotionBlur" in A.__all__


def test_errors_match_the_reference():
    # validation runs before anything touches a device, so these raise the reference's errors on a machine without one
    KF = K.filters
    with pytest.raises(Exception, match="Kernel size must be an odd integer bigger than 2. Gotcha 4"):
        KF.get_motion_kernel2d(4, 30.0, 0.5)
    with pytest.raises(Exception, match="Kernel size must be an odd integer bigger than 2. Gotcha 1"):
        KF.get_motion_kernel2d(1, 30.0, 0.5)
    with pytest.raises(Exception, match="Shape dimension mismatch"):
        KF.get_motion_kernel2d(5, torch.zeros(2, 2), torch.zeros(2, 2))
    with pytest.raises(Exception, match="direction and angle must have the same length"):
        KF.get_motion_kernel2d(5, torch.zeros(3), torch.zeros(2))
    with pytest.raises(Exception, match="direction and angle must have the same length"):
        KF.get_motion_kernel2d(5, torch.zeros(3), 0.5)
    with pytest.raises(Exception, match="not in the same device and dtype"):
        KF.get_motion_kernel2d(5, torch.zeros(1), torch.zeros(1, dtype=torch.float64))
    with pytest.raises(AssertionError, match="`kernel_size` must be odd and greater than 3. Got 4."):
        A.RandomMotionBlur(4, 35.0, 0.5)
    with pytest.raises(AssertionError, match=r"`kernel_size` must be \(2,\) if it is a tuple"):
        A.RandomMotionBlur((3, 5, 7), 35.0, 0.5)
    with pytest.raises(TypeError, match="Unsupported type"):
        A.RandomMotionBlur([3, 5], 35.0, 0.5)
    with pytest.raises(ValueError):
        A.RandomMotionBlur(3, -35.0, 0.5)
    with pytest.raises(ValueError):
        A.RandomMotionBlur(3, 35.0, (-2.0, 0.5))


def _params(outs):
    return {k[len("param_"):]: v for k, v in outs.items() if k.startswith("param_")}


@pytest.mark.parametrize("name", G.names("RandomMotionBlur"))
def test_same_seed_same_parameters_as_the_reference(name):
    _, kw, ins, outs = _case(name)
    ctor = {k: (tuple(v) if isinstance(v, list) else v) for k, v in kw["ctor"].items()}
    aug = A.RandomMotionBlur(**ctor)
    torch.manual_seed(kw["seed"])
    got = aug.forward_parameters(tuple(ins["input"].shape))
    want = _params(outs)
    assert set(got) == set(want), (sorted(got), sorted(want))
    for k, w in want.items():
        assert got[k].shape == w.shape and got[k].dtype == w.dtype and got[k].device == w.device, (k, got[k], w)
        assert torch.equal(got[k], w), (k, got[k], w)


@pytest.mark.parametrize("name", G.names("RandomMotionBlur"))
def test_replayed_parameters_reproduce_the_reference_with_the_oracle(name, monkeypatch):
    _, kw, ins, outs = _case(name)
    ctor = {k: (tuple(v) if isinstance(v, list) else v) for k, v in kw["ctor"].items()}
    aug = A.RandomMotionBlur(**ctor)
    monkeypatch.setattr(A, "motion_blur", lambda input, **k: MR.motion_blur(input, **k))
    out = aug(ins["input"], params=_params(outs))
    torch.testing.assert_close(out, outs["out"], rtol=1e-6, atol=1e-6)


_MOTION_MODULES = {
    "filters/kernels_geometry": "def get_motion_kernel2d(): pass",
    "filters/motion": "from .filter import filter2d\nfrom .kernels_geometry import get_motion_kernel2d\ndef motion_blur(): pass",
    "filters/__init__": helpers._STANDIN_KORNIA["filters/__init__"] + "\nfrom .kernels_geometry import get_motion_kernel2d\nfrom .motion import motion_blur",
    "augmentation/_2d/intensity/__init__": "from . import gaussian_blur, motion_blur",
    "augmentation/_2d/intensity/motion_blur": "from kornia.filters import motion_blur",
}


def test_install_rebinds_every_motion_importer(tmp_path, monkeypatch):
    monkeypatch.setattr(helpers, "_STANDIN_KORNIA", {**helpers._STANDIN_KORNIA, **_MOTION_MODULES})
    with helpers.standin_kornia(tmp_path) as kornia:
        import sys

        motion = sys.modules["kornia.filters.motion"]
        geo = sys.modules["kornia.filters.kernels_geometry"]
        aug = sys.modules["kornia.augmentation._2d.intensity.motion_blur"]
        orig_blur, orig_kernel = motion.motion_blur, geo.get_motion_kernel2d
        try:
            K.install(kornia)
            assert motion.motion_blur is K.filters.motion_blur and kornia.filters.motion_blur is K.filters.motion_blur
            assert aug.motion_blur is K.filters.motion_blur
            assert geo.get_motion_kernel2d is K.filters.get_motion_kernel2d
            assert motion.get_motion_kernel2d is K.filters.get_motion_kernel2d
            assert kornia.filters.get_motion_kernel2d is K.filters.get_motion_kernel2d
            assert motion.filter2d is K.filters.filter2d
            # the package attribute that names the submodule is not a function to rebind
            assert inspect.ismodule(sys.modules["kornia.augmentation._2d.intensity"].motion_blur)
        finally:
            K.uninstall()
        assert motion.motion_blur is orig_blur and geo.get_motion_kernel2d is orig_kernel


def test_install_skips_motion_modules_a_package_lacks(tmp_path):
    with helpers.standin_kornia(tmp_path) as kornia:
        try:
            K.install(kornia)
            assert kornia.filters.filter2d is K.filters.filter2d
            assert not hasattr(kornia.filters, "motion_blur")
        finally:
            K.uninstall()
