"""ScalePyramid on the host (no GPU): the plain-torch restatement (tests/scale_pyramid_restated.py) reproduces the
reference's goldens and their input gradients; the public signature, defaults, repr and buffer names match the
reference's; install() rebinds the class on a stand-in package whose detector imports it, and still succeeds on a
package whose pyramid module does not define it."""
import importlib
import inspect
import sys

import pytest
import torch

import helpers
import scale_pyramid_restated as SR
from conftest import golden

K = importlib.import_module("kornia_b200")
P = importlib.import_module("kornia_b200.geometry.transform.pyramid")
G = golden("scale_pyramid")


@pytest.mark.parametrize("name", G.names())
def test_restatement_reproduces_the_goldens_and_their_gradients(name):
    op, kw, ins, outs = G.case(name)
    assert op == "ScalePyramid"
    x = ins["input"].clone().requires_grad_(True)
    pyr, sigmas, pds = SR.scale_pyramid(x, **kw)
    assert len(pyr) == len([k for k in outs if k.startswith("pyr")])
    for o, p in enumerate(pyr):
        want = outs[f"pyr{o}"]
        torch.testing.assert_close(p.detach(), want, rtol=0, atol=1e-5 * float(want.abs().max()))
        assert torch.equal(sigmas[o], outs[f"sig{o}"]) and torch.equal(pds[o], outs[f"pd{o}"])
    (g,) = torch.autograd.grad(sum((p * ins[f"cot{o}"]).sum() for o, p in enumerate(pyr)), [x])
    torch.testing.assert_close(g, outs["grad_input"], rtol=0, atol=1e-5 * float(outs["grad_input"].abs().max()))


def test_signature_defaults_repr_and_buffers_match_reference():
    # kornia/geometry/transform/pyramid.py:206-235,244-265
    params = inspect.signature(P.ScalePyramid.__init__).parameters.values()
    sig = "(" + ", ".join(p.name if p.default is inspect._empty else f"{p.name}={p.default!r}" for p in params) + ")"
    assert sig == "(self, n_levels=3, init_sigma=1.6, min_size=15, double_image=False, extra_levels=3)"
    sp = P.ScalePyramid()
    assert repr(sp) == ("ScalePyramid(n_levels=3, init_sigma=1.6, min_size=15, extra_levels=3, border=6, "
                        "sigma_step=1.2599210498948732, double_image=False)")
    assert list(sp.state_dict()) == ["_gk_init", "_gk_0", "_gk_1", "_gk_2", "_gk_3", "_gk_4"]
    assert [sp.state_dict()[k].shape[0] for k in sp.state_dict()] == [13, 11, 13, 17, 21, 25]
    assert (sp.n_levels, sp.extra_levels, sp.init_sigma, sp.min_size, sp.border, sp.double_image) == (3, 3, 1.6, 15, 6, False)
    assert list(P.ScalePyramid(3, 1.6, 16, extra_levels=2).state_dict()) == ["_gk_init", "_gk_0", "_gk_1", "_gk_2", "_gk_3"]
    assert [v.shape[0] for v in P.ScalePyramid(3, 1.6, 32, double_image=True).state_dict().values()] == [11, 11, 13, 17, 21, 25]
    nb = P.ScalePyramid(1, 0.25)
    assert nb._gk_init is None and list(nb.state_dict()) == ["_gk_0", "_gk_1", "_gk_2"]
    init, levels = SR.kernels()
    assert torch.equal(sp._gk_init, init) and all(torch.equal(getattr(sp, f"_gk_{i}"), k) for i, k in enumerate(levels))
    assert sp.get_kernel_size(1.5) == 13 and sp.get_kernel_size(1.25) == 11
    assert K.geometry.ScalePyramid is P.ScalePyramid and K.geometry.transform.ScalePyramid is P.ScalePyramid
    assert "ScalePyramid" in K.geometry.__all__ and "ScalePyramid" in K.geometry.transform.__all__


def test_loaded_state_dict_updates_the_kernel_taps():
    sp = P.ScalePyramid()
    sd = {k: v * 2 for k, v in sp.state_dict().items()}
    sp.load_state_dict(sd, strict=True)
    assert sp._host_taps["_gk_2"] == [float(v) for v in sd["_gk_2"].tolist()]


_DETECTOR_MODULES = {
    "geometry/transform/pyramid": "from kornia.filters import filter2d, gaussian_blur2d\nclass ScalePyramid:\n    pass",
    "geometry/transform/__init__": "from .imgwarp import warp_perspective, warp_affine, remap, get_perspective_transform\n"
                                   "from . import affwarp, crop2d, pyramid\nfrom .pyramid import ScalePyramid",
    "__init__": "from . import filters, geometry, metrics, losses, augmentation, feature",
    "feature/__init__": "from .scale_space_detector import ScaleSpaceDetector",
    "feature/scale_space_detector": "from kornia.geometry.transform import ScalePyramid\nclass ScaleSpaceDetector:\n    pass",
}


def test_install_rebinds_scale_pyramid(tmp_path, monkeypatch):
    monkeypatch.setattr(helpers, "_STANDIN_KORNIA", {**helpers._STANDIN_KORNIA, **_DETECTOR_MODULES})
    with helpers.standin_kornia(tmp_path) as kornia:
        pyr = sys.modules["kornia.geometry.transform.pyramid"]
        ssd = sys.modules["kornia.feature.scale_space_detector"]
        orig = pyr.ScalePyramid
        try:
            K.install(kornia)
            assert pyr.ScalePyramid is P.ScalePyramid
            assert kornia.geometry.transform.ScalePyramid is P.ScalePyramid
            assert ssd.ScalePyramid is P.ScalePyramid
        finally:
            K.uninstall()
        assert pyr.ScalePyramid is orig and ssd.ScalePyramid is orig


def test_install_skips_a_pyramid_module_without_scale_pyramid(tmp_path):
    with helpers.standin_kornia(tmp_path) as kornia:
        try:
            K.install(kornia)
            assert kornia.filters.filter2d is K.filters.filter2d
            assert not hasattr(sys.modules["kornia.geometry.transform.pyramid"], "ScalePyramid")
        finally:
            K.uninstall()
