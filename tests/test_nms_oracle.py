"""Non-maximum suppression on the host (no GPU): the plain-torch restatement (tests/nms_restated.py) and the library's
composition both reproduce the reference's goldens bit for bit (NaN equals NaN, -0 and +0 differ), errors included; the
public signatures, defaults, reprs, buffers and validation match the reference's; a reference-layout state_dict loads
with strict=True; install() rebinds the five names on a stand-in package and on every module that imports them, and
skips a package without geometry/subpix/nms.py."""
import importlib
import inspect
import sys

import pytest
import torch

import helpers
import nms_restated as NR
from conftest import golden

K = importlib.import_module("kornia_b200")
N = importlib.import_module("kornia_b200.geometry.subpix.nms")
G = golden("nms")


def _same(a, b):
    assert a.shape == b.shape and a.dtype == b.dtype, (a.shape, b.shape, a.dtype, b.dtype)
    if a.dtype == torch.bool:
        return torch.equal(a, b)
    return bool(((a.view(torch.int32) == b.view(torch.int32)) | (a.isnan() & b.isnan())).all())


def _run(mod, op, kw, x):
    if op == "nms2d":
        return {"out": mod.nms2d(x, tuple(kw["kernel_size"]), kw["mask_only"])}
    if op == "nms3d":
        return {"out": mod.nms3d(x, tuple(kw["kernel_size"]), kw["mask_only"])}
    mx, mn = mod.nms3d_minmax(x)
    return {"max": mx, "min": mn}


@pytest.mark.parametrize("impl", ["restated", "composed"])
@pytest.mark.parametrize("name", G.names())
def test_reproduces_the_goldens(name, impl):
    op, kw, ins, outs = G.case(name)
    mod = NR if impl == "restated" else N
    if "error" in kw:
        with pytest.raises(RuntimeError) as e:
            _run(mod, op, kw, ins["input"])
        assert type(e.value).__name__ == kw["error"] and str(e.value) == kw["message"]
        return
    got = _run(mod, op, kw, ins["input"])
    for k, want in outs.items():
        assert _same(got[k], want), k


def test_goldens_cover_the_special_cases():
    names = G.names()
    for k in (3, 5, 7, 9, 15):
        for form in ("mask", "values"):
            assert f"nms2d_k{k}_special_{form}" in names and f"nms2d_k{k}_negpeaks_{form}" in names
    assert {"nms2d_error_4x4", "nms2d_error_3x5", "nms2d_error_5x3", "nms3d_error_5x5x5"} <= set(names)
    # the general form drops the negative isolated peaks that the explicit forms keep
    _, _, _, o3 = G.case("nms2d_k3_negpeaks_mask")
    _, _, _, o9 = G.case("nms2d_k9_negpeaks_mask")
    assert int(o3["out"].sum()) > 0 and int(o9["out"].sum()) < int(o3["out"].sum())


def _sig(fn):
    params = inspect.signature(fn).parameters.values()
    return "(" + ", ".join(p.name if p.default is inspect._empty else f"{p.name}={p.default!r}" for p in params) + ")"


def test_signatures_reprs_buffers_match_reference():
    assert _sig(N.nms2d) == "(input, kernel_size, mask_only=False)"
    assert _sig(N.nms3d) == "(input, kernel_size, mask_only=False)"
    assert _sig(N.nms3d_minmax) == "(input)"
    assert _sig(N.NonMaximaSuppression2d.__init__) == "(self, kernel_size)"
    assert _sig(N.NonMaximaSuppression2d.forward) == "(self, x, mask_only=False)"
    assert _sig(N.NonMaximaSuppression3d.forward) == "(self, x, mask_only=False)"
    m2 = N.NonMaximaSuppression2d((15, 15))
    m3 = N.NonMaximaSuppression3d((3, 3, 3))
    assert repr(m2) == "NonMaximaSuppression2d()" and repr(m3) == "NonMaximaSuppression3d()"
    assert list(m2.state_dict()) == ["kernel"] and list(m3.state_dict()) == []
    assert m2.kernel.shape == (225, 1, 15, 15) and m3.kernel.shape == (27, 1, 3, 3, 3)
    want = torch.eye(225)
    want[112, 112] = 0
    assert torch.equal(m2.kernel, want.view(225, 1, 15, 15))
    assert m2.padding == (7, 7, 7, 7) and m3.padding == (3, 3, 3, 3, 3, 3)
    assert N.NonMaximaSuppression2d((3, 5)).kernel.shape == (15, 1, 5, 3)
    for name in N.__all__:
        assert getattr(K.geometry, name) is getattr(N, name) and getattr(K.geometry.subpix, name) is getattr(N, name)
        assert name in K.geometry.__all__ and name in K.geometry.subpix.__all__


def test_reference_state_dict_loads_strict():
    # MultiResolutionDetector holds its NonMaximaSuppression2d as `nms`: its state_dict key is nms.kernel
    holder = torch.nn.Module()
    holder.nms = N.NonMaximaSuppression2d((15, 15))
    assert list(holder.state_dict()) == ["nms.kernel"]
    weight = torch.eye(225)
    weight[112, 112] = 0
    holder.load_state_dict({"nms.kernel": weight.view(225, 1, 15, 15)}, strict=True)


def test_errors_match_reference():
    x4, x5 = torch.rand(1, 1, 8, 8), torch.rand(1, 1, 3, 8, 8)
    for call, exc, arg in [
        (lambda: N.nms2d(x5, (3, 3)), AssertionError, x5.shape),
        (lambda: N.NonMaximaSuppression2d((3, 3))(x5), AssertionError, x5.shape),
        (lambda: N.nms2d(x4, [3, 3]), AssertionError, list),
        (lambda: N.nms2d(x4, (3, 3, 3)), AssertionError, (3, 3, 3)),
        (lambda: N.nms3d(x4, (3, 3, 3)), AssertionError, x4.shape),
        (lambda: N.nms3d(x5, [3, 3, 3]), AssertionError, list),
        (lambda: N.nms3d(x5, (3, 3)), AssertionError, (3, 3)),
        (lambda: N.nms3d_minmax(x4), AssertionError, x4.shape),
    ]:
        with pytest.raises(exc) as e:
            call()
        assert e.value.args == (arg,)


def test_values_gradient_is_upstream_times_mask():
    x = torch.rand(1, 2, 12, 13, dtype=torch.float64, requires_grad=True)
    for f in (lambda t: N.nms2d(t, (3, 3)), lambda t: N.nms2d(t, (9, 9)), lambda t: N.nms3d(t.view(1, 1, 2, 12, 13), (3, 3, 3))):
        out = f(x)
        g = torch.rand_like(out)
        (gx,) = torch.autograd.grad((out * g).sum(), [x])
        assert torch.equal(gx, (g * (out != 0)).view_as(x))


_NMS_MODULES = {
    "geometry/__init__": "from . import transform, calibration, subpix\nfrom .transform import warp_perspective, warp_affine, remap\n"
                         "from .subpix import *",
    "geometry/subpix/__init__": "from .nms import NonMaximaSuppression2d, NonMaximaSuppression3d, nms2d, nms3d, nms3d_minmax\n"
                                "from .spatial_soft_argmax import conv_soft_argmax3d",
    "geometry/subpix/nms": "def nms2d(): pass\ndef nms3d(): pass\ndef nms3d_minmax(): pass\n"
                           "class NonMaximaSuppression2d: pass\nclass NonMaximaSuppression3d: pass",
    "geometry/subpix/spatial_soft_argmax": "from .nms import nms3d\ndef conv_soft_argmax3d(): pass",
    "__init__": "from . import filters, geometry, metrics, losses, augmentation, feature",
    "feature/__init__": "from . import scale_space_detector, xfeat\nfrom .disk import detector\nfrom .aliked import aliked",
    "feature/scale_space_detector": "from kornia.geometry.subpix import NonMaximaSuppression2d, nms3d_minmax",
    "feature/disk/__init__": "",
    "feature/disk/detector": "from kornia.geometry.subpix import nms2d",
    "feature/xfeat": "from kornia.geometry.subpix import nms2d",
    "feature/aliked/__init__": "",
    "feature/aliked/aliked": "from kornia.geometry.subpix import nms2d",
}
# importer module -> names it holds
_IMPORTERS = {
    "kornia.geometry.subpix.nms": N.__all__,
    "kornia.geometry.subpix": N.__all__,
    "kornia.geometry": N.__all__,
    "kornia.geometry.subpix.spatial_soft_argmax": ["nms3d"],
    "kornia.feature.scale_space_detector": ["NonMaximaSuppression2d", "nms3d_minmax"],
    "kornia.feature.disk.detector": ["nms2d"],
    "kornia.feature.xfeat": ["nms2d"],
    "kornia.feature.aliked.aliked": ["nms2d"],
}


def test_install_rebinds_nms_everywhere(tmp_path, monkeypatch):
    monkeypatch.setattr(helpers, "_STANDIN_KORNIA", {**helpers._STANDIN_KORNIA, **_NMS_MODULES})
    with helpers.standin_kornia(tmp_path) as kornia:
        origs = {(m, n): getattr(sys.modules[m], n) for m, names in _IMPORTERS.items() for n in names}
        assert all(getattr(sys.modules["kornia.geometry.subpix.nms"], n) is origs[("kornia.geometry.subpix.nms", n)] for n in N.__all__)
        try:
            K.install(kornia)
            for (m, n), orig in origs.items():
                assert getattr(sys.modules[m], n) is getattr(N, n), (m, n)
        finally:
            K.uninstall()
        for (m, n), orig in origs.items():
            assert getattr(sys.modules[m], n) is orig, (m, n)


def test_install_skips_a_package_without_nms(tmp_path, monkeypatch):
    with helpers.standin_kornia(tmp_path) as kornia:  # no geometry/subpix at all
        try:
            K.install(kornia)
            assert kornia.filters.filter2d is K.filters.filter2d
            assert "kornia.geometry.subpix.nms" not in sys.modules
        finally:
            K.uninstall()
    partial = {**helpers._STANDIN_KORNIA, **_NMS_MODULES, "geometry/subpix/nms": "def nms2d(): pass"}
    partial["geometry/subpix/__init__"] = "from .nms import nms2d"
    partial.pop("geometry/subpix/spatial_soft_argmax")
    partial["geometry/__init__"] = "from . import transform, calibration, subpix"
    partial["feature/scale_space_detector"] = "from kornia.geometry.subpix import nms2d"
    monkeypatch.setattr(helpers, "_STANDIN_KORNIA", partial)
    with helpers.standin_kornia(tmp_path / "partial") as kornia:  # a module that defines only nms2d
        try:
            K.install(kornia)
            assert sys.modules["kornia.geometry.subpix.nms"].nms2d is N.nms2d
            assert sys.modules["kornia.feature.xfeat"].nms2d is N.nms2d
            assert not hasattr(sys.modules["kornia.geometry.subpix.nms"], "nms3d")
        finally:
            K.uninstall()
