"""SIFTDescriptor and PatchDominantGradientOrientation on the host (no GPU): the plain-torch restatement
(tests/sift_restated.py) and the library's compositions reproduce the reference's goldens to 1e-5 with identical NaN
positions, gradients with respect to the input and the modules' weights included; the public signatures, reprs,
state_dict keys, strict loading of a reference-shaped state_dict, the kernel helpers and the errors match the
reference's; install() rebinds the three names on a stand-in package with the reference's feature/ layout."""
import importlib
import inspect
import sys

import pytest
import torch
from torch import nn

import helpers
import sift_restated as SR
from conftest import golden

K = importlib.import_module("kornia_b200")
F = importlib.import_module("kornia_b200.feature")
SD = importlib.import_module("kornia_b200.feature.siftdesc")
OR = importlib.import_module("kornia_b200.feature.orientation")
KF = importlib.import_module("kornia_b200.filters")
G = golden("sift")


def close(got, want, atol=1e-5):
    assert got.shape == want.shape, (got.shape, want.shape)
    assert torch.equal(got.isnan(), want.isnan())
    ok = ~want.isnan()
    torch.testing.assert_close(got[ok], want[ok], rtol=0, atol=atol)


class _HostGradient(nn.Module):
    def forward(self, x):
        return SR.gradient(x, SR.SOBEL)


@pytest.fixture
def host_gradients(monkeypatch):
    """The library's spatial_gradient is CUDA-only: on the host its compositions run over the restated stencils."""
    monkeypatch.setattr(SD, "spatial_gradient", lambda x, mode: SR.gradient(x, SR.DIFF if mode == "diff" else SR.SOBEL))


def _library_module(op, kw, ins=None):
    if op == "sift":
        return F.SIFTDescriptor(kw["patch_size"], kw["num_ang_bins"], kw["num_spatial_bins"], kw["rootsift"], kw["clipval"])
    m = F.PatchDominantGradientOrientation(kw["patch_size"], kw["num_angular_bins"])
    if ins is not None and "smooth" in ins:
        m.load_state_dict({"angular_smooth.weight": ins["smooth"]}, strict=True)
    m.gradient = _HostGradient()
    return m


def tie_angles(x, m, n):
    """The angles of the first and the last maximal smoothed bin (restated), for the exact-tie golden."""
    _, hist = SR.orientation(x, m.weighting, m.angular_smooth.weight.detach(), n, return_hist=True)
    top = (hist[0] == hist[0].max()).nonzero().view(-1).tolist()

    def angle(i):
        l, r = hist[0, (i - 1) % n], hist[0, (i + 1) % n]
        return float(-((2.0 * SR.PI * (i + 0.5 * (l - r) / (l + r - 2.0 * hist[0, i])) / float(n)) - SR.PI))

    return top, angle(top[0]), angle(top[-1])


def _restated(op, kw, x, m):
    if op == "sift":
        ks, stride, pad = SR.sift_params(kw["patch_size"], kw["num_spatial_bins"])
        return SR.sift(x, SR.sift_gk(kw["patch_size"]), m.pk.weight, kw["num_ang_bins"], kw["num_spatial_bins"], stride, pad, kw["rootsift"],
                       kw["clipval"])
    return SR.orientation(x, m.weighting, m.angular_smooth.weight, kw["num_angular_bins"])


def _weight(op, m):
    return m.pk.weight if op == "sift" else m.angular_smooth.weight


CASES = G.names("sift") + G.names("orientation")


@pytest.mark.parametrize("impl", ["restated", "library"])
@pytest.mark.parametrize("name", CASES)
def test_goldens_and_their_gradients(name, impl, host_gradients):
    op, kw, ins, outs = G.case(name)
    m = _library_module(op, kw, ins)
    run = (lambda x: _restated(op, kw, x, m)) if impl == "restated" else m
    x = ins["input"]
    if "error" in kw:
        assert kw["error"] == "RuntimeError"  # N = 0: view(B, -1) of an empty tensor
        with pytest.raises(RuntimeError, match="cannot reshape tensor of 0 elements"):
            with torch.no_grad():
                run(x)
        return
    if "grad_input" not in outs:
        with torch.no_grad():
            got = run(x)
        close(got, outs["out"])
        if kw.get("tie"):  # two non-adjacent maximal bins: torch.max's first index decides, 4 bins from the last one
            top, first, last = tie_angles(x, m, kw["num_angular_bins"])
            assert top == [kw["first_index"], kw["last_index"]]
            assert abs(float(got[0]) - first) < 1e-6 and abs(float(got[0]) - last) > 0.1
        return
    xg = x.clone().requires_grad_(True)
    out = run(xg)
    close(out.detach(), outs["out"])
    w = _weight(op, m)
    gx, gw = torch.autograd.grad((out * outs["cot"]).sum(), [xg, w])
    # the sub-bin fit divides by a difference of histogram values: its gradients carry fp32 reordering noise near 1e-5 relative
    close(gx, outs["grad_input"], 1e-4 * max(1.0, float(outs["grad_input"].abs().max())))
    close(gw, outs["grad_weight"], 1e-4 * max(1.0, float(outs["grad_weight"].abs().max())))


def test_sift_describe_golden(host_gradients):
    _, _, ins, outs = G.case("sift_describe_default")
    with torch.no_grad():
        close(F.sift_describe(ins["input"]), outs["out"])


def test_kernel_helpers_match_the_reference():
    for name in G.names("pooling_kernel"):
        _, kw, _, outs = G.case(name)
        assert torch.equal(F.get_sift_pooling_kernel(kw["ksize"]), outs["out"])
    _, kw, _, _ = G.case("bin_ksize_stride_pad")
    for key, want in kw["params"].items():
        p, s = map(int, key.split("_"))
        assert list(F.get_sift_bin_ksize_stride_pad(p, s)) == want
    for name in G.names("discrete"):
        _, kw, ins, outs = G.case(name)
        got = KF.get_gaussian_discrete_kernel1d(kw["kernel_size"], ins.get("sigma", kw.get("sigma")))
        torch.testing.assert_close(got, outs["out"], rtol=0, atol=1e-7)


def _sig(fn):
    params = inspect.signature(fn).parameters.values()
    return "(" + ", ".join(p.name if p.default is inspect._empty else f"{p.name}={p.default!r}" for p in params) + ")"


def test_signatures_reprs_and_state_dicts_match_the_reference():
    want = {
        F.SIFTDescriptor.__init__: "(self, patch_size=41, num_ang_bins=8, num_spatial_bins=4, rootsift=True, clipval=0.2)",
        F.sift_describe: "(input, patch_size=41, num_ang_bins=8, num_spatial_bins=4, rootsift=True, clipval=0.2)",
        F.get_sift_pooling_kernel: "(ksize=25)",
        F.get_sift_bin_ksize_stride_pad: "(patch_size, num_spatial_bins)",
        F.PatchDominantGradientOrientation.__init__: "(self, patch_size=32, num_angular_bins=36, eps=1e-08)",
        KF.get_gaussian_discrete_kernel1d: "(kernel_size, sigma, force_even=False, device=None, dtype=None)",
    }
    for fn, sig in want.items():
        assert _sig(fn) == sig, fn.__qualname__
    for name in G.names("sift") + G.names("orientation"):
        _, kw, _, _ = G.case(name)
        assert repr(_library_module(*G.case(name)[:2])).startswith(kw["repr"].split("(")[0])
        m = _library_module(*G.case(name)[:2])
        if isinstance(m, OR.PatchDominantGradientOrientation):
            m.gradient = OR.SpatialGradient("sobel", 1)
        assert repr(m) == kw["repr"]
    d = F.SIFTDescriptor()
    assert list(d.state_dict()) == ["pk.weight"] and d.eps == 1e-10 and isinstance(d.pk, nn.Conv2d)
    assert (d.bin_ksize, d.bin_stride, d.pad) == (16, 10, 4) and d.gk.shape == (1, 41, 41) and not isinstance(d.gk, nn.Parameter)
    assert torch.equal(d.get_pooling_kernel(), d.pk.weight.detach()) and torch.equal(d.get_weighting_kernel(), d.gk)
    ref_shaped = {"pk.weight": torch.rand(1, 1, 16, 16)}
    d.load_state_dict(ref_shaped, strict=True)
    assert torch.equal(d.pk.weight.detach(), ref_shaped["pk.weight"])
    o = F.PatchDominantGradientOrientation()
    assert list(o.state_dict()) == ["angular_smooth.weight"] and o.num_ang_bins == 36 and o.eps == 1e-8
    assert isinstance(o.gradient, KF.SpatialGradient) and o.weighting.shape == (1, 32, 32)
    assert o.angular_smooth.padding_mode == "circular" and o.angular_smooth.weight.requires_grad
    torch.testing.assert_close(o.angular_smooth.weight.detach().view(5), KF.get_gaussian_discrete_kernel1d(5, 1.6).view(5), rtol=0, atol=0)
    o.load_state_dict({"angular_smooth.weight": torch.rand(1, 1, 5)}, strict=True)
    for name in ("SIFTDescriptor", "sift_describe", "get_sift_pooling_kernel", "get_sift_bin_ksize_stride_pad",
                 "PatchDominantGradientOrientation"):
        assert name in F.__all__


def test_errors_match_the_reference():
    calls = {
        "incompatible": lambda: F.SIFTDescriptor(4, 8, 4),
        "incompatible_fn": lambda: F.get_sift_bin_ksize_stride_pad(10, 6),
        "sift_shape": lambda: F.SIFTDescriptor(32)(torch.zeros(2, 1, 41, 41)),
        "sift_ndim": lambda: F.SIFTDescriptor(32)(torch.zeros(1, 32, 32)),
        "orientation_shape": lambda: F.PatchDominantGradientOrientation(19)(torch.zeros(2, 1, 32, 32)),
        "orientation_channels": lambda: F.PatchDominantGradientOrientation(19)(torch.zeros(2, 3, 19, 19)),
    }
    for name in G.names("error"):
        _, kw, _, _ = G.case(name)
        with pytest.raises(Exception) as e:
            calls[kw["case"]]()
        if kw["error"] in ("ValueError", "TypeError"):
            assert type(e.value).__name__ == kw["error"] and str(e.value) == kw["message"], (name, str(e.value))
        else:  # KORNIA_CHECK_SHAPE's ShapeError: the message's first line
            assert type(e.value).__name__ == kw["error"], (name, type(e.value))
            assert str(e.value).splitlines()[0] == kw["message"].splitlines()[0], (name, str(e.value))


_SIFT_MODULES = {
    "__init__": helpers._STANDIN_KORNIA["__init__"] + ", feature",
    "feature/__init__": ("from .siftdesc import SIFTDescriptor, sift_describe\nfrom .orientation import PatchDominantGradientOrientation, "
                         "LAFOrienter\nfrom . import integrated"),
    "feature/siftdesc": "class SIFTDescriptor: pass\ndef sift_describe(): pass",
    "feature/orientation": ("class PatchDominantGradientOrientation: pass\n"
                            "class LAFOrienter:\n    def __init__(self, patch_size=32):\n"
                            "        self.angle_detector = PatchDominantGradientOrientation()\n"),
    "feature/integrated": ("from .orientation import LAFOrienter, PatchDominantGradientOrientation\nfrom .siftdesc import SIFTDescriptor\n"
                           "class SIFTFeature:\n    def __init__(self):\n        self.descriptor = SIFTDescriptor()\n"
                           "        self.orienter = LAFOrienter(19)\n"),
}


def test_install_rebinds_sift_and_orientation(tmp_path, monkeypatch):
    monkeypatch.setattr(helpers, "_STANDIN_KORNIA", {**helpers._STANDIN_KORNIA, **_SIFT_MODULES})
    with helpers.standin_kornia(tmp_path) as kornia:
        sd, ori, integ = (sys.modules[f"kornia.feature.{m}"] for m in ("siftdesc", "orientation", "integrated"))
        before = integ.SIFTFeature()
        orig = sd.SIFTDescriptor
        try:
            K.install(kornia)
            assert sd.SIFTDescriptor is F.SIFTDescriptor and sd.sift_describe is F.sift_describe
            assert ori.PatchDominantGradientOrientation is F.PatchDominantGradientOrientation
            assert kornia.feature.SIFTDescriptor is F.SIFTDescriptor and integ.SIFTDescriptor is F.SIFTDescriptor
            assert integ.PatchDominantGradientOrientation is F.PatchDominantGradientOrientation
            after = integ.SIFTFeature()
            assert isinstance(after.descriptor, F.SIFTDescriptor)
            assert isinstance(after.orienter.angle_detector, F.PatchDominantGradientOrientation)
            assert not isinstance(before.descriptor, F.SIFTDescriptor)  # built before install(): keeps what it holds
        finally:
            K.uninstall()
        assert sd.SIFTDescriptor is orig


def test_a_module_built_under_inference_mode_gives_its_gk_to_the_kernel():
    # gk is then an inference tensor, which has no version counter: the device copy is keyed on its values
    with torch.inference_mode():
        m = F.SIFTDescriptor(19, 5, 3)
        assert m.gk.is_inference()
        a = m._gk_on(torch.device("meta"))
        assert m._gk_on(torch.device("meta")) is a  # unchanged values: the cached copy
        m.gk.mul_(0.5)
        b = m._gk_on(torch.device("meta"))
        assert b is not a and b.shape == m.gk.shape
    m = F.SIFTDescriptor(19, 5, 3)
    assert m._gk_on(torch.device("cpu")) is not None and m._gk_on(torch.device("meta")) is m._gk_on(torch.device("meta"))


def test_the_operators_reject_what_the_kernels_cannot_read():
    # checked by the fake kernels too (meta tensors here), so a wrong-sized weight never reaches a kernel
    ops = torch.ops.kornia_b200
    m = lambda *shape: torch.empty(*shape, device="meta")  # noqa: E731
    assert ops.sift_describe_fwd(m(3, 1, 41, 41), m(1, 41, 41), m(1, 1, 16, 16), 8, 4, 10, 4, True, 0.2, 1e-10).shape == (3, 128)
    assert ops.patch_orientation_fwd(m(3, 1, 19, 19), m(1, 19, 19), m(1, 1, 5), 36, 1e-8).shape == (3,)
    bad_sift = [(m(3, 1, 41, 41), m(1, 40, 41), m(1, 1, 16, 16)), (m(3, 1, 41, 41), m(1, 41, 41), m(1, 1, 16, 15)),
                (m(3, 2, 41, 41), m(1, 41, 41), m(1, 1, 16, 16)), (m(3, 1, 41, 40), m(1, 41, 41), m(1, 1, 16, 16)),
                (m(3, 1, 41, 41), m(1, 41, 41).double(), m(1, 1, 16, 16))]
    for x, gk, pk in bad_sift:
        with pytest.raises(RuntimeError):
            ops.sift_describe_fwd(x, gk, pk, 8, 4, 10, 4, True, 0.2, 1e-10)
    for x, w, sm in [(m(3, 1, 19, 19), m(1, 19, 18), m(1, 1, 5)), (m(3, 1, 19, 19), m(1, 19, 19), m(1, 1, 4))]:
        with pytest.raises(RuntimeError):
            ops.patch_orientation_fwd(x, w, sm, 36, 1e-8)
