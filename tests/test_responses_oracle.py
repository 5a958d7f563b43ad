"""Feature responses on the host (no GPU): public signatures and reprs, the reference's error types and messages, and
install() on stand-in packages with and without ``feature/responses.py``."""
import importlib
import inspect

import pytest
import torch

import helpers
import responses_restated as RR
from conftest import golden

K = importlib.import_module("kornia_b200")
F = importlib.import_module("kornia_b200.feature")
G = golden("responses")


def _call(fn, op, kw, ins, x):
    sig = ins.get("sigmas")
    if op == "harris_response":
        return fn["harris"](x, ins["k"] if "k" in ins else kw["k"], kw["grads_mode"], sig)
    return fn[op[: -len("_response")]](x, kw["grads_mode"], sig)


@pytest.mark.parametrize("name", G.names())
def test_oracle_reproduces_the_goldens_and_their_gradients(name):
    op, kw, ins, outs = G.case(name)
    x = ins["input"].clone().requires_grad_(True)
    out = _call({"harris": RR.harris_response, "gftt": RR.gftt_response, "hessian": RR.hessian_response}, op, kw, ins, x)
    torch.testing.assert_close(out.detach(), outs["out"], rtol=1e-5, atol=1e-7)
    (g,) = torch.autograd.grad((out * ins["cot"]).sum(), [x])
    torch.testing.assert_close(g, outs["grad_input"], rtol=1e-5, atol=1e-6)


def _sig(fn):
    params = inspect.signature(fn).parameters.values()
    return "(" + ", ".join(p.name if p.default is inspect._empty else f"{p.name}={p.default!r}" for p in params) + ")"


def test_signatures_and_reprs_match_reference():
    # kornia/feature/responses.py:39-44,129-131,206-208,388,421,449
    want = {
        F.harris_response: "(input, k=0.04, grads_mode='sobel', sigmas=None)",
        F.gftt_response: "(input, grads_mode='sobel', sigmas=None)",
        F.hessian_response: "(input, grads_mode='sobel', sigmas=None)",
        F.CornerHarris.__init__: "(self, k, grads_mode='sobel')",
        F.CornerGFTT.__init__: "(self, grads_mode='sobel')",
        F.BlobHessian.__init__: "(self, grads_mode='sobel')",
    }
    for fn, sig in want.items():
        assert _sig(fn) == sig, fn.__qualname__
    harris = F.CornerHarris(0.04)
    assert "k" in dict(harris.named_buffers()) and harris.k.dtype == torch.float32 and harris.k.dim() == 0
    assert repr(harris) == "CornerHarris(k=0.03999999910593033, grads_mode=sobel)"
    k = torch.tensor([0.05])
    assert F.CornerHarris(k, "diff").k is k
    assert repr(F.CornerGFTT("diff")) == "CornerGFTT(grads_mode=diff)"
    assert repr(F.BlobHessian()) == "BlobHessian(grads_mode=sobel)"
    assert K.feature is F and "feature" in K.__all__


def test_errors_match_the_reference():
    # validation runs before anything touches a device
    x = torch.zeros(2, 1, 8, 8)
    for fn in (F.harris_response, F.gftt_response, F.hessian_response):
        with pytest.raises(Exception, match="Shape dimension mismatch"):
            fn(torch.zeros(1, 8, 8))
    with pytest.raises(TypeError, match="sigmas type is not a torch.Tensor. Got <class 'list'>"):
        F.harris_response(x, sigmas=[1.0, 2.0])
    with pytest.raises(ValueError, match=r"Invalid sigmas shape, we expect B == input.size\(0\). Got: torch.Size\(\[3\]\)"):
        F.harris_response(x, sigmas=torch.ones(3))
    with pytest.raises(TypeError, match="sigmas type is not a torch.Tensor"):
        F.hessian_response(x, sigmas=1.0)
    with pytest.raises(ValueError, match="Invalid sigmas shape"):
        F.hessian_response(x, sigmas=torch.ones(2, 1))
    # gftt_response validates no sigmas (reference behaviour): the call gets past validation and reaches the CUDA-only engine
    with pytest.raises(RuntimeError, match="CUDA-only"):
        F.gftt_response(x, sigmas=[1.0, 2.0])


_FEATURE_MODULES = {
    "__init__": helpers._STANDIN_KORNIA["__init__"] + ", feature",
    "feature/__init__": "from .responses import gftt_response, harris_response, hessian_response\nfrom . import integrated",
    "feature/responses": "def harris_response(): pass\ndef gftt_response(): pass\ndef hessian_response(): pass",
    "feature/integrated": "from .responses import gftt_response",
}


def test_install_rebinds_the_responses(tmp_path, monkeypatch):
    monkeypatch.setattr(helpers, "_STANDIN_KORNIA", {**helpers._STANDIN_KORNIA, **_FEATURE_MODULES})
    with helpers.standin_kornia(tmp_path) as kornia:
        import sys

        resp = sys.modules["kornia.feature.responses"]
        orig = resp.gftt_response
        try:
            K.install(kornia)
            for name in ("harris_response", "gftt_response", "hessian_response"):
                assert getattr(resp, name) is getattr(F, name)
                assert getattr(kornia.feature, name) is getattr(F, name)
            assert sys.modules["kornia.feature.integrated"].gftt_response is F.gftt_response
        finally:
            K.uninstall()
        assert resp.gftt_response is orig


def test_install_skips_a_package_without_responses(tmp_path):
    with helpers.standin_kornia(tmp_path) as kornia:
        try:
            K.install(kornia)
            assert kornia.filters.filter2d is K.filters.filter2d
            assert not hasattr(kornia, "feature")
        finally:
            K.uninstall()
