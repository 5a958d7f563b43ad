"""Feature responses on the H100: the fused kernels (corner_vwalk_kernel for Harris / GFTT, grad_tiled_kernel's Hessian
epilogue) against the composition of this library's spatial_gradient / gaussian_blur2d and torch ops, bit for bit, plus
launch counts, gradients, torch.compile, opcheck and install() on a reference-layout stand-in package."""
import ctypes
import importlib
import zlib

import pytest
import torch

import helpers

pytestmark = pytest.mark.gpu

K = importlib.import_module("kornia_b200")
R = importlib.import_module("kornia_b200.feature.responses")
_ops = importlib.import_module("kornia_b200._ops")
_lib = importlib.import_module("kornia_b200._lib")
from kornia_b200.filters.gaussian import _constant_taps  # noqa: E402
from kornia_b200.filters.sobel import _host_taps  # noqa: E402

from conftest import golden  # noqa: E402

KINDS = {"harris": _ops.HARRIS, "gftt": _ops.GFTT, "hessian": _ops.HESSIAN}


def _bits_equal(a, b):
    assert a.shape == b.shape and a.dtype == b.dtype
    same = (a.view(torch.int32) == b.view(torch.int32)) | (a.isnan() & b.isnan())
    return bool(same.all())


def _composed(kind, x, mode, sigmas, k):
    if kind == "harris":
        return R._composed_harris(x, k, mode, sigmas)
    if kind == "gftt":
        return R._composed_gftt(x, mode, sigmas)
    return R._composed_hessian(x, mode, sigmas)


def _public(kind, x, mode, sigmas, k):
    if kind == "harris":
        return K.feature.harris_response(x, k, mode, sigmas)
    if kind == "gftt":
        return K.feature.gftt_response(x, mode, sigmas)
    return K.feature.hessian_response(x, mode, sigmas)


def _fused_into_nan(kind, x, mode, sigmas, k):
    """The C entry point writing into an output prefilled with NaN: every element must be written."""
    B, C, H, W = x.shape
    taps, _, sk = _host_taps(mode, 2 if kind == "hessian" else 1, True, x.dtype)
    blur = None if kind == "hessian" else _constant_taps((7, 7), (1.0, 1.0), True, x.device, x.dtype)[0]
    kt = k if isinstance(k, torch.Tensor) else None
    s4 = None if sigmas is None else sigmas.pow(4)
    out = torch.full_like(x, float("nan"))
    host = (ctypes.c_double * len(taps))(*taps)
    _lib.call("kb200_feature_response_forward", x.data_ptr(), host, None if blur is None else blur.data_ptr(), 0.0 if kt is not None else float(k),
              None if kt is None else kt.data_ptr(), None if s4 is None else s4.data_ptr(), out.data_ptr(), B * C, C, H, W, sk,
              0 if blur is None else 7, KINDS[kind], _lib.F32, torch.cuda.current_stream().cuda_stream)
    return out


def _image(B, C, H, W, special=False, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.rand(B, C, H, W, device="cuda", generator=g)
    if special:
        flat = x.view(-1)
        n = flat.numel()
        idx = torch.randint(0, n, (max(8, n // 500),), device="cuda", generator=g)
        vals = torch.tensor([float("nan"), float("inf"), -float("inf"), -0.0, 1e-40, -1e-41, 1e-38, 3e38], device="cuda")
        flat[idx] = vals[torch.arange(idx.numel(), device="cuda") % vals.numel()]
        flat[:3] = torch.tensor([1e-40, -0.0, 1e-39], device="cuda")
        flat[-2:] = torch.tensor([float("inf"), -0.0], device="cuda")
    return x


SHAPES = [(2, 1, 4, 4), (37, 3, 200, 520), (1, 1, 1080, 1920), (1, 3, 1080, 1920), (3, 2, 61, 68)]


@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("mode", ["sobel", "diff"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("special", [False, True], ids=["finite", "special"])
def test_fused_equals_composition_bitwise(kind, mode, shape, special):
    x = _image(*shape, special=special, seed=zlib.crc32(repr((kind, mode, shape, special)).encode()))
    B = shape[0]
    sig_opts = [None, torch.rand(B, device="cuda") * 2 + 0.5]
    k_opts = [0.04, torch.tensor(0.05, device="cuda"), torch.tensor(0.06, device="cuda", dtype=torch.float64)] if kind == "harris" else [0.0]
    with torch.no_grad():
        for sigmas in sig_opts:
            for k in k_opts:
                want = _composed(kind, x, mode, sigmas, k)
                assert want.dtype == torch.float32
                got = _fused_into_nan(kind, x, mode, sigmas, k if not isinstance(k, torch.Tensor) else k.float())
                assert _bits_equal(got, want), (kind, mode, shape, sigmas is not None, k)
                assert _bits_equal(_public(kind, x, mode, sigmas, k), want)


_G = golden("responses")


@pytest.mark.parametrize("name", _G.names())
def test_goldens_within_the_response_scale(name):
    """The public functions (fused inside the envelope, composed outside it) on the GPU against the reference's CPU goldens:
    within 1e-5 of the case's largest response (cuDNN / CPU convolutions and the blur sum in different orders)."""
    op, kw, ins, outs = _G.case(name)
    x = ins["input"].cuda()
    sig = ins["sigmas"].cuda() if "sigmas" in ins else None
    k = ins["k"].cuda() if "k" in ins else kw.get("k")
    with torch.no_grad():
        got = _public(op[: -len("_response")], x, kw["grads_mode"], sig, k).cpu()
    want = outs["out"]
    scale = want.abs().max().item()
    torch.testing.assert_close(got, want, rtol=0, atol=1e-5 * scale + 1e-12)
    xg = x.clone().requires_grad_(True)
    out = _public(op[: -len("_response")], xg, kw["grads_mode"], sig, k)
    (g,) = torch.autograd.grad((out * ins["cot"].cuda()).sum(), [xg])
    torch.testing.assert_close(g.cpu(), outs["grad_input"], rtol=0, atol=1e-5 * outs["grad_input"].abs().max().item() + 1e-12)


def _tags(fn):
    """Names of the library's forward kernels ``fn`` launches, in order."""
    _ops.kernel_events = []
    try:
        out = fn()
        return out, [tag for tag, _, _ in _ops.kernel_events]
    finally:
        _ops.kernel_events = None


@pytest.mark.parametrize("kind", list(KINDS))
def test_one_launch_inside_the_envelope_and_composition_outside(kind):
    x = _image(2, 3, 64, 96)
    sig = torch.rand(2, device="cuda") + 0.5
    with torch.no_grad():
        _public(kind, x, "sobel", sig, 0.04)
        _, tags = _tags(lambda: _public(kind, x, "sobel", sig, 0.04))
        assert tags == ["feature_response_forward"]
        for y, s in ((_image(2, 3, 64, 98), sig), (x.double(), sig.double()), (x, sig.double())):
            out, tags = _tags(lambda: _public(kind, y, "sobel", s, 0.04))
            assert "feature_response_forward" not in tags and tags[0] == "spatial_gradient_forward"
            assert _bits_equal(out.float(), _composed(kind, y, "sobel", s, 0.04).float())
    x.requires_grad_(True)
    _, tags = _tags(lambda: _public(kind, x, "sobel", None, 0.04))
    assert "feature_response_forward" not in tags


def test_harris_k_forms_and_cpu_scalar():
    x = _image(2, 1, 40, 64)
    with torch.no_grad():
        want = R._composed_harris(x, torch.tensor(0.05), "sobel", None)
        assert _bits_equal(K.feature.harris_response(x, torch.tensor(0.05), "sobel"), want)
        want = R._composed_harris(x, 3, "diff", None)
        assert _bits_equal(K.feature.harris_response(x, 3, "diff"), want)
        kk = torch.tensor([0.04], device="cuda")  # a sized k takes part in type promotion: composition
        out, tags = _tags(lambda: K.feature.harris_response(x, kk))
        assert "feature_response_forward" not in tags
        assert _bits_equal(out, R._composed_harris(x, kk, "sobel", None))


@pytest.mark.parametrize("device", ["cuda", "cpu"])
def test_a_k_that_requires_grad_takes_the_differentiable_path(device):
    x = _image(2, 1, 40, 64)
    k = torch.tensor(0.04, device=device, requires_grad=True)
    out, tags = _tags(lambda: K.feature.harris_response(x, k))
    assert "feature_response_forward" not in tags and out.grad_fn is not None
    out.sum().backward()
    kr = k.detach().clone().requires_grad_(True)
    R._composed_harris(x, kr, "sobel", None).sum().backward()
    assert k.grad is not None and torch.equal(k.grad, kr.grad)


def test_gftt_sigmas_that_is_not_a_tensor_fails_like_the_reference():
    with pytest.raises(AttributeError, match="'list' object has no attribute 'pow'"):
        K.feature.gftt_response(_image(2, 1, 16, 16), sigmas=[1.0, 2.0])


@pytest.mark.parametrize("kind", list(KINDS))
def test_gradcheck_of_the_composition(kind):
    x = torch.rand(1, 2, 9, 8, device="cuda", dtype=torch.float64, requires_grad=True)
    sig = torch.rand(1, device="cuda", dtype=torch.float64) + 0.5
    assert torch.autograd.gradcheck(lambda t: _public(kind, t, "sobel", sig, 0.04), (x,), eps=1e-6, atol=1e-5)


@pytest.mark.parametrize("module", ["BlobHessian", "CornerGFTT"])
def test_torch_compile_fullgraph_matches_eager(module):
    m = getattr(K.feature, module)()
    x = _image(2, 3, 48, 64)
    sig = torch.rand(2, device="cuda") + 0.5
    torch._dynamo.reset()
    compiled = torch.compile(m, fullgraph=True)
    with torch.no_grad():
        assert _bits_equal(compiled(x), m(x))
        # the compiled graph computes sigmas.pow(4) with inductor's own rounding: a few ulp, nothing in the kernel
        torch.testing.assert_close(compiled(x, sig), m(x, sig), rtol=1e-6, atol=0)


def test_opcheck():
    x = _image(2, 3, 16, 32)
    taps, _, sk = _host_taps("sobel", 1, True, x.dtype)
    blur = _constant_taps((7, 7), (1.0, 1.0), True, x.device, x.dtype)[0]
    s4 = torch.rand(2, device="cuda")
    torch.library.opcheck(torch.ops.kornia_b200.feature_response_fwd, (x, list(taps), sk, blur, 0.04, None, s4, _ops.HARRIS))
    taps2, _, sk2 = _host_taps("sobel", 2, True, x.dtype)
    torch.library.opcheck(torch.ops.kornia_b200.feature_response_fwd, (x, list(taps2), sk2, None, 0.0, None, None, _ops.HESSIAN))


_FEATURE_MODULES = {
    "__init__": helpers._STANDIN_KORNIA["__init__"] + ", feature",
    "feature/__init__": "from .responses import CornerGFTT, gftt_response, harris_response, hessian_response",
    # the reference's module layout: CornerGFTT.forward calls the module-global gftt_response (responses.py:413-438)
    "feature/responses": "import torch\n"
                         "def harris_response(): pass\n"
                         "def gftt_response(): pass\n"
                         "def hessian_response(): pass\n"
                         "class CornerGFTT(torch.nn.Module):\n"
                         "    def __init__(self, grads_mode='sobel'):\n"
                         "        super().__init__()\n"
                         "        self.grads_mode = grads_mode\n"
                         "    def forward(self, input, sigmas=None):\n"
                         "        return gftt_response(input, self.grads_mode, sigmas)\n",
}


def test_install_runs_the_reference_modules_on_the_fused_kernel(tmp_path, monkeypatch):
    monkeypatch.setattr(helpers, "_STANDIN_KORNIA", {**helpers._STANDIN_KORNIA, **_FEATURE_MODULES})
    with helpers.standin_kornia(tmp_path) as kornia:
        try:
            K.install(kornia)
            x = _image(2, 3, 64, 128)
            with torch.no_grad():
                n0 = _ops.launch_count
                got = kornia.feature.responses.CornerGFTT()(x)
                assert _ops.launch_count - n0 == 1
                assert _bits_equal(got, R._composed_gftt(x, "sobel", None))
        finally:
            K.uninstall()
