"""Motion blur on the GPU: the zero-skipping filter2d kernel (odd K 9..31) against the generic kernel bit for bit, motion_blur
against the goldens and the same-device reference composition, gradients, RandomMotionBlur, torch.compile and install()."""
import importlib
import math

import pytest
import torch

import helpers
import motion_restated as MR
from conftest import golden
from kornia_b200 import _lib, config
from kornia_b200._ops import _dtype_code, _ptr, _stream

K = importlib.import_module("kornia_b200")
A = importlib.import_module("kornia_b200.augmentation")
KF = K.filters
pytestmark = pytest.mark.gpu
DEV = "cuda"
FP32 = dict(rtol=1e-4, atol=1e-5)
G = golden("motion")
BORDERS = ("constant", "reflect", "replicate")


def _bits(t):
    return t.contiguous().view(torch.int32)


def _assert_bits(got, want):
    same = _bits(got) == _bits(want)
    assert bool(same.all()), f"{(~same).sum().item()} / {same.numel()} outputs differ in their bits"


def _kernels(kind, n, K_, gen):
    if kind == "dense":
        return (torch.rand(n, K_, K_, generator=gen) - 0.5).to(DEV)
    angle = (torch.rand(n, generator=gen) * 360.0 - 180.0).to(DEV)
    direction = (torch.rand(n, generator=gen) * 2.0 - 1.0).to(DEV)
    return KF.get_motion_kernel2d(K_, angle, direction, kind)


def _both(x, k, border):
    """(new kernel, generic kernel) outputs of filter2d."""
    new = KF.filter2d(x, k, border)
    with config.override(tiled_filter=0):
        ref = KF.filter2d(x, k, border)
    return new, ref


@pytest.mark.parametrize("K_", (9, 11, 15, 21, 31))
@pytest.mark.parametrize("border", BORDERS)
@pytest.mark.parametrize("bk", ("one", "per_sample", "cycling"))
@pytest.mark.parametrize("kind", ("nearest", "bilinear", "dense"))
def test_taps_kernel_is_bit_identical_to_the_generic_kernel(K_, border, bk, kind):
    gen = torch.Generator().manual_seed(K_ * 100 + len(border) * 10 + len(bk) + len(kind))
    B = 6
    x = torch.rand(B, 3, 70, 132, generator=gen).to(DEV)
    k = _kernels(kind, {"one": 1, "per_sample": B, "cycling": 3}[bk], K_, gen)
    new, ref = _both(x, k, border)
    _assert_bits(new, ref)


@pytest.mark.parametrize("shape,K_,kind", [((37, 3, 200, 520), 15, "nearest"), ((2, 3, 1080, 1920), 31, "bilinear"),
                                           ((3, 1, 33, 36), 9, "dense"), ((1, 2, 17, 20), 31, "nearest")])
@pytest.mark.parametrize("border", BORDERS)
def test_taps_kernel_partial_tiles_many_strips_and_1080p(shape, K_, kind, border):
    gen = torch.Generator().manual_seed(shape[0] + K_)
    x = torch.rand(*shape, generator=gen).to(DEV)
    k = _kernels(kind, shape[0], K_, gen)
    new, ref = _both(x, k, border)
    _assert_bits(new, ref)


@pytest.mark.parametrize("K_", (9, 15, 31))
@pytest.mark.parametrize("border", BORDERS)
def test_taps_kernel_with_special_values(K_, border):
    """NaN, +-Inf, -0 and subnormal texels in some tiles, tiny texels whose products with the taps underflow, subnormal
    taps: the tiles they touch take the dense loop and every output keeps the generic kernel's bits."""
    gen = torch.Generator().manual_seed(K_)
    B, C, H, W = 4, 2, 100, 300
    x = torch.rand(B, C, H, W, generator=gen) * 2 - 1
    flat = x.view(-1)
    specials = torch.tensor([float("nan"), float("inf"), float("-inf"), -0.0, 1e-40, -3e-39])
    idx = torch.randint(0, flat.numel(), (24,), generator=gen)
    flat[idx] = specials.repeat(4)
    x[2] *= 1e-30  # sample 2: products with sample 2's subnormal taps underflow
    x[3, :, :40] = -0.0
    k = _kernels("nearest", B, K_, gen)
    k[2] *= 1e-38  # subnormal taps
    new, ref = _both(x.to(DEV), k, border)
    _assert_bits(new, ref)


def test_taps_kernel_writes_every_output():
    gen = torch.Generator().manual_seed(5)
    B, C, H, W, K_ = 3, 2, 77, 204, 21
    x = torch.rand(B, C, H, W, generator=gen).to(DEV)
    k = _kernels("bilinear", B, K_, gen).contiguous()
    out = torch.full_like(x, float("nan"))
    _lib.call("kb200_filter2d_forward", _ptr(x), _ptr(k), _ptr(out), B, C, H, W, B, K_, K_, _lib.BORDERS["reflect"], 1, _dtype_code(x), _stream(x))
    with config.override(tiled_filter=0):
        ref = KF.filter2d(x, k, "reflect")
    _assert_bits(out, ref)


# ------------------------------------------------------------------------------------------ motion_blur
def _args(kw, ins, dev):
    angle = ins["angle"].to(dev) if "angle" in ins else kw["angle"]
    direction = ins["direction"].to(dev) if "direction" in ins else kw["direction"]
    return angle, direction


@pytest.mark.parametrize("name", G.names("get_motion_kernel2d"))
def test_kernel_matches_golden_and_same_device_reference(name):
    _, kw, ins, outs = G.case(name)
    angle, direction = _args(kw, ins, DEV)
    got = KF.get_motion_kernel2d(kw["kernel_size"], angle, direction, kw["mode"])
    assert got.device.type == "cuda" and got.dtype == outs["kernel"].dtype
    torch.testing.assert_close(got.cpu(), outs["kernel"], rtol=1e-4, atol=1e-4)
    want = MR.get_motion_kernel2d(kw["kernel_size"], angle, direction, kw["mode"], device=torch.device(DEV))
    if kw["mode"] == "nearest":  # the rotation copies taps: same device, same taps
        assert torch.equal(got, want), (got - want).abs().max()
    else:  # warp_affine's bilinear weights are not grid_sample's op sequence: they agree to a few ulp (measured <= 1.5e-8)
        torch.testing.assert_close(got, want, rtol=1e-6, atol=5e-8)


@pytest.mark.parametrize("name", G.names("motion_blur"))
def test_motion_blur_matches_golden_and_same_device_reference(name):
    _, kw, ins, outs = G.case(name)
    x = ins["input"].to(DEV)
    angle, direction = _args(kw, ins, DEV)
    got = KF.motion_blur(x, kw["kernel_size"], angle, direction, kw["border_type"], kw["mode"])
    torch.testing.assert_close(got.cpu(), outs["out"], rtol=1e-4, atol=1e-4)
    want = MR.motion_blur(x, kw["kernel_size"], angle, direction, kw["border_type"], kw["mode"], device=torch.device(DEV))
    torch.testing.assert_close(got, want, **FP32)
    mod = KF.MotionBlur(kw["kernel_size"], 30.0, -0.3, kw["border_type"])
    assert torch.equal(mod(x), KF.motion_blur(x, kw["kernel_size"], 30.0, -0.3, kw["border_type"]))


@pytest.mark.parametrize("name", [n for n in G.names("motion_blur") if "number" not in n])
def test_motion_blur_gradients_match_golden(name):
    _, kw, ins, outs = G.case(name)
    leaves = [ins[k].to(DEV).requires_grad_(True) for k in ("input", "angle", "direction")]
    out = KF.motion_blur(leaves[0], kw["kernel_size"], leaves[1], leaves[2], kw["border_type"], kw["mode"])
    grads = torch.autograd.grad((out * outs["cot"].to(DEV)).sum(), leaves, allow_unused=True)
    for g, key in zip(grads, ("grad_input", "grad_angle", "grad_direction")):
        g = torch.zeros_like(leaves[0] if key == "grad_input" else leaves[1]) if g is None else g
        # d/dangle and d/ddirection are each one fp32 sum over the whole batch: summed in another order than the reference's
        # CPU reduction, they agree to ~1e-4 (measured 1.1e-4 at worst); the per-pixel input gradient to 1e-4
        tol = 1e-4 if key == "grad_input" else 1e-3
        assert helpers.rel_l2(g.cpu(), outs[key]) < tol or outs[key].abs().max() == 0, key


@pytest.mark.parametrize("mode", ("nearest", "bilinear"))
def test_motion_blur_gradcheck_fp64(mode):
    gen = torch.Generator().manual_seed(3)
    x = torch.rand(2, 2, 9, 12, generator=gen, dtype=torch.float64).to(DEV).requires_grad_(True)
    angle = torch.tensor([20.0, -65.0], dtype=torch.float64, device=DEV)
    direction = torch.tensor([0.3, -0.6], dtype=torch.float64, device=DEV)
    assert torch.autograd.gradcheck(lambda t: KF.motion_blur(t, 5, angle, direction, "reflect", mode), (x,))
    if mode == "bilinear":
        a, d = angle.clone().requires_grad_(True), direction.clone().requires_grad_(True)
        # the matrix gradient of warp_affine accumulates with atomics: repeated backward passes differ in the last bits
        assert torch.autograd.gradcheck(lambda aa, dd: KF.motion_blur(x.detach(), 5, aa, dd, "constant", mode), (a, d), nondet_tol=1e-9)


@pytest.mark.parametrize("dtype", (torch.float16, torch.bfloat16, torch.float64))
def test_motion_blur_other_dtypes(dtype):
    gen = torch.Generator().manual_seed(4)
    x = torch.rand(2, 3, 40, 64, generator=gen).to(DEV)
    angle = torch.tensor([10.0, 100.0], device=DEV)
    direction = torch.tensor([0.2, -0.4], device=DEV)
    got = KF.motion_blur(x.to(dtype), 9, angle, direction, "reflect")
    assert got.dtype == dtype
    want = KF.motion_blur(x, 9, angle, direction, "reflect")
    tol = 1e-5 if dtype == torch.float64 else 2e-2
    torch.testing.assert_close(got.float(), want, rtol=tol, atol=max(tol, 1e-6))


def test_motion_blur_builds_its_kernel_on_the_image_device():
    x = torch.rand(1, 3, 32, 40, device=DEV)
    k = KF.get_motion_kernel2d(9, 35.0, 0.5)
    assert k.device.type == "cuda"
    assert torch.equal(KF.motion_blur(x, 9, 35.0, 0.5), KF.filter2d(x, k, "constant"))
    cpu_angle = torch.tensor([35.0])
    assert torch.equal(KF.motion_blur(x, 9, cpu_angle, torch.tensor([0.5])), KF.filter2d(x, k, "constant"))


def test_motion_blur_compiles_to_one_graph():
    graphs = []

    def backend(gm, example_inputs):
        graphs.append(gm)
        return gm.forward

    fn = torch.compile(lambda x, a, d: KF.motion_blur(x, 11, a, d, "reflect", "bilinear"), backend=backend, fullgraph=True)
    x = torch.rand(2, 3, 48, 64, device=DEV)
    a = torch.tensor([15.0, -40.0], device=DEV)
    d = torch.tensor([0.1, 0.8], device=DEV)
    got = fn(x, a, d)
    assert len(graphs) == 1
    assert torch.equal(got, KF.motion_blur(x, 11, a, d, "reflect", "bilinear"))


# ------------------------------------------------------------------------------------------ RandomMotionBlur
def test_random_motion_blur_docstring_answer():
    torch.manual_seed(0)
    out = A.RandomMotionBlur(3, 35.0, 0.5, p=1.0)(torch.ones(1, 1, 5, 5, device=DEV))
    row = torch.tensor([0.5773, 1.0000, 1.0000, 1.0000, 0.7561], device=DEV)
    torch.testing.assert_close(out, row.expand(1, 1, 5, 5), rtol=0, atol=1e-4)


@pytest.mark.parametrize("ksize", (9, (3, 15)))
def test_random_motion_blur_is_motion_blur_with_the_drawn_parameters(ksize):
    torch.manual_seed(11)
    x = torch.rand(5, 3, 60, 80, device=DEV)
    aug = A.RandomMotionBlur(ksize, (-50.0, 80.0), 0.7, border_type="reflect", resample="BILINEAR", p=1.0)
    out = aug(x)
    p = aug._params
    k = ksize if isinstance(ksize, int) else int(p["ksize_factor"][int(p["idx"][0])])
    assert torch.equal(out, KF.motion_blur(x, k, p["angle_factor"], p["direction_factor"], "reflect", "bilinear"))
    assert torch.equal(aug(x, params=p), out)


def test_random_motion_blur_applies_with_probability_p():
    torch.manual_seed(12)
    x = torch.rand(16, 3, 32, 48, device=DEV)
    aug = A.RandomMotionBlur(11, 90.0, 1.0, p=0.5)
    out = aug(x)
    p = aug._params
    on = (p["batch_prob"] > 0.5).to(DEV)
    assert 0 < int(on.sum()) < 16
    assert torch.equal(out[~on], x[~on])
    want = KF.motion_blur(x, 11, p["angle_factor"], p["direction_factor"])
    assert torch.equal(out[on], want[on])


# ------------------------------------------------------------------------------------------ install()
_STANDIN_MOTION = {
    "filters/kernels_geometry": "def get_motion_kernel2d(kernel_size, angle, direction=0.0, mode='nearest'):\n"
                                "    raise RuntimeError('the stand-in builds its kernel on the CPU')",
    "filters/motion": "from .filter import filter2d\nfrom .kernels_geometry import get_motion_kernel2d\n"
                      "def motion_blur(input, kernel_size, angle, direction, border_type='constant', mode='nearest'):\n"
                      "    return filter2d(input, get_motion_kernel2d(kernel_size, angle, direction, mode), border_type)\n"
                      "class MotionBlur:\n"
                      "    def __init__(self, kernel_size, angle, direction, border_type='constant'):\n"
                      "        self.args = (kernel_size, angle, direction, border_type)\n"
                      "    def __call__(self, x):\n"
                      "        return motion_blur(x, *self.args)",
    "filters/__init__": helpers._STANDIN_KORNIA["filters/__init__"] + "\nfrom .kernels_geometry import get_motion_kernel2d\n"
                                                                      "from .motion import motion_blur, MotionBlur",
}


def test_install_runs_the_references_motion_blur_on_a_cuda_image(tmp_path, monkeypatch):
    monkeypatch.setattr(helpers, "_STANDIN_KORNIA", {**helpers._STANDIN_KORNIA, **_STANDIN_MOTION})
    x = torch.rand(2, 3, 40, 60, device=DEV)
    with helpers.standin_kornia(tmp_path) as kornia:
        try:
            K.install(kornia)
            got = kornia.filters.MotionBlur(9, 35.0, 0.5)(x)
            k = kornia.filters.get_motion_kernel2d(5, 35.0, 0.5)
        finally:
            K.uninstall()
    assert torch.equal(got, KF.motion_blur(x, 9, 35.0, 0.5))
    assert k.device.type == "cuda" and math.isclose(float(k.sum()), 1.0, rel_tol=1e-6)
