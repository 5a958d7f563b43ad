"""ScalePyramid on the H100: the octave kernel (csrc/octave_vwalk.cuh) against the composition of this library's
filter2d_separable / gaussian_blur2d and torch.stack, bit for bit (-0 and +0 differ, NaN equals NaN), for every
instantiated chain in both stage-0 modes; the public module against the composition and the reference's goldens; which
kernels run inside and outside the kernel's envelope; gradcheck, torch.compile, opcheck and a reference-layout
state_dict."""
import ctypes
import importlib

import pytest
import torch

import scale_pyramid_restated as SR
from conftest import golden

pytestmark = pytest.mark.gpu

K = importlib.import_module("kornia_b200")
P = importlib.import_module("kornia_b200.geometry.transform.pyramid")
_ops = importlib.import_module("kornia_b200._ops")
_lib = importlib.import_module("kornia_b200._lib")

# the module whose chain each instantiation serves: ScalePyramid(), ScaleSpaceDetector's, the double_image one
MODULES = {"default": {}, "detector": {"min_size": 16, "extra_levels": 2}, "double": {"min_size": 32, "double_image": True}}


def _bits_equal(a, b):
    assert a.shape == b.shape and a.dtype == b.dtype
    return bool(((a.view(torch.int32) == b.view(torch.int32)) | (a.isnan() & b.isnan())).all())


def _image(B, C, H, W, specials=False, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.rand(B, C, H, W, device="cuda", generator=g) * 3 - 1
    if specials:
        flat = x.view(-1)
        vals = torch.tensor([float("nan"), float("inf"), float("-inf"), -0.0, 1e-40, -1e-41, 1e-38, 3e38], device="cuda")
        idx = torch.randint(0, flat.numel(), (max(8, flat.numel() // 500),), device="cuda", generator=g)
        flat[idx] = vals[torch.arange(idx.numel(), device="cuda") % 8]
        x[0, 0, : H // 4] = -0.0
    return x


def _octave_into_nan(sp, x, blur_first):
    """The C entry point writing into an output prefilled with NaN: every element must be written."""
    B, C, H, W = x.shape
    L = sp.n_levels + sp.extra_levels
    names = (["_gk_init"] if blur_first else []) + [f"_gk_{i}" for i in range(L - 1)]
    taps = [v for n in names for v in sp._host_taps[n]]
    ks = ([len(sp._host_taps["_gk_init"])] if blur_first else [0]) + [len(sp._host_taps[f"_gk_{i}"]) for i in range(L - 1)]
    out = torch.full((B, C, L, H, W), float("nan"), device="cuda")
    _lib.call("kb200_scale_octave_forward", x.data_ptr(), (ctypes.c_double * len(taps))(*taps), (ctypes.c_int * L)(*ks), L, out.data_ptr(),
              B * C, H, W, _lib.F32, torch.cuda.current_stream().cuda_stream)
    return out


def _composed(sp, x, blur_first):
    return torch.stack(sp._composed_octave(x, blur_first, 1.0 if sp.double_image else 0.5), 2)


@pytest.mark.parametrize("shape", [(1, 1, 1080, 1920), (2, 3, 720, 1280), (3, 1, 200, 520), (1, 1, 61, 68), "limit"])
@pytest.mark.parametrize("module", list(MODULES))
@pytest.mark.parametrize("blur_first", [True, False])
@pytest.mark.parametrize("specials", [False, True])
def test_octave_kernel_bit_identical_to_composition(shape, module, blur_first, specials):
    sp = P.ScalePyramid(**MODULES[module]).cuda()
    if shape == "limit":  # the smallest side equals the largest tap count
        kmax = max(len(v) for v in sp._host_taps.values() if v is not None)
        shape = (2, 1, kmax, (kmax + 3) // 4 * 4)
    x = _image(*shape, specials=specials)
    with torch.no_grad():
        got = _octave_into_nan(sp, x, blur_first)
        assert _bits_equal(got, _composed(sp, x, blur_first))


@pytest.mark.parametrize("module", list(MODULES))
@pytest.mark.parametrize("specials", [False, True])
def test_module_equals_composition_every_octave(module, specials):
    sp = P.ScalePyramid(**MODULES[module]).cuda()
    x = _image(2, 1, 240, 320, specials=specials, seed=3)
    with torch.no_grad():
        pyr, sig, pd = sp(x)
        cpyr, csig, cpd = sp._composed_pyramid(x)
    assert len(pyr) == len(cpyr) >= 3
    for a, b in zip(pyr, cpyr):
        assert _bits_equal(a, b)
    for a, b in zip(sig + pd, csig + cpd):
        assert torch.equal(a, b)


G = golden("scale_pyramid")


@pytest.mark.parametrize("name", G.names())
def test_module_matches_reference_goldens(name):
    _, kw, ins, outs = G.case(name)
    x = ins["input"].cuda().requires_grad_(True)
    pyr, sig, pd = P.ScalePyramid(**kw).cuda()(x)
    assert len(pyr) == len([k for k in outs if k.startswith("pyr")])
    for o, p in enumerate(pyr):
        want = outs[f"pyr{o}"].cuda()
        torch.testing.assert_close(p.detach(), want, rtol=0, atol=1e-5 * float(want.abs().max()))
        assert torch.equal(sig[o].cpu(), outs[f"sig{o}"]) and torch.equal(pd[o].cpu(), outs[f"pd{o}"])
    (g,) = torch.autograd.grad(sum((p * ins[f"cot{o}"].cuda()).sum() for o, p in enumerate(pyr)), [x])
    torch.testing.assert_close(g.cpu(), outs["grad_input"], rtol=0, atol=1e-5 * float(outs["grad_input"].abs().max()))
    with torch.no_grad():  # the same case without a gradient: fused where the kernel's envelope allows
        for o, p in enumerate(P.ScalePyramid(**kw).cuda()(x.detach())[0]):
            want = outs[f"pyr{o}"].cuda()
            torch.testing.assert_close(p, want, rtol=0, atol=1e-5 * float(want.abs().max()))


def _tags(fn):
    _ops.kernel_events = []
    try:
        out = fn()
        return out, [tag for tag, _, _ in _ops.kernel_events]
    finally:
        _ops.kernel_events = None


def test_kernel_runs_inside_the_envelope_and_the_composition_outside():
    x = _image(1, 2, 120, 160)
    with torch.no_grad():
        for kw in MODULES.values():
            (pyr, _, _), tags = _tags(lambda: P.ScalePyramid(**kw).cuda()(x))
            assert tags == ["scale_octave_forward"] * len(pyr)
        (pyr, _, _), tags = _tags(lambda: P.ScalePyramid(min_size=8).cuda()(x))  # last octave 15 x 20: below 25 taps
        assert tags[:3] == ["scale_octave_forward"] * 3 and len(pyr) == 4 and "scale_octave_forward" not in tags[3:]
        for sp, y in ((P.ScalePyramid().cuda(), _image(1, 1, 120, 166)),     # W % 4 != 0 in every octave (166, 83, 41)
                      (P.ScalePyramid().cuda(), x.double()),
                      (P.ScalePyramid(n_levels=4).cuda(), x)):                 # a chain that is not instantiated
            (pyr, _, _), tags = _tags(lambda: sp(y))
            assert "scale_octave_forward" not in tags and "sepfilter_forward" in tags
            for a, b in zip(pyr, sp._composed_pyramid(y)[0]):
                assert _bits_equal(a.float(), b.float())
    xg = x.clone().requires_grad_(True)
    (pyr, _, _), tags = _tags(lambda: P.ScalePyramid().cuda()(xg))
    assert "scale_octave_forward" not in tags and pyr[0].grad_fn is not None


@pytest.mark.parametrize("hw", [(7, 9), (33, 40)])
def test_gradcheck_fp64(hw):
    sp = P.ScalePyramid().cuda()
    x = torch.rand(1, 1, *hw, device="cuda", dtype=torch.float64, requires_grad=True)
    assert torch.autograd.gradcheck(lambda t: tuple(sp(t)[0]), (x,), eps=1e-6, atol=1e-5, rtol=1e-4)


@pytest.mark.parametrize("dynamic", [False, True])
def test_torch_compile_equals_eager(dynamic):
    torch._dynamo.reset()
    sp = P.ScalePyramid(3, 1.6, 16, extra_levels=2).cuda()
    x = _image(1, 1, 96, 128, seed=5)
    with torch.no_grad():
        want = sp(x)
        got = torch.compile(sp, fullgraph=True, dynamic=dynamic)(x)
        exact = torch.compile(sp, fullgraph=True, dynamic=dynamic, backend="aot_eager")(x)
    for out in (got, exact):
        assert len(out[0]) == len(want[0]) == 3
        # octave 0 is the octave kernel on the input: the same bits as eager
        assert _bits_equal(out[0][0], want[0][0])
        for a, b in zip(out[1] + out[2], want[1] + want[2]):
            assert torch.equal(a, b)
        # the traced graph decomposes the bilinear resize of the octave seeds into its own ops: a few ulp there, carried
        # through the later octaves
        for a, b in zip(out[0][1:], want[0][1:]):
            torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)


def test_opcheck():
    sp = P.ScalePyramid()
    L = 6
    names = ["_gk_init"] + [f"_gk_{i}" for i in range(L - 1)]
    taps = [v for n in names for v in sp._host_taps[n]]
    ks = [13, 11, 13, 17, 21, 25]
    torch.library.opcheck(torch.ops.kornia_b200.scale_octave_fwd, (_image(1, 2, 40, 64), taps, ks))
    torch.library.opcheck(torch.ops.kornia_b200.scale_octave_fwd, (_image(2, 1, 32, 36), taps[13:], [0] + ks[1:]))


def test_reference_layout_state_dict_loads():
    init, levels = SR.kernels(3, 1.6, False, 2)
    sd = {"_gk_init": init, **{f"_gk_{i}": k for i, k in enumerate(levels)}}
    sp = P.ScalePyramid(3, 1.6, 16, extra_levels=2)
    sp.load_state_dict(sd, strict=True)
    sp = sp.cuda()
    x = _image(1, 1, 64, 96)
    with torch.no_grad():
        _, tags = _tags(lambda: sp(x))
        assert "scale_octave_forward" in tags
        for a, b in zip(sp(x)[0], sp._composed_pyramid(x)[0]):
            assert _bits_equal(a, b)
