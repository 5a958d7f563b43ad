"""Non-maximum suppression on the H100: the 2-D and 3-D kernels (csrc/nms.cuh) against the library's composition run on
the same GPU, bit for bit (masks byte for byte into outputs prefilled with 0xFF, values as int32 with any NaN equal to any
NaN), for every instantiated K, on random, heavily tied and special texels, full-HD frames, the widths of ScalePyramid's
later octaves and tiny images; permuted (B, C, L, H, W) views read in place; the public functions against the
reference's goldens; which kernels run inside and outside the envelope; gradcheck; torch.compile; opcheck; install()."""
import importlib
import sys

import pytest
import torch

import helpers
from conftest import golden

pytestmark = pytest.mark.gpu

K = importlib.import_module("kornia_b200")
N = importlib.import_module("kornia_b200.geometry.subpix.nms")
_ops = importlib.import_module("kornia_b200._ops")
_lib = importlib.import_module("kornia_b200._lib")

SIZES = list(range(3, 32, 2))
SMALL = [(2, 1, 67, 120), (1, 3, 33, 60), (2, 1, 16, 30), (1, 1, 8, 15), (1, 1, 61, 68), (1, 1, 2, 2), (1, 1, 1, 1)]
BIG = [(1, 1, 1080, 1920), (1, 2, 720, 1280)]


def _bits_equal(a, b):
    assert a.shape == b.shape and a.dtype == b.dtype
    if a.dtype == torch.bool:
        return torch.equal(a, b)
    return bool(((a.view(torch.int32) == b.view(torch.int32)) | (a.isnan() & b.isnan())).all())


def _texels(shape, kind, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if kind == "tied":
        return torch.round(torch.rand(shape, device="cuda", generator=g) * 6) / 4 - 0.5
    x = torch.rand(shape, device="cuda", generator=g) * 2 - 1
    if kind == "special":
        flat = x.view(-1)
        vals = torch.tensor([float("nan"), float("inf"), float("-inf"), -0.0, 1e-40, -1e-41, 2e-45, 0.0, -0.25, 3e38], device="cuda")
        idx = torch.randint(0, flat.numel(), (max(10, flat.numel() // 300),), device="cuda", generator=g)
        flat[idx] = vals[torch.arange(idx.numel(), device="cuda") % vals.numel()]
        x[..., : max(1, x.shape[-2] // 5), :] = -0.75  # a negative plateau: ties, and negative peaks next to it
    return x


def _kernel2d(x, k, mask_only):
    """The C entry point into an output prefilled with 0xFF bytes (mask) or NaN (values): every element must be written."""
    B, C, H, W = x.shape
    out = torch.full((B, C, H, W), 255, device="cuda", dtype=torch.uint8) if mask_only else torch.full((B, C, H, W), float("nan"), device="cuda")
    _lib.call("kb200_nms2d_forward", x.data_ptr(), out.data_ptr(), B, C, H, W, x.stride(0), x.stride(1), k, 0 if mask_only else 1, _lib.F32,
              torch.cuda.current_stream().cuda_stream)
    return out


def _composed2d(x, k, mask_only):
    m = N.NonMaximaSuppression2d((k, k)).cuda()
    return N._composed_nms2d(x, m.kernel_size, m.padding, m.kernel, mask_only)


def _check2d(x, k):
    with torch.no_grad():
        for mask_only in (True, False):
            got, want = _kernel2d(x, k, mask_only), _composed2d(x, k, mask_only)
            if mask_only:
                assert torch.equal(got, want.to(torch.uint8)), (k, "mask")
            else:
                assert _bits_equal(got, want), (k, "values")


@pytest.mark.parametrize("kind", ["random", "tied", "special"])
@pytest.mark.parametrize("shape", SMALL)
@pytest.mark.parametrize("k", SIZES)
def test_nms2d_kernel_bit_identical_small(k, shape, kind):
    _check2d(_texels(shape, kind, seed=k), k)


@pytest.mark.parametrize("kind", ["random", "tied", "special"])
@pytest.mark.parametrize("shape", BIG)
@pytest.mark.parametrize("k", [3, 5, 7, 9, 15, 31])
def test_nms2d_kernel_bit_identical_full_frames(k, shape, kind):
    if k == 31 and shape == BIG[0]:
        shape = (1, 1, 540, 960)  # the composition's 961 neighbour planes of a full-HD frame would take 16 GB
    _check2d(_texels(shape, kind, seed=k), k)


def _kernel3d(x, mode):
    B, C, L, H, W = x.shape
    nan_or_ff = (lambda: torch.full(x.shape, float("nan"), device="cuda")) if mode == 1 else (lambda: torch.full(x.shape, 255, device="cuda", dtype=torch.uint8))
    out0 = nan_or_ff()
    out1 = torch.full(x.shape, 255, device="cuda", dtype=torch.uint8)
    _lib.call("kb200_nms3d_forward", x.data_ptr(), out0.data_ptr(), out1.data_ptr(), B, C, L, H, W, x.stride(0), x.stride(1), x.stride(2), mode,
              _lib.F32, torch.cuda.current_stream().cuda_stream)
    return out0, out1


SHAPES3 = [(1, 1, 5, 1080, 1920), (2, 3, 4, 135, 240), (1, 2, 5, 16, 30), (1, 1, 3, 8, 15), (1, 1, 1, 1, 1), (1, 1, 3, 2, 2), (1, 1, 2, 61, 68)]


@pytest.mark.parametrize("kind", ["random", "tied", "special"])
@pytest.mark.parametrize("permuted", [False, True])
@pytest.mark.parametrize("shape", SHAPES3)
def test_nms3d_kernel_bit_identical(shape, permuted, kind):
    B, C, L, H, W = shape
    x = _texels((B, L, C, H, W), kind, seed=L).permute(0, 2, 1, 3, 4) if permuted else _texels(shape, kind, seed=L)
    m3 = N.NonMaximaSuppression3d((3, 3, 3))
    with torch.no_grad():
        mx, _ = _kernel3d(x, 0)
        assert torch.equal(mx, N._composed_nms3d(x, m3.kernel_size, m3.padding, m3.kernel, True).to(torch.uint8))
        vals, _ = _kernel3d(x, 1)
        assert _bits_equal(vals, N._composed_nms3d(x, m3.kernel_size, m3.padding, m3.kernel, False))
        mx, mn = _kernel3d(x, 2)
        wmx, wmn = N._composed_nms3d_minmax(x)
        assert torch.equal(mx, wmx.to(torch.uint8)) and torch.equal(mn, wmn.to(torch.uint8))


def _cuda_kernels(fn):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    return out, [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def test_permuted_views_are_read_in_place():
    base = _texels((2, 5, 3, 64, 96), "tied")
    x = base.permute(0, 2, 1, 3, 4)  # ScaleSpaceDetector's (B, C, L, H, W) view of a (B, L, C, H, W) response
    assert not x.is_contiguous()
    N.nms3d_minmax(x)
    (mx, mn), names = _cuda_kernels(lambda: N.nms3d_minmax(x))
    assert len(names) == 1 and "nms3d_kernel" in names[0], names
    wmx, wmn = N._composed_nms3d_minmax(x)
    assert torch.equal(mx, wmx) and torch.equal(mn, wmn)
    y = _texels((3, 2, 50, 70), "tied").transpose(0, 1)  # (B, C) strides swapped, planes dense
    out, names = _cuda_kernels(lambda: N.nms2d(y, (9, 9), True))
    assert len(names) == 1 and "nms2d_kernel" in names[0], names
    assert torch.equal(out, _composed2d(y, 9, True))


G = golden("nms")


@pytest.mark.parametrize("name", G.names())
def test_public_functions_match_reference_goldens(name):
    op, kw, ins, outs = G.case(name)
    x = ins["input"].cuda()
    ks = tuple(kw.get("kernel_size", ()))
    run = {"nms2d": lambda: {"out": N.nms2d(x, ks, kw["mask_only"])},
           "nms3d": lambda: {"out": N.nms3d(x, ks, kw["mask_only"])},
           "nms3d_minmax": lambda: dict(zip(("max", "min"), N.nms3d_minmax(x)))}[op]
    if "error" in kw:
        with pytest.raises(RuntimeError) as e:
            run()
        assert str(e.value) == kw["message"]
        return
    with torch.no_grad():
        got = run()
    for k, want in outs.items():
        assert _bits_equal(got[k].cpu(), want), k


def _tags(fn):
    _ops.kernel_events = []
    try:
        out = fn()
        return out, [tag for tag, _, _ in _ops.kernel_events]
    finally:
        _ops.kernel_events = None


def test_kernel_runs_inside_the_envelope_and_the_composition_outside():
    x = _texels((1, 2, 40, 52), "tied")
    v = _texels((1, 2, 4, 40, 52), "tied")
    with torch.no_grad():
        for k in SIZES:
            for mask_only in (True, False):
                _, tags = _tags(lambda: N.nms2d(x, (k, k), mask_only))
                assert tags == ["nms2d_forward"], (k, mask_only)
                _, tags = _tags(lambda: N.NonMaximaSuppression2d((k, k)).cuda()(x, mask_only))
                assert tags == ["nms2d_forward"], (k, mask_only)
        for mask_only in (True, False):
            assert _tags(lambda: N.nms3d(v, (3, 3, 3), mask_only))[1] == ["nms3d_forward"]
        assert _tags(lambda: N.nms3d_minmax(v))[1] == ["nms3d_forward"]
        for fn in (lambda: N.nms2d(x.double(), (5, 5)), lambda: N.nms2d(x, (33, 33)), lambda: N.nms3d(v.double(), (3, 3, 3)),
                   lambda: N.nms3d_minmax(v.double()), lambda: N.nms2d(x.half(), (3, 3), True)):
            out, tags = _tags(fn)
            assert tags == []
        out, tags = _tags(lambda: N.nms2d(x.double(), (9, 9), True))
        assert tags == [] and torch.equal(out, _composed2d(x, 9, True))
        for ks in ((4, 4), (3, 5)):
            with pytest.raises(RuntimeError):
                N.nms2d(x, ks, True)
    xg = x.clone().requires_grad_(True)
    vg = v.clone().requires_grad_(True)
    out, tags = _tags(lambda: N.nms2d(xg, (15, 15)))
    assert tags == [] and out.grad_fn is not None
    out, tags = _tags(lambda: N.nms3d(vg, (3, 3, 3)))
    assert tags == [] and out.grad_fn is not None
    out, tags = _tags(lambda: N.nms2d(xg, (15, 15), True))  # the mask needs no gradient: fused
    assert tags == ["nms2d_forward"] and torch.equal(out, _composed2d(x, 15, True))
    assert _tags(lambda: N.nms3d_minmax(vg))[1] == ["nms3d_forward"]


@pytest.mark.parametrize("k", [3, 9])
def test_gradcheck_values_fp64(k):
    x = torch.rand(1, 2, 11, 13, device="cuda", dtype=torch.float64, requires_grad=True)
    assert torch.autograd.gradcheck(lambda t: N.nms2d(t, (k, k)), (x,), eps=1e-6, atol=1e-7)
    v = torch.rand(1, 1, 4, 9, 10, device="cuda", dtype=torch.float64, requires_grad=True)
    assert torch.autograd.gradcheck(lambda t: N.nms3d(t, (3, 3, 3)), (v,), eps=1e-6, atol=1e-7)


class _Detector(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.nms = N.NonMaximaSuppression2d((15, 15))

    def forward(self, resp, octave):
        mx, mn = N.nms3d_minmax(octave)
        return self.nms(resp, True), self.nms(resp), N.nms2d(resp, (5, 5), True), N.nms3d(octave, (3, 3, 3)), mx, mn


@pytest.mark.parametrize("dynamic", [False, True])
def test_torch_compile_equals_eager(dynamic):
    torch._dynamo.reset()
    det = _Detector().cuda()
    with torch.no_grad():
        for H, W in ((48, 64), (40, 56)):
            resp, octave = _texels((1, 2, H, W), "special"), _texels((1, 1, 5, H, W), "tied")
            want = det(resp, octave)
            got = torch.compile(det, fullgraph=True, dynamic=dynamic)(resp, octave)
            for a, b in zip(got, want):
                assert _bits_equal(a, b)


def test_opcheck():
    x = _texels((2, 3, 20, 27), "tied")  # opcheck compares with assert_close, where NaN != NaN
    for k in (3, 15):
        for mask_only in (True, False):
            torch.library.opcheck(torch.ops.kornia_b200.nms2d_fwd, (x, k, mask_only))
    v = _texels((1, 2, 4, 18, 21), "tied")
    for mask_only in (True, False):
        torch.library.opcheck(torch.ops.kornia_b200.nms3d_fwd, (v, mask_only))
    torch.library.opcheck(torch.ops.kornia_b200.nms3d_minmax_fwd, (v,))
    torch.library.opcheck(torch.ops.kornia_b200.nms3d_minmax_fwd, (v.permute(0, 2, 1, 3, 4),))


_CALLERS = {
    "__init__": "from . import filters, geometry, metrics, losses, augmentation, feature",
    "geometry/__init__": "from . import transform, calibration, subpix\nfrom .transform import warp_perspective, warp_affine, remap",
    "geometry/subpix/__init__": "from .nms import nms2d, nms3d_minmax",
    "geometry/subpix/nms": "def nms2d(*a, **k): raise AssertionError('reference nms2d')\ndef nms3d_minmax(*a): raise AssertionError('reference')",
    "feature/__init__": "from . import scale_space_detector, xfeat",
    "feature/scale_space_detector": "from kornia.geometry.subpix import nms3d_minmax\ndef octave_masks(r):\n    return nms3d_minmax(r)",
    "feature/xfeat": "from kornia.geometry.subpix import nms2d\ndef keypoints(s):\n    return nms2d(s, (5, 5), True)",
}


def test_install_runs_the_fused_kernels_by_global_name(tmp_path, monkeypatch):
    monkeypatch.setattr(helpers, "_STANDIN_KORNIA", {**helpers._STANDIN_KORNIA, **_CALLERS})
    resp = _texels((1, 3, 5, 40, 48), "tied").permute(0, 2, 1, 3, 4)
    score = _texels((2, 1, 40, 48), "tied")
    with helpers.standin_kornia(tmp_path):
        ssd = sys.modules["kornia.feature.scale_space_detector"]
        xfeat = sys.modules["kornia.feature.xfeat"]
        try:
            K.install(sys.modules["kornia"])
            with torch.no_grad():
                (mx, mn), tags = _tags(lambda: ssd.octave_masks(resp))
                assert tags == ["nms3d_forward"]
                assert all(torch.equal(a, b) for a, b in zip((mx, mn), N._composed_nms3d_minmax(resp)))
                m, tags = _tags(lambda: xfeat.keypoints(score))
                assert tags == ["nms2d_forward"] and torch.equal(m, _composed2d(score, 5, True))
        finally:
            K.uninstall()
