"""Sub-pixel refinement on the H100: the kernel (csrc/quad_interp.cuh) through its C entry point against the library's
composition run on the same GPU, bit for bit (values as int32 with any NaN equal to any NaN, into outputs prefilled with
NaN), for both forms and every parameter the goldens cover, with and without a mask, on random, tied, special and
detector-response volumes, full-HD octaves, the widths of later octaves, tiny volumes and permuted (B, C, L, H, W) views;
the goldens; which kernels run inside and outside the envelope; CUDA-graph replay; torch.compile; gradcheck through the
composition; opcheck; and the fused detector pipeline against the composed one."""
import importlib
import itertools
import json
import os
import subprocess
import sys

import pytest
import torch

from conftest import golden

pytestmark = pytest.mark.gpu

K = importlib.import_module("kornia_b200")
Q = importlib.import_module("kornia_b200.geometry.subpix.quad_interp")
_ops = importlib.import_module("kornia_b200._ops")
_lib = importlib.import_module("kornia_b200._lib")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bits_equal(a, b):
    assert a.shape == b.shape and a.dtype == b.dtype and a.stride() == b.stride(), (a.shape, b.shape, a.stride(), b.stride())
    bits = torch.int64 if a.dtype == torch.float64 else torch.int32
    return bool(((a.view(bits) == b.view(bits)) | (a.isnan() & b.isnan())).all())


def _volume(shape, kind, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if kind == "tied":
        return torch.round(torch.rand(shape, device="cuda", generator=g) * 4) / 4
    x = torch.randn(shape, device="cuda", generator=g)
    if kind == "special":
        flat = x.view(-1)
        vals = torch.tensor([float("nan"), float("inf"), float("-inf"), -0.0, 1e-40, -1e-41, 2e-45, 0.0, 3e38], device="cuda")
        idx = torch.randint(0, flat.numel(), (max(9, flat.numel() // 200),), device="cuda", generator=g)
        flat[idx] = vals[torch.arange(idx.numel(), device="cuda") % vals.numel()]
    if kind == "response" and min(shape[-2:]) >= 7:  # BlobHessian of a smooth volume: maxima that rarely move
        B, C, L, H, W = shape
        img = K.filters.gaussian_blur2d(torch.rand(B * C * L, 1, H, W, device="cuda", generator=g), (7, 7), (1.5, 1.5))
        x = K.feature.hessian_response(img).view(shape)
    return x


def _kernel(x, mask, n_iters, bonus, shift, radius, allow):
    """The C entry point into outputs prefilled with NaN: every element must be written."""
    B, C, D, H, W = x.shape
    coords = torch.full((B, C, 3, D, H, W), float("nan"), device="cuda")
    y = torch.empty_like(x).fill_(float("nan"))
    _lib.call("kb200_quad_interp3d_forward", x.data_ptr(), None if mask is None else mask.data_ptr(), coords.data_ptr(), y.data_ptr(),
              B, C, D, H, W, x.stride(0), x.stride(1), x.stride(2), *y.stride(), n_iters, radius, shift, bonus, bonus > 0, allow, _lib.F32,
              torch.cuda.current_stream().cuda_stream)
    return coords, y


def _composed(x, mask, n_iters, bonus, shift, radius, allow):
    if radius:
        return Q._composed_conv_quad_interp3d(x, n_iters, bonus, shift, mask, radius, allow)
    return Q._composed_iterative_quad_interp3d(x, n_iters, bonus, shift, allow, mask, None)


def _masks(x):
    mx, _ = K.geometry.nms3d_minmax(x)
    g = torch.Generator(device="cuda").manual_seed(7)
    border = torch.rand(x.shape, device="cuda", generator=g) < 0.03
    border[..., :, 0, :] = True
    border[..., 0, :, -1] = True
    return {"none": None, "max": mx, "border": border.contiguous()}


FULL = list(itertools.product((0, 1, 5), (0.0, 10.0), (0.6, 0.3), (0, 1, 2), (True, False)))  # n_iters, bonus, shift, radius, allow
DEFAULTS = [(5, 10.0, 0.6, 1, True), (5, 0.0, 0.6, 0, True), (5, 10.0, 0.3, 2, False), (1, 0.0, 0.3, 1, True)]


def _check(x, params):
    # the conv composition views the input as one dimension: a permuted view with C > 1 is composed from a contiguous copy,
    # and its y laid out again at x's strides
    xc = x if x.is_contiguous() or x.shape[1] == 1 else x.contiguous()
    with torch.no_grad():
        for mname, mask in _masks(x).items():
            for n_iters, bonus, shift, radius, allow in params:
                got, want = _kernel(x, mask, n_iters, bonus, shift, radius, allow), _composed(xc, mask, n_iters, bonus, shift, radius, allow)
                want = (want[0], torch.empty_like(x).copy_(want[1]))
                tag = (mname, n_iters, bonus, shift, radius, allow)
                assert _bits_equal(got[0], want[0]), ("coords",) + tag
                assert _bits_equal(got[1], want[1]), ("y",) + tag


SMALL = [(1, 3, 4, 61, 68), (1, 1, 5, 34, 60), (1, 1, 5, 17, 30), (1, 1, 5, 8, 15), (2, 2, 5, 20, 26), (1, 1, 3, 3, 3),
         (1, 1, 2, 9, 9), (1, 2, 4, 2, 9), (1, 1, 4, 7, 1)]


@pytest.mark.parametrize("kind", ["random", "tied", "special", "response"])
@pytest.mark.parametrize("shape", SMALL)
def test_kernel_bit_identical_small(shape, kind):
    _check(_volume(shape, kind, seed=shape[-1]), FULL)


@pytest.mark.parametrize("kind", ["random", "tied", "special", "response"])
@pytest.mark.parametrize("shape", [(1, 1, 5, 1080, 1920), (2, 1, 5, 540, 960), (1, 1, 5, 135, 240)])
def test_kernel_bit_identical_octaves(shape, kind):
    _check(_volume(shape, kind, seed=shape[-1]), DEFAULTS)


@pytest.mark.parametrize("kind", ["random", "special", "response"])
@pytest.mark.parametrize("shape", [(2, 3, 5, 40, 52), (1, 1, 5, 270, 480)])
def test_permuted_views_read_in_place(shape, kind):
    B, C, L, H, W = shape
    x = _volume((B, L, C, H, W), kind, seed=W).permute(0, 2, 1, 3, 4)  # ScaleSpaceDetector's view of a (B, L, C, H, W) response
    _check(x, DEFAULTS)


# The profiler run happens in a fresh interpreter: in a process where a profiler session was followed by torch.compile
# (as test_nms_gpu.py does), later torch.profiler sessions on this torch return no CUDA events at all.
_PROFILE = r"""
import json, torch
import kornia_b200 as K
from kornia_b200.geometry.subpix import quad_interp as Q

def kernels(fn):
    fn()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]

g = torch.Generator(device="cuda").manual_seed(0)
img = K.filters.gaussian_blur2d(torch.rand(5, 1, 96, 128, device="cuda", generator=g), (7, 7), (1.5, 1.5))
x = K.feature.hessian_response(img).view(1, 5, 1, 96, 128).permute(0, 2, 1, 3, 4)  # the detector's (B, C, L, H, W) view
mask, _ = K.geometry.nms3d_minmax(x)
with torch.no_grad():
    inside = [kernels(fn) for fn in (lambda: Q.conv_quad_interp3d(x, precomputed_nms_mask=mask), lambda: Q.conv_quad_interp3d(x),
                                     lambda: Q.iterative_quad_interp3d(x), lambda: Q.AdaptiveQuadInterp3d(strict_maxima_bonus=0.0)(x, mask))]
    outside = kernels(lambda: Q.conv_quad_interp3d(x.double(), precomputed_nms_mask=mask))
print(json.dumps({"inside": inside, "outside": outside}))
"""


def test_one_kernel_per_call_on_the_detector_view():
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT] + [p for p in os.environ.get("PYTHONPATH", "").split(os.pathsep) if p]))
    run = subprocess.run([sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _PROFILE], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert run.returncode == 0, run.stdout[-2000:] + run.stderr[-4000:]
    got = json.loads(run.stdout.strip().splitlines()[-1])
    for names in got["inside"]:
        assert len(names) == 1 and "quad_interp3d_kernel" in names[0], names
    # outside the envelope (fp64) the composition runs: many ATen kernels, none of them the fused one
    assert len(got["outside"]) > 10 and not any("quad_interp3d_kernel" in n for n in got["outside"]), got["outside"]


G = golden("subpix")
ERRORS = {
    "type": lambda x: Q.conv_quad_interp3d(x.cpu().numpy()),
    "type_iterative": lambda x: Q.iterative_quad_interp3d([1.0]),
    "ndim": lambda x: Q.conv_quad_interp3d(x[0]),
    "ndim_iterative": lambda x: Q.iterative_quad_interp3d(x[:, :, 0]),
    "view": lambda x: Q.conv_quad_interp3d(x.transpose(1, 2)),
    "mode": lambda x: Q.AdaptiveQuadInterp3d("fast"),
}


@pytest.mark.parametrize("name", G.names())
def test_public_functions_match_reference_goldens(name):
    op, kw, ins, outs = G.case(name)
    if "plateau" in name and ("max_candidates=5" in kw.get("repr", "") or kw.get("max_candidates")):
        pytest.skip("max_candidates ranks tied responses with torch.topk, whose order among ties differs between CPU and CUDA")
    x = ins["input"].cuda()
    mask = ins["mask"].cuda() if "mask" in ins else None
    if "error" in kw:
        with pytest.raises((TypeError, ValueError, RuntimeError)) as e:
            ERRORS[kw["case"]](x)
        assert type(e.value).__name__ == kw["error"] and str(e.value) == kw["message"]
        return
    with torch.no_grad():
        if op == "module":
            m = eval(kw["repr"], {n: getattr(Q, n) for n in Q.__all__})
            coords, y = m(x, mask)
        elif op == "conv":
            coords, y = Q.conv_quad_interp3d(x, kw["n_iters"], kw["strict_maxima_bonus"], kw["max_subpixel_shift"], mask, kw["dilation_radius"],
                                             kw["allow_scale_steps"])
        else:
            coords, y = Q.iterative_quad_interp3d(x, kw["n_iters"], kw["strict_maxima_bonus"], kw["max_subpixel_shift"], kw["allow_scale_steps"],
                                                  mask, kw.get("max_candidates"))
    assert _bits_equal(coords.cpu(), outs["coords"]) and _bits_equal(y.cpu(), outs["y"])


def _tags(fn):
    _ops.kernel_events = []
    try:
        out = fn()
        return out, [tag for tag, _, _ in _ops.kernel_events]
    finally:
        _ops.kernel_events = None


def test_kernel_runs_inside_the_envelope_and_the_composition_outside():
    x = _volume((1, 2, 4, 30, 41), "random")
    mx, _ = K.geometry.nms3d_minmax(x)
    with torch.no_grad():
        for fn in (lambda: Q.conv_quad_interp3d(x), lambda: Q.conv_quad_interp3d(x, precomputed_nms_mask=mx),
                   lambda: Q.conv_quad_interp3d(x, dilation_radius=3), lambda: Q.iterative_quad_interp3d(x, precomputed_nms_mask=mx),
                   lambda: Q.ConvQuadInterp3d()(x), lambda: Q.IterativeQuadInterp3d()(x, mx), lambda: Q.AdaptiveQuadInterp3d()(x, mx)):
            assert _tags(fn)[1] == ["quad_interp3d_forward"]
        outside = [
            (lambda: Q.conv_quad_interp3d(x.double()), lambda: Q._composed_conv_quad_interp3d(x.double(), 5, 10.0, 0.6, None, 1, True)),
            (lambda: Q.conv_quad_interp3d(x, dilation_radius=0), lambda: Q._composed_conv_quad_interp3d(x, 5, 10.0, 0.6, None, 0, True)),
            (lambda: Q.iterative_quad_interp3d(x, max_candidates=10),
             lambda: Q._composed_iterative_quad_interp3d(x, 5, 10.0, 0.6, True, None, 10)),
            (lambda: Q.conv_quad_interp3d(x, precomputed_nms_mask=mx.to(torch.uint8)),
             lambda: Q._composed_conv_quad_interp3d(x, 5, 10.0, 0.6, mx.to(torch.uint8), 1, True)),
            (lambda: Q.iterative_quad_interp3d(x, precomputed_nms_mask=mx.transpose(3, 4).contiguous().transpose(3, 4)),
             lambda: Q._composed_iterative_quad_interp3d(x, 5, 10.0, 0.6, True, mx, None)),
            (lambda: Q.AdaptiveQuadInterp3d("patch", max_candidates=3)(x), lambda: Q._composed_iterative_quad_interp3d(x, 5, 10.0, 0.6, True, None, 3)),
        ]
        for fn, want in outside:
            out, tags = _tags(fn)
            assert "quad_interp3d_forward" not in tags and all(_bits_equal(a, b) for a, b in zip(out, want()))  # nms3d may run fused
    xg = x.clone().requires_grad_(True)
    (coords, y), tags = _tags(lambda: Q.conv_quad_interp3d(xg))
    assert tags == ["nms3d_forward"] and y.grad_fn is not None  # the mask needs no gradient; the refinement is composed


def test_cuda_graph_replay_equals_eager():
    x = _volume((2, 1, 5, 90, 120), "random")
    mx, _ = K.geometry.nms3d_minmax(x)
    with torch.no_grad():
        want = [Q.conv_quad_interp3d(x, precomputed_nms_mask=mx), Q.conv_quad_interp3d(x), Q.iterative_quad_interp3d(x, 5, 0.0, 0.3)]
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                Q.conv_quad_interp3d(x, precomputed_nms_mask=mx)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            got = [Q.conv_quad_interp3d(x, precomputed_nms_mask=mx), Q.conv_quad_interp3d(x), Q.iterative_quad_interp3d(x, 5, 0.0, 0.3)]
        x.copy_(_volume(x.shape, "special", seed=3))  # new data in the captured buffers
        mx.copy_(K.geometry.nms3d_minmax(x)[0])
        graph.replay()
        torch.cuda.synchronize()
        want = [Q.conv_quad_interp3d(x, precomputed_nms_mask=mx), Q.conv_quad_interp3d(x), Q.iterative_quad_interp3d(x, 5, 0.0, 0.3)]
    for a, b in zip(got, want):
        assert _bits_equal(a[0], b[0]) and _bits_equal(a[1], b[1])


class _Refiner(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.conv = Q.ConvQuadInterp3d(strict_maxima_bonus=0.0)
        self.adaptive = Q.AdaptiveQuadInterp3d()

    def forward(self, resp):
        mx, mn = K.geometry.nms3d_minmax(resp)
        return self.adaptive(resp, mx) + self.adaptive(-resp, mn) + self.conv(resp) + Q.iterative_quad_interp3d(resp, 3, 1.0, 0.3)


@pytest.mark.parametrize("dynamic", [False, True])
def test_torch_compile_equals_eager(dynamic):
    torch._dynamo.reset()
    det = _Refiner()
    with torch.no_grad():
        for H, W in ((48, 64), (40, 56)):
            resp = _volume((1, 5, 1, H, W), "random").permute(0, 2, 1, 3, 4)
            want = det(resp)
            got = torch.compile(det, fullgraph=True, dynamic=dynamic)(resp)
            for a, b in zip(got, want):
                assert _bits_equal(a, b)


def test_gradcheck_through_the_composition_fp64():
    x = torch.randn(1, 1, 4, 9, 10, device="cuda", dtype=torch.float64, requires_grad=True)
    for f in (lambda t: Q.conv_quad_interp3d(t, 3, 1.0, 0.3)[1], lambda t: Q.iterative_quad_interp3d(t, 3, 1.0, 0.3)[1],
              lambda t: Q.conv_quad_interp3d(t, 3, 1.0, 0.3)[0]):
        assert torch.autograd.gradcheck(f, (x,), eps=1e-6, atol=1e-6)


def test_opcheck():
    x = _volume((1, 2, 4, 18, 21), "random")
    mx, _ = K.geometry.nms3d_minmax(x)
    for mask, radius in ((None, 1), (mx, 2), (None, 0), (mx, 0)):
        torch.library.opcheck(torch.ops.kornia_b200.quad_interp3d_fwd, (x, mask, 5, 0.6, 10.0, radius, True))
    torch.library.opcheck(torch.ops.kornia_b200.quad_interp3d_fwd, (x.permute(0, 2, 1, 3, 4), None, 3, 0.3, 0.0, 1, False))


def _detector_octave(img):
    """ScalePyramid -> hessian_response of each level -> nms3d_minmax -> AdaptiveQuadInterp3d with the max mask, as
    ScaleSpaceDetector chains them for its first octave."""
    pyr, sigmas, _ = K.geometry.ScalePyramid(3, 1.6, 15)(img)
    octave, sig = pyr[0], sigmas[0]
    B, C, L, H, W = octave.shape
    resp = K.feature.hessian_response(octave.permute(0, 2, 1, 3, 4).reshape(B * L, C, H, W), sigmas=sig.reshape(-1))
    resp = resp.view(B, L, C, H, W).permute(0, 2, 1, 3, 4)
    mx, _ = K.geometry.nms3d_minmax(resp)
    return Q.AdaptiveQuadInterp3d(strict_maxima_bonus=0.0)(resp, mx)


def test_fused_pipeline_equals_composed_pipeline_full_hd():
    g = torch.Generator(device="cuda").manual_seed(5)
    img = K.filters.gaussian_blur2d(torch.rand(1, 1, 1080, 1920, device="cuda", generator=g), (9, 9), (2.0, 2.0))
    with torch.no_grad():
        fused = _detector_octave(img)
    composed = _detector_octave(img.clone().requires_grad_(True))  # a gradient-tracked input takes every stage's composition
    assert composed[1].grad_fn is not None
    assert _bits_equal(fused[0], composed[0].detach()) and _bits_equal(fused[1], composed[1].detach())
