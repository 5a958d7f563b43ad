"""GPU parity of the callers either side of the hot path (SURVEY.md 8f rows 1-3) through the C ABI:
golden vectors recorded from the reference (fp32 CPU), the oracle in fp64, and size-independent
properties at full image sizes.  Tolerances as in test_parity_gpu.py."""
import pytest
import torch

import kornia_b200 as K
from conftest import golden
from helpers import family_grads, rel_l2, run_family_case
from oracle import kornia_restated as R

pytestmark = pytest.mark.gpu
FAM = golden("family")
FP32 = dict(rtol=1e-4, atol=1e-5)
DEV = "cuda"
FWD = [n for n in FAM.names() if not FAM.meta[n]["op"].endswith("_grad")]
GRAD = [n for n in FAM.names() if FAM.meta[n]["op"].endswith("_grad")]


def _impl(op):
    base = op[:-5] if op.endswith("_grad") else op
    return K.filters if hasattr(K.filters, base) else K.geometry.transform


def _tieflip(got, want, frac=0.02):
    bad = (got - want).abs() > (1e-5 + 1e-4 * want.abs())
    assert bad.float().mean().item() <= frac, f"{bad.sum().item()} / {bad.numel()} mismatches"


@pytest.mark.parametrize("name", FWD)
def test_family_forward_matches_reference(name):
    op, kw, ins, outs = FAM.case(name)
    got = run_family_case(_impl(op), op, kw, ins, device=DEV)
    assert got.is_cuda and got.dtype == outs["out"].dtype and got.shape == outs["out"].shape
    assert got.is_contiguous() or got.dim() == 3  # images come back dense; the (B,2,3) builders return a row slice like the reference
    if kw.get("mode") == "nearest":
        _tieflip(got.cpu(), outs["out"])
    else:
        torch.testing.assert_close(got.cpu(), outs["out"], **FP32)


@pytest.mark.parametrize("name", GRAD)
def test_family_grads_match_reference(name):
    op, kw, ins, outs = FAM.case(name)
    got = family_grads(_impl(op), op, kw, ins, outs, device=DEV)
    for key, want in outs.items():
        if key != "cot":
            assert rel_l2(got[key].cpu(), want) < 1e-4, (key, rel_l2(got[key].cpu(), want))


@pytest.mark.parametrize("name", [n for n in FWD if FAM.meta[n]["op"] in ("spatial_gradient", "sobel", "laplacian", "box_blur")][::3])
def test_family_filters_fp64_match_oracle(name):
    op, kw, ins, _ = FAM.case(name)
    got = run_family_case(K.filters, op, kw, ins, device=DEV, dtype=torch.float64)
    want = run_family_case(R, op, kw, ins, dtype=torch.float64)
    # fp64-grade agreement (four orders beyond fp32); the host BLAS behind the oracle's fp64 convolution differs from
    # box to box at the 1e-11 level (observed), hence not tighter
    torch.testing.assert_close(got.cpu(), want, rtol=1e-9, atol=1e-10)


@pytest.mark.parametrize("name", [n for n in GRAD if FAM.meta[n]["op"] in ("spatial_gradient_grad", "sobel_grad")])
def test_family_filter_grads_fp64_match_oracle(name):
    op, kw, ins, outs = FAM.case(name)
    got = family_grads(K.filters, op, kw, ins, outs, device=DEV, dtype=torch.float64)
    want = family_grads(R, op, kw, ins, outs, dtype=torch.float64)
    for key in want:
        assert rel_l2(got[key].cpu(), want[key]) < 1e-9, key


def test_spatial_gradient_gradcheck():
    x = torch.rand(2, 2, 6, 7, device=DEV, dtype=torch.float64, requires_grad=True)
    for mode, order in (("sobel", 1), ("diff", 2), ("sobel", 2)):
        assert torch.autograd.gradcheck(lambda t: K.filters.spatial_gradient(t, mode, order), (x,), fast_mode=True)
    assert torch.autograd.gradcheck(K.filters.sobel, (x,), fast_mode=True)


def test_sobel_fused_equals_composed_path():
    """The one-kernel magnitude (no-grad call) and the differentiable composition are the same numbers."""
    x = torch.rand(3, 3, 67, 92, device=DEV)
    fused = K.filters.sobel(x)
    composed = K.filters.sobel(x.clone().requires_grad_(True)).detach()
    torch.testing.assert_close(fused, composed, rtol=1e-6, atol=1e-7)
    assert K._ops.launch_count > 0


def test_spatial_gradient_unaligned_and_many_planes():
    # storage offset of one float: the vector path must be skipped, results unchanged
    buf = torch.rand(2 * 3 * 16 * 32 + 1, device=DEV)
    x = buf[1:].view(2, 3, 16, 32)
    assert x.is_contiguous() and x.data_ptr() % 16 != 0
    torch.testing.assert_close(K.filters.spatial_gradient(x), K.filters.spatial_gradient(x.clone()), rtol=0, atol=0)
    torch.testing.assert_close(K.filters.sobel(x), K.filters.sobel(x.clone()), rtol=0, atol=0)
    # more planes than gridDim.z holds: the kernels loop over planes
    # the oracle's convolutions run with cuDNN off, as in test_parity_gpu.py: cuDNN may pick TF32 kernels for an fp32 conv
    many = torch.rand(70000, 1, 4, 4, device=DEV)
    got = K.filters.spatial_gradient(many)
    with torch.backends.cudnn.flags(enabled=False):
        want = R.spatial_gradient(many[-9:])
    torch.testing.assert_close(got[-9:], want, **FP32)
    g = torch.rand_like(got)
    leaf = many.clone().requires_grad_(True)
    (K.filters.spatial_gradient(leaf) * g).sum().backward()
    ref_leaf = many[-5:].clone().requires_grad_(True)
    with torch.backends.cudnn.flags(enabled=False):
        (R.spatial_gradient(ref_leaf) * g[-5:]).sum().backward()
    torch.testing.assert_close(leaf.grad[-5:], ref_leaf.grad, **FP32)


def test_full_size_properties():
    """1080p, size-independent checks: a plane a*x + b*y + c has constant derivatives (a, b) away from
    the border (replicate padding flattens the border itself), zero second derivatives and zero Laplacian;
    a box blur leaves it unchanged in the interior; rotate by 0 and a unit scale are identities."""
    H, W = 1080, 1920
    ys, xs = torch.meshgrid(torch.arange(H, device=DEV, dtype=torch.float32), torch.arange(W, device=DEV, dtype=torch.float32),
                            indexing="ij")
    a, b, c = 0.25, -0.5, 3.0
    plane = (a * xs + b * ys + c)[None, None].expand(2, 3, H, W).contiguous()
    g = K.filters.spatial_gradient(plane, "sobel", 1, normalized=True)
    torch.testing.assert_close(g[:, :, 0, 1:-1, 1:-1], torch.full_like(g[:, :, 0, 1:-1, 1:-1], a), rtol=0, atol=2e-4)
    torch.testing.assert_close(g[:, :, 1, 1:-1, 1:-1], torch.full_like(g[:, :, 1, 1:-1, 1:-1], b), rtol=0, atol=2e-4)
    g2 = K.filters.spatial_gradient(plane, "diff", 2, normalized=False)
    assert float(g2[:, :, :, 2:-2, 2:-2].abs().max()) < 2e-3
    mag = K.filters.sobel(plane, eps=0.0)
    torch.testing.assert_close(mag[:, :, 1:-1, 1:-1], torch.full_like(mag[:, :, 1:-1, 1:-1], (a * a + b * b) ** 0.5), rtol=0, atol=3e-4)
    assert float(K.filters.laplacian(plane, 5)[:, :, 2:-2, 2:-2].abs().max()) < 5e-3
    torch.testing.assert_close(K.filters.box_blur(plane, (5, 7))[:, :, 2:-2, 3:-3], plane[:, :, 2:-2, 3:-3], rtol=1e-5, atol=1e-3)
    noise = torch.rand(2, 3, H, W, device=DEV)
    torch.testing.assert_close(K.geometry.transform.rotate(noise, torch.zeros(2, device=DEV)), noise, rtol=0, atol=1e-3)
    torch.testing.assert_close(K.geometry.transform.scale(noise, torch.ones(2, 2, device=DEV)), noise, rtol=0, atol=1e-3)
    torch.testing.assert_close(K.geometry.transform.center_crop(noise, (H - 2, W - 2)), noise[:, :, 1:-1, 1:-1], rtol=0, atol=1e-3)
    # unsharp_mask = 2*x - blur(x): against the blur kernel itself
    blur = K.filters.gaussian_blur2d(noise, (5, 5), (1.5, 1.5))
    torch.testing.assert_close(K.filters.unsharp_mask(noise, (5, 5), (1.5, 1.5)), 2 * noise - blur, rtol=1e-5, atol=1e-6)


def test_mid_size_matches_oracle_on_device():
    """270x480 batches: CUDA path vs the oracle (the reference's torch composition) on the same device."""
    x = torch.rand(4, 3, 270, 480, device=DEV)
    for mode, order in (("sobel", 1), ("sobel", 2), ("diff", 1), ("diff", 2)):
        torch.testing.assert_close(K.filters.spatial_gradient(x, mode, order), R.spatial_gradient(x, mode, order), **FP32)
    torch.testing.assert_close(K.filters.sobel(x), R.sobel(x), **FP32)
    torch.testing.assert_close(K.filters.box_blur(x, 5), R.box_blur(x, 5), **FP32)
    torch.testing.assert_close(K.filters.box_blur(x, (3, 7), "replicate", True), R.box_blur(x, (3, 7), "replicate", True), **FP32)
    torch.testing.assert_close(K.filters.laplacian(x, 7), R.laplacian(x, 7), **FP32)
    torch.testing.assert_close(K.filters.unsharp_mask(x, (7, 7), (2.0, 2.0)), R.unsharp_mask(x, (7, 7), (2.0, 2.0)), **FP32)
    ang = torch.tensor([10.0, -33.0, 170.0, 91.0], device=DEV)
    smooth = torch.nn.functional.interpolate(torch.rand(4, 3, 9, 16, device=DEV), size=(270, 480), mode="bicubic", align_corners=True)
    # the one-launch rotation matrix may differ from the torch op sequence in the last bit: a sample then crosses a texel
    # or the image border a hair earlier or later (the reference's own CPU and CUDA outputs differ the same way)
    _tieflip(K.geometry.transform.rotate(smooth, ang), R.rotate(smooth, ang), frac=1e-3)
    boxes = torch.tensor([[[10.0, 20.0], [300.0, 25.0], [310.0, 200.0], [5.0, 180.0]]], device=DEV).expand(4, 4, 2).contiguous()
    _tieflip(K.geometry.transform.crop_and_resize(smooth, boxes, (128, 160)), R.crop_and_resize(smooth, boxes, (128, 160)), frac=1e-3)


def _jittered_quads(B, H, W, dtype):
    g = torch.Generator().manual_seed(7)
    quad = torch.tensor([[0.0, 0.0], [W - 1.0, 0.0], [W - 1.0, H - 1.0], [0.0, H - 1.0]]).expand(B, 4, 2)
    return quad.contiguous().to(DEV, dtype), (quad + 8.0 * torch.randn(B, 4, 2, generator=g)).to(DEV, dtype)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_fused_perspective_from_points_matches_torch_ops(dtype, monkeypatch):
    """One-launch get_perspective_transform vs the reference's torch op sequence on the same device."""
    KT = K.geometry.transform
    src, dst = _jittered_quads(64, 1080, 1920, dtype)
    before = K._ops.launch_count
    fused = KT.get_perspective_transform(src, dst)
    assert K._ops.launch_count == before + 1
    K.config.set("torch_prelude", 1)
    plain = KT.get_perspective_transform(src, dst)
    assert K._ops.launch_count == before + 1
    K.config.set("torch_prelude", 0)
    tol = dict(rtol=2e-5, atol=1e-6) if dtype == torch.float32 else dict(rtol=1e-12, atol=1e-13)
    torch.testing.assert_close(fused, plain, **tol)
    torch.testing.assert_close(fused.cpu(), R.perspective_from_points(src.cpu(), dst.cpu()), rtol=1e-4, atol=1e-5)
    print(f"fused perspective {dtype}: {(fused == plain).float().mean().item() * 100:.1f}% of entries bit-identical to the torch ops")
    # gradients flow through the fused forward
    a, b = src.clone().requires_grad_(True), dst.clone().requires_grad_(True)
    cot = torch.rand(64, 3, 3, device=DEV, dtype=dtype)
    ga, gb = torch.autograd.grad((KT.get_perspective_transform(a, b) * cot).sum(), [a, b])
    K.config.set("torch_prelude", 1)
    a2, b2 = src.clone().requires_grad_(True), dst.clone().requires_grad_(True)
    ga2, gb2 = torch.autograd.grad((KT.get_perspective_transform(a2, b2) * cot).sum(), [a2, b2])
    assert rel_l2(ga, ga2) < 1e-5 and rel_l2(gb, gb2) < 1e-5


def test_points_to_warp_pipeline_matches_oracle():
    """The RandomPerspective data path: corner points -> homography -> warp, against the oracle's composition."""
    src, dst = _jittered_quads(4, 270, 480, torch.float32)
    img = torch.nn.functional.interpolate(torch.rand(4, 3, 9, 16, device=DEV), size=(270, 480), mode="bicubic", align_corners=True)
    got = K.warp_perspective(img, K.geometry.transform.get_perspective_transform(src, dst), (270, 480), align_corners=False)
    want = R.warp_perspective(img, R.perspective_from_points(src, dst), (270, 480), align_corners=False)
    torch.testing.assert_close(got, want, **FP32)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_fused_rotation_matrix_matches_torch_ops(dtype, monkeypatch):
    """One-launch get_rotation_matrix2d vs the reference's torch op sequence on the same device, and through rotate()."""
    KT = K.geometry.transform
    g = torch.Generator().manual_seed(11)
    center = (torch.rand(64, 2, generator=g) * 1000).to(DEV, dtype)
    angle = ((torch.rand(64, generator=g) - 0.5) * 720).to(DEV, dtype)
    scale = (0.5 + torch.rand(64, 2, generator=g)).to(DEV, dtype)
    before = K._ops.launch_count
    fused = KT.get_rotation_matrix2d(center, angle, scale)
    assert K._ops.launch_count == before + 1 and fused.shape == (64, 2, 3)
    K.config.set("torch_prelude", 1)
    plain = KT.get_rotation_matrix2d(center, angle, scale)
    assert K._ops.launch_count == before + 1
    K.config.set("torch_prelude", 0)
    tol = dict(rtol=1e-5, atol=2e-4) if dtype == torch.float32 else dict(rtol=1e-12, atol=1e-10)  # translations reach ~1e3
    torch.testing.assert_close(fused, plain, **tol)
    torch.testing.assert_close(fused.cpu(), R.rotation_matrix2d(center.cpu(), angle.cpu(), scale.cpu()), rtol=1e-4, atol=1e-3)
    print(f"fused rotation matrix {dtype}: {(fused == plain).float().mean().item() * 100:.1f}% of entries bit-identical to the torch ops")
    # a center that requires grad keeps the differentiable torch path
    leaf = center.clone().requires_grad_(True)
    KT.get_rotation_matrix2d(leaf, angle, scale).sum().backward()
    assert leaf.grad is not None and K._ops.launch_count == before + 1
    img = torch.rand(8, 3, 96, 128, device=DEV, dtype=dtype)
    ang8 = angle[:8]
    fused_img = KT.rotate(img, ang8)
    K.config.set("torch_prelude", 1)
    torch.testing.assert_close(fused_img, KT.rotate(img, ang8), rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("ks,border", [(3, "reflect"), (5, "replicate"), (7, "constant"), (11, "reflect")])
def test_fused_unsharp_equals_blur_then_lerp(ks, border):
    """unsharp_mask in the blur kernel's epilogue vs blur + torch.lerp (the reference's two steps) on the same device."""
    x = torch.rand(3, 3, 131, 260, device=DEV)
    before = K._ops.launch_count
    fused = K.filters.unsharp_mask(x, (ks, ks), (1.3, 1.7), border)
    assert K._ops.launch_count == before + 1, "one kernel"
    two_step = torch.lerp(K.filters.gaussian_blur2d(x, (ks, ks), (1.3, 1.7), border), x, weight=2.0)
    torch.testing.assert_close(fused, two_step, rtol=1e-6, atol=1e-6)
    print(f"unsharp k={ks}: {(fused == two_step).float().mean().item() * 100:.2f}% bit-identical to blur + torch.lerp")
    torch.testing.assert_close(fused, R.unsharp_mask(x, (ks, ks), (1.3, 1.7), border), **FP32)
    from test_nonfinite_gpu import classes_equal, diff, special_image

    xs = special_image(*x.shape, seed=ks)   # NaN / Inf / -0 / subnormal texels: the same classes, the same tolerance
    fused = K.filters.unsharp_mask(xs, (ks, ks), (1.3, 1.7), border)
    two_step = torch.lerp(K.filters.gaussian_blur2d(xs, (ks, ks), (1.3, 1.7), border), xs, weight=2.0)
    assert classes_equal(fused, two_step, rtol=1e-6, atol=1e-6), diff(fused, two_step)
    # outside the fused envelope (non-square kernel, gradient needed): the composition
    torch.testing.assert_close(K.filters.unsharp_mask(x, (3, 5), (1.0, 1.0)), R.unsharp_mask(x, (3, 5), (1.0, 1.0)), **FP32)
    leaf = x.clone().requires_grad_(True)
    K.filters.unsharp_mask(leaf, (ks, ks), (1.3, 1.7), border).sum().backward()
    assert leaf.grad is not None


def test_install_on_a_package_with_the_references_layout(tmp_path, monkeypatch):
    """install() on the GPU box, where the reference itself cannot be imported: a throw-away package with Kornia's module layout
    (defining modules, re-export sites, a caller that did ``from ..geometry.transform import warp_perspective`` and one that
    captured the function at import) is rebound, its callers then run on the CUDA kernels, uninstall() restores it."""
    import importlib
    import sys
    import textwrap

    root = tmp_path / "fakekornia"
    files = {
        "__init__.py": "from . import geometry, filters, metrics, augmentation\n",
        "geometry/__init__.py": "from .transform import *\n",
        "geometry/transform/__init__.py": "from .imgwarp import *\n",
        "geometry/transform/imgwarp.py": """
            __all__ = ["warp_perspective", "warp_affine", "remap", "get_perspective_transform"]
            def warp_perspective(*a, **k): raise AssertionError("the original warp_perspective ran")
            def warp_affine(*a, **k): raise AssertionError("the original warp_affine ran")
            def remap(*a, **k): raise AssertionError("the original remap ran")
            def get_perspective_transform(*a, **k): raise AssertionError("the original get_perspective_transform ran")
            """,
        "filters/__init__.py": "from .filter import filter2d, filter2d_separable\nfrom .gaussian import gaussian_blur2d\nfrom .sobel import spatial_gradient, sobel\n",
        "filters/filter.py": "def filter2d(*a, **k): raise AssertionError('original')\ndef filter2d_separable(*a, **k): raise AssertionError('original')\n",
        "filters/gaussian.py": "def gaussian_blur2d(*a, **k): raise AssertionError('original')\n",
        "filters/sobel.py": "def spatial_gradient(*a, **k): raise AssertionError('original')\ndef sobel(*a, **k): raise AssertionError('original')\n",
        "metrics/__init__.py": "from .ssim import ssim\n",
        "metrics/ssim.py": "def ssim(*a, **k): raise AssertionError('original')\n",
        "augmentation/__init__.py": """
            from ..geometry.transform import get_perspective_transform, warp_perspective
            from ..filters import gaussian_blur2d
            def random_perspective(x, src, dst):
                return warp_perspective(x, get_perspective_transform(src, dst), tuple(x.shape[-2:]))
            def blur(x):
                return gaussian_blur2d(x, (5, 5), (1.0, 1.0))
            """,
    }
    for rel, text in files.items():
        path = root / rel
        path.parent.mkdir(parents=True, exist_ok=True)
        path.write_text(textwrap.dedent(text))
    monkeypatch.syspath_prepend(str(tmp_path))
    fake = importlib.import_module("fakekornia")
    try:
        x = torch.rand(4, 3, 64, 96, device=DEV)
        quad = torch.tensor([[0.0, 0], [95, 0], [95, 63], [0, 63]], device=DEV)[None].repeat(4, 1, 1)
        dst = quad + torch.randn(4, 4, 2, device=DEV)
        with pytest.raises(AssertionError):
            fake.augmentation.random_perspective(x, quad, dst)
        K.install(fake)
        before = K._ops.launch_count
        out = fake.augmentation.random_perspective(x, quad, dst)
        blurred = fake.augmentation.blur(x)
        assert K._ops.launch_count >= before + 3 and out.shape == x.shape and blurred.shape == x.shape
        assert torch.equal(out, K.warp_perspective(x, K.geometry.transform.get_perspective_transform(quad, dst), (64, 96)))
        assert fake.geometry.warp_affine is K.warp_affine and fake.filters.filter2d is K.filter2d and fake.metrics.ssim is K.metrics.ssim
        K.uninstall()
        with pytest.raises(AssertionError):
            fake.augmentation.blur(x)
    finally:
        K.uninstall()
        for name in [n for n in sys.modules if n == "fakekornia" or n.startswith("fakekornia.")]:
            del sys.modules[name]
