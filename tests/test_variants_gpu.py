"""Kernel variants against the kernels they stand in for (kornia_b200.config switches).  The ones that measured faster are the
defaults.  Each test flips a switch, runs both kernels on the same inputs and compares bit for bit
where the arithmetic is the same, and checks the golden vectors recorded from the reference."""
import pytest
import torch

import kornia_b200 as K
from conftest import golden

pytestmark = [pytest.mark.gpu]
DEV = "cuda"


# ------------------------------------------------------------------------------------------ fused pyrdown
@pytest.mark.parametrize("border", ["reflect", "replicate", "constant"])
@pytest.mark.parametrize("shape", [(2, 3, 64, 128), (1, 2, 70, 132), (3, 1, 34, 260), (1, 3, 4, 4), (1, 1, 1080, 1920)])
def test_fused_pyrdown_equals_composition(border, shape):
    """kb200_pyrdown_forward == filter2d (tiled 5x5) + F.interpolate(bilinear, align_corners=False), bit for bit (-0 != +0), on
    a random image and on one with NaN / Inf / -0 / subnormal texels at the tile seams.  Documented exception: no 3e38 texels --
    the fused epilogue adds the four filtered taps before it scales them by 1/4, the composition scales each by 1/2 twice, so
    four values near FLT_MAX overflow to Inf in the first and not in the second."""
    from test_nonfinite_gpu import bits_equal, special_image

    KT = K.geometry.transform
    for x in (torch.rand(*shape, device=DEV), special_image(*shape, seed=1, huge=False)):
        K.config.set("fused_pyrdown", 0)
        want = KT.pyrdown(x, border)
        before = K._ops.launch_count
        K.config.set("fused_pyrdown", 1)
        got = KT.pyrdown(x, border)
        assert K._ops.launch_count == before + 1, "the fused kernel did not run"
        assert got.shape == want.shape and got.is_contiguous()
        assert bits_equal(got, want), float((got - want).abs().nan_to_num().max())


def test_fused_pyrdown_golden_and_fallbacks():
    K.config.set("fused_pyrdown", 1)
    KT = K.geometry.transform
    WID = golden("wider")
    for name in WID.names("pyrdown") + WID.names("build_pyramid"):
        op, kw, ins, outs = WID.case(name)
        kw = {k: (tuple(v) if isinstance(v, list) else v) for k, v in kw.items()}
        got = getattr(KT, op)(ins["input"].to(DEV), **kw)
        got = got if isinstance(got, list) else [got]
        for i, g in enumerate(got):
            torch.testing.assert_close(g.cpu(), outs["out" if "out" in outs else f"out{i}"], rtol=1e-4, atol=1e-5)
    # outside the envelope (odd size, align_corners, factor, grad) the composition runs: same numbers as with the switch off
    x = torch.rand(1, 2, 17, 23, device=DEV)
    a = KT.pyrdown(x)
    K.config.set("fused_pyrdown", 0)
    assert torch.equal(a, KT.pyrdown(x))
    K.config.set("fused_pyrdown", 1)
    xg = torch.rand(1, 1, 16, 16, device=DEV, requires_grad=True)
    KT.pyrdown(xg).sum().backward()
    assert xg.grad is not None and xg.grad.shape == xg.shape


# ------------------------------------------------------------------------------------------ tiled derivatives
@pytest.mark.parametrize("shape", [(2, 3, 64, 128), (1, 2, 70, 132), (3, 1, 33, 260), (1, 1, 3, 4), (1, 3, 1080, 1920)])
@pytest.mark.parametrize("mode,order", [("sobel", 1), ("diff", 1), ("sobel", 2), ("diff", 2)])
@pytest.mark.parametrize("normalized", [True, False])
def test_tiled_spatial_gradient_bit_identical(shape, mode, order, normalized):
    """grad_tiled_kernel (KB200_TILED_GRADIENT=1) == spatial_gradient_fwd, bit for bit (same taps, same FMA order; -0 != +0), on a
    random image and on one with NaN / Inf / -0 / subnormal texels at the tile seams."""
    from test_nonfinite_gpu import bits_equal, special_image

    for x in (torch.rand(*shape, device=DEV), special_image(*shape, seed=2)):
        K.config.set("tiled_gradient", 0)
        want = K.filters.spatial_gradient(x, mode, order, normalized)
        K.config.set("tiled_gradient", 1)
        got = K.filters.spatial_gradient(x, mode, order, normalized)
        assert got.shape == want.shape and bits_equal(got, want), float((got - want).abs().nan_to_num().max())


@pytest.mark.parametrize("shape", [(2, 3, 64, 128), (1, 2, 70, 132), (1, 3, 1080, 1920)])
def test_tiled_sobel_bit_identical_and_golden(shape):
    x = torch.rand(*shape, device=DEV)
    K.config.set("tiled_gradient", 0)
    want = K.filters.sobel(x)
    K.config.set("tiled_gradient", 1)
    got = K.filters.sobel(x)
    assert torch.equal(got, want), float((got - want).abs().max())
    FAM = golden("family")
    for name in FAM.names("sobel") + FAM.names("spatial_gradient"):
        op, kw, ins, outs = FAM.case(name)
        res = getattr(K.filters, op)(ins["input"].to(DEV), **kw)
        torch.testing.assert_close(res.cpu(), outs["out"], rtol=1e-4, atol=1e-5)


# ------------------------------------------------------------------------------------------ band-walking SSIM
@pytest.mark.parametrize("window,shape", [(w, s) for w in (3, 5, 7, 9, 11)
                                          for s in ((2, 3, 70, 132), (1, 1, 32, 64), (3, 2, 33, 8), (1, 2, 97, 260), (1, 1, 6, 8), (1, 3, 1080, 1920))
                                          if min(s[-2:]) > w // 2])  # a reflect fold needs an image larger than the half-window
def test_band_walk_ssim_bit_identical(window, shape):
    """ssim_vwalk_kernel == the library's own differentiable composition (five one-pass blurs + torch elementwise ops, the path
    taken when a gradient is needed), bit for bit (-0 != +0); also with NaN / Inf / -0 / subnormal texels at the tile seams."""
    from test_nonfinite_gpu import bits_equal, special_image

    a = torch.rand(*shape, device=DEV)
    b = (a + 0.1 * torch.randn(*shape, device=DEV)).clamp(0, 1)
    for a, b in ((a, b), (special_image(*shape, seed=3), b)):
        want = K.metrics.ssim(a.clone().requires_grad_(True), b, window).detach()
        before = K._ops.launch_count
        got = K.metrics.ssim(a, b, window)
        assert K._ops.launch_count == before + 1, "the fused kernel did not run"
        assert bits_equal(got, want), float((got - want).abs().nan_to_num().max())


def test_band_walk_ssim_many_segments_and_golden():
    a = torch.rand(40, 3, 200, 260, device=DEV)   # 120 planes x 5 bands = 600 bands > the persistent grid (2 CTAs per SM): segments start inside bands
    b = a.flip(-1).contiguous()
    got = K.metrics.ssim(a, b, 11)
    assert torch.equal(got, K.metrics.ssim(a.clone().requires_grad_(True), b, 11).detach())
    SS = golden("ssim")
    for name in SS.names("ssim"):
        op, kw, ins, outs = SS.case(name)
        res = K.metrics.ssim(ins["img1"].to(DEV), ins["img2"].to(DEV), **kw)
        torch.testing.assert_close(res.cpu(), outs["out"], rtol=1e-4, atol=1e-5)


# ------------------------------------------------------------------------------------------ tiled backward kernels
@pytest.mark.parametrize("stride1", [0, 1])
@pytest.mark.parametrize("pad", ["zeros", "border"])
@pytest.mark.parametrize("ac", [True, False])
@pytest.mark.parametrize("C", [3, 1])
def test_tiled_backward_matches_generic(stride1, pad, ac, C):
    """warp_bwd_tma2 (column-pair lanes / conflict-free stride-1 lanes, switch bwd_stride1) against the generic atomics kernel:
    same per-pixel arithmetic; d/dsrc differs only by the order of the adds, d/dM by the grouping of the partial sums."""
    from test_parity_gpu import _bench_homographies, _generic, _wild_matrices
    from helpers import rel_l2

    H, W = 120, 256
    M = torch.cat([_wild_matrices(H, W), _bench_homographies(6, H, W, 9, sigma=3.0)]).to(DEV)
    B = M.shape[0]
    g = torch.Generator().manual_seed(C)
    src = torch.rand(B, C, H, W, generator=g).to(DEV)
    for dsize in ((H, W), (96, 200), (33, 66)):
        cot = (torch.rand(B, C, *dsize, generator=g) - 0.5).to(DEV)

        def grads(kind, want=(True, True)):
            s = src.clone().requires_grad_(want[0])
            if kind == "persp":
                mm = M.clone().requires_grad_(want[1])
                out = K.warp_perspective(s, mm, dsize, padding_mode=pad, align_corners=ac)
            else:
                mm = M[:, :2].clone().requires_grad_(want[1])
                out = K.warp_affine(s, mm, dsize, padding_mode=pad, align_corners=ac)
            return torch.autograd.grad(out, [t for t, w in zip((s, mm), want) if w], grad_outputs=cot)

        for kind in ("persp", "affine"):
            gs0, gm0 = _generic(lambda: grads(kind), check_variant=False)
            K.config.set("bwd_stride1", stride1)
            gs2, gm2 = grads(kind)
            (gs_only,) = grads(kind, (True, False))
            (gm_only,) = grads(kind, (False, True))
            for ref in (gs0,):
                assert rel_l2(gs2, ref) < 2e-6, (kind, dsize, rel_l2(gs2, ref))
                torch.testing.assert_close(gs2, ref, rtol=1e-4, atol=2e-5)
            assert rel_l2(gs_only, gs2) < 2e-6
            for b in range(B):
                if not torch.isfinite(gm0[b]).all():
                    continue
                assert rel_l2(gm2[b], gm0[b]) < 1e-4, (kind, dsize, b, rel_l2(gm2[b], gm0[b]))
                assert rel_l2(gm_only[b], gm2[b]) < 1e-5


def test_backward_work_drawn_at_run_time_matches_the_static_deal():
    """warp_bwd_tma2<DYN> (every warp draws its next 4-row slice of a chunk of tiles from a counter; switch dyn_sched) against the
    static deal at a shape with enough strips for the dispatcher to take it: d/dsrc up to the order of the reduce-adds, d/dM up to
    the grouping of the partial sums; and each gradient alone."""
    from helpers import rel_l2
    from test_parity_gpu import _bench_homographies

    B, H, W = 400, 96, 192   # 1 200 strips of three tiles
    g = torch.Generator().manual_seed(2)
    src = torch.rand(B, 3, H, W, generator=g).to(DEV)
    M = _bench_homographies(B, H, W, 11, sigma=2.0).to(DEV)
    cot = (torch.rand(B, 3, H, W, generator=g) - 0.5).to(DEV)

    def grads(want=(True, True)):
        s, mm = src.clone().requires_grad_(want[0]), M.clone().requires_grad_(want[1])
        out = K.warp_perspective(s, mm, (H, W))
        return torch.autograd.grad(out, [t for t, w in zip((s, mm), want) if w], grad_outputs=cot)

    with K.config.override(dyn_sched=0):
        gs0, gm0 = grads()
    with K.config.override(dyn_sched=1):
        gs1, gm1 = grads()
        (gs_only,) = grads((True, False))
        (gm_only,) = grads((False, True))
        gs2, gm2 = grads()
    assert rel_l2(gs1, gs0) < 2e-6 and rel_l2(gs_only, gs0) < 2e-6
    torch.testing.assert_close(gs1, gs0, rtol=1e-4, atol=2e-5)
    for b in range(B):
        assert rel_l2(gm1[b], gm0[b]) < 1e-4, (b, rel_l2(gm1[b], gm0[b]))
    assert torch.equal(gm1, gm2) and torch.equal(gm_only, gm1)   # the record rows are summed in a fixed order: run-to-run identical


@pytest.mark.parametrize("stride1", [0, 1])
def test_tiled_backward_720p_and_goldens(stride1):
    """cfg4's shape at reduced batch against the reference's autograd on CPU, and every golden gradient case."""
    K.config.set("bwd_stride1", stride1)
    from helpers import rel_l2, run_case
    from oracle import kornia_restated as R
    from test_parity_gpu import _bench_homographies

    H, W, B = 720, 1280, 2
    M = _bench_homographies(B, H, W, 7).to(DEV)
    yy, xx = torch.linspace(0, 1, H)[:, None], torch.linspace(0, 1, W)[None, :]
    smooth = torch.stack([torch.stack([0.5 + 0.25 * torch.sin(6.2831853 * ((c + 1) * xx + (b + 2) * yy)) +
                                       0.2 * torch.cos(6.2831853 * (5 * xx - 3 * yy + 0.1 * c)) for c in range(3)]) for b in range(B)])
    target = smooth.flip(-1) * 0.5 + 0.25

    def run(mod, s, m, t):
        s, m = s.clone().requires_grad_(True), m.clone().requires_grad_(True)
        return torch.autograd.grad(((mod.warp_perspective(s, m, (H, W)) - t) ** 2).mean(), [s, m])

    gs, gm = run(K, smooth.to(DEV), M, target.to(DEV))
    gs_ref, gm_ref = run(R, smooth, M.cpu(), target)
    assert rel_l2(gs.cpu(), gs_ref) < 1e-4 and rel_l2(gm.cpu(), gm_ref) < 1e-3, (rel_l2(gs.cpu(), gs_ref), rel_l2(gm.cpu(), gm_ref))
    WARP = golden("warp")
    for op in ("warp_perspective_grad", "warp_affine_grad"):
        for name in WARP.names(op):
            _, kw, ins, outs = WARP.case(name)
            got = run_case(K, op, kw, ins, device=DEV)
            for key, want in outs.items():
                if key != "cot":
                    assert rel_l2(got[key].cpu(), want) < 1e-4, (name, key)


# ------------------------------------------------------------------------------------------ fused undistort_image
@pytest.mark.parametrize("ncoef", [4, 5, 8, 12, 14])
@pytest.mark.parametrize("shape", [(2, 3, 64, 128), (1, 1, 70, 132), (3, 3, 270, 480), (1, 3, 1080, 1920)])
def test_fused_undistort_equals_composition(ncoef, shape):
    """kb200_undistort_forward (lens model in registers) == distort_points (torch ops) + remap, bit for bit: the kernel
    evaluates the reference's op sequence with one rounding per op on the exact integer grid.  The second image has NaN / Inf /
    -0 / subnormal texels at the tile seams; the comparison is bit for bit with -0 != +0."""
    from test_nonfinite_gpu import bits_equal, special_image

    KC = K.geometry.calibration
    B, C, H, W = shape
    g = torch.Generator().manual_seed(ncoef)
    img = torch.rand(*shape, generator=g).to(DEV)
    cam = torch.tensor([[0.8 * W, 0.0, 0.5 * W - 3.0], [0.0, 0.75 * W, 0.5 * H + 2.0], [0.0, 0.0, 1.0]]).expand(B, 3, 3).clone()
    cam[:, 0, 0] += torch.arange(B) * 7.0
    scale = torch.tensor([0.25, 0.08, 0.003, 0.003, 0.02, 0.05, 0.02, 0.004, 0.003, 0.001, 0.002, 0.0015, 0.0, 0.0])[:ncoef]
    dist = (torch.rand(B, ncoef, generator=g) - 0.5) * 2 * scale   # tilt terms zero: the fused envelope
    cam, dist = cam.to(DEV), dist.to(DEV)
    for img in (img, special_image(*shape, seed=ncoef)):
        K.config.set("fused_undistort", 0)
        want = KC.undistort_image(img, cam, dist)
        before = K._ops.launch_count
        K.config.set("fused_undistort", 1)
        got = KC.undistort_image(img, cam, dist)
        assert K._ops.launch_count == before + 1, "the fused kernel did not run"
        assert bits_equal(got, want), float((got - want).abs().nan_to_num().max())


def test_fused_undistort_golden_and_fallbacks():
    K.config.set("fused_undistort", 1)
    KC = K.geometry.calibration
    WID = golden("wider")
    for name in WID.names("undistort_image"):   # includes unbatched K, (C,H,W) and 5-D inputs, and the tilted 14-coefficient case
        op, kw, ins, outs = WID.case(name)
        got = KC.undistort_image(**{k: v.to(DEV) for k, v in ins.items()})
        torch.testing.assert_close(got.cpu(), outs["out"], rtol=1e-4, atol=1e-5)
    img = torch.rand(1, 3, 32, 64, device=DEV, requires_grad=True)
    cam = torch.tensor([[[50.0, 0, 32], [0, 50.0, 16], [0, 0, 1]]], device=DEV)
    KC.undistort_image(img, cam, torch.tensor([[0.1, 0.0, 0.0, 0.0]], device=DEV)).sum().backward()   # grad: composition
    assert img.grad is not None


# ------------------------------------------------------------------------------------------ fused undistort at full size
def test_fused_undistort_full_size():
    img = torch.rand(2, 3, 1080, 1920, device=DEV)
    cam = torch.tensor([[1500.0, 0.0, 960.0], [0.0, 1500.0, 540.0], [0.0, 0.0, 1.0]], device=DEV).expand(2, 3, 3).contiguous()
    dist = torch.tensor([[-0.2, 0.05, 0.001, -0.002, 0.01]], device=DEV).expand(2, 5).contiguous()
    KC = K.geometry.calibration
    before = K._ops.launch_count
    b = KC.undistort_image(img, cam, dist)                 # lens model inside the sampling kernel
    assert K._ops.launch_count == before + 1
    K.config.set("fused_undistort", 0)
    c = KC.undistort_image(img, cam, dist)                 # maps (torch) + the tiled remap
    assert torch.equal(b, c)


# ------------------------------------------------------------------------------------------ fast filter backward
@pytest.mark.parametrize("border", ["reflect", "replicate", "constant"])
@pytest.mark.parametrize("ksize", [3, 11])
@pytest.mark.parametrize("shape", [(2, 3, 70, 132), (1, 1, 20, 36), (1, 3, 360, 640)])
def test_fast_filter_backward_matches_composition(border, ksize, shape):
    """switch fast_filter_bwd: d/dinput of gaussian_blur2d through the forward kernel with flipped taps + exact border bands,
    against the autograd composition (four generic passes) -- different summation order, fp32 rounding apart."""
    from helpers import rel_l2

    x = torch.rand(*shape, device=DEV)
    cot = torch.rand(*shape, device=DEV) - 0.5

    def grad():
        xx = x.clone().requires_grad_(True)
        (g,) = torch.autograd.grad(K.gaussian_blur2d(xx, (ksize, ksize), (1.7, 1.7), border), [xx], cot)
        return g

    K.config.set("fast_filter_bwd", 0)
    want = grad()
    K.config.set("fast_filter_bwd", 1)
    got = grad()
    assert rel_l2(got, want) < 2e-6, rel_l2(got, want)
    torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-6)


def test_fast_filter_backward_ssim_loss_and_goldens():
    from helpers import family_grads, rel_l2

    K.config.set("fast_filter_bwd", 1)
    SS, FIL = golden("ssim"), golden("filter")
    for name in SS.names("ssim_grad") + SS.names("ssim_loss_grad"):
        op, kw, ins, outs = SS.case(name)
        impl = K.losses if op.startswith("ssim_loss") else K.metrics
        got = family_grads(impl, op, kw, ins, outs, device=DEV)
        for key, want in outs.items():
            if key != "cot":
                assert rel_l2(got[key].cpu(), want) < 1e-4, (name, key)
    from helpers import run_case
    for name in FIL.names("gaussian_blur2d_grad") + FIL.names("filter2d_separable_grad"):
        op, kw, ins, outs = FIL.case(name)
        got = run_case(K, op, kw, ins, device=DEV)
        for key, want in outs.items():
            if key != "cot":
                assert rel_l2(got[key].cpu(), want) < 1e-4, (name, key)


# ------------------------------------------------------------------------------------------ more planes than one launch takes
def test_feature_map_sized_plane_counts():
    """B * C above the 65535-plane limit of one filter launch (ADVICE r1: e.g. B=256, C=256 feature maps): served by several
    launches over batch slices, per-sample kernels keep cycling, the kernel gradient folds the slices."""
    from oracle import kornia_restated as R

    B, C, H, W = 300, 256, 8, 12
    x = torch.rand(B, C, H, W, device=DEV)
    k1 = torch.randn(1, 3, 3, device=DEV)
    kb = torch.randn(B, 3, 3, device=DEV)
    for kern in (k1, kb):
        got = K.filter2d(x, kern)
        want = torch.cat([R.filter2d(x[i:i + 50], kern if kern.shape[0] == 1 else kern[i:i + 50]) for i in range(0, B, 50)])
        torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-5)
    kx, ky = torch.randn(1, 5, device=DEV), torch.randn(B, 5, device=DEV)
    got = K.filter2d_separable(x, kx, ky)
    want = torch.cat([R.filter2d_separable(x[i:i + 50], kx, ky[i:i + 50]) for i in range(0, B, 50)])
    torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-5)
    xs = x[:, :, :6, :8].contiguous().requires_grad_(True)
    kg = torch.randn(2, 3, 3, device=DEV, requires_grad=True)   # two kernels cycling over 300 samples
    gx, gk = torch.autograd.grad(K.filter2d(xs, kg).square().sum(), [xs, kg])
    xr, kr = xs.detach().clone().requires_grad_(True), kg.detach().clone().requires_grad_(True)
    gx_r, gk_r = torch.autograd.grad(R.filter2d(xr, kr).square().sum(), [xr, kr])
    torch.testing.assert_close(gx, gx_r, rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(gk, gk_r, rtol=1e-3, atol=1e-2)
