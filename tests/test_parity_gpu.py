"""Parity of the CUDA path (through the C ABI) against the golden vectors recorded from the
reference and against the CPU oracle.  Tolerances: the reference's own fp32 test tolerance
(testing/base.py:34-40: rtol 1e-4, atol 1e-5) element-wise on the small cases; 1e-4 norm-relative
(BASELINE.json north_star) on gradients, whose entries span several orders of magnitude."""
import pytest
import torch

import kornia_b200 as K
from conftest import golden
from helpers import rel_l2, run_case
from oracle import kornia_restated as R

pytestmark = pytest.mark.gpu
WARP = golden("warp")
FILT = golden("filter")
FP32 = dict(rtol=1e-4, atol=1e-5)
DEV = "cuda"


def _close_or_tieflip(got, want, frac=0.01):
    """'nearest' picks a different tap when fp32 rounding puts a coordinate on the other side of .5;
    the reference itself flips such taps between CPU and CUDA.  Require all but a handful equal."""
    bad = (got - want).abs() > (1e-5 + 1e-4 * want.abs())
    assert bad.float().mean().item() <= frac, f"{bad.sum().item()} / {bad.numel()} mismatches"


FWD_WARP = WARP.names("warp_perspective") + WARP.names("warp_affine") + WARP.names("remap")


@pytest.mark.parametrize("name", FWD_WARP)
def test_warp_forward_matches_reference(name):
    op, kw, ins, outs = WARP.case(name)
    got = run_case(K, op, kw, ins, device=DEV).cpu()
    assert got.is_contiguous() and got.dtype == outs["out"].dtype
    if kw["mode"] == "nearest":
        _close_or_tieflip(got, outs["out"])
    else:
        torch.testing.assert_close(got, outs["out"], **FP32)


@pytest.mark.parametrize("name", FWD_WARP[::2])
def test_warp_forward_fp64_matches_oracle(name):
    """Same op in float64: CUDA kernel vs the oracle run in float64 on the SAME device (tight: the
    reference builds its base grid in fp32 even for fp64 input, imgwarp.py:157, and torch's CUDA and CPU
    fp32 divisions differ by an ulp there, so CPU-vs-CUDA agreement is only fp32-grade -- measured
    1.5e-6 -- for the reference itself) and on the CPU (fp32-grade)."""
    op, kw, ins, _ = WARP.case(name)
    got = run_case(K, op, kw, ins, device=DEV, dtype=torch.float64)
    was = torch.backends.cudnn.enabled
    torch.backends.cudnn.enabled = False
    try:
        same_dev = run_case(R, op, kw, ins, device=DEV, dtype=torch.float64)
    finally:
        torch.backends.cudnn.enabled = was
    want = run_case(R, op, kw, ins, dtype=torch.float64)
    if kw["mode"] == "nearest":
        _close_or_tieflip(got, same_dev, frac=0.002)
        _close_or_tieflip(got.cpu(), want, frac=0.01)
    else:
        torch.testing.assert_close(got, same_dev, rtol=1e-12, atol=1e-13)
        torch.testing.assert_close(got.cpu(), want, rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("name", FWD_WARP)
def test_warp_forward_fp32_equals_the_same_device_reference(name):
    """fp32, every golden case (3 interpolations x 4 paddings x both align_corners, remap included) against the reference
    composition on the SAME GPU with cuDNN off: the coordinate chain is replicated op for op, so there is no tie to flip and
    no tolerance to grant -- nearest included.  (The tolerance of the CPU-golden tests above is the reference's own CPU-vs-CUDA
    gap, not this library's.)"""
    op, kw, ins, _ = WARP.case(name)
    got = run_case(K, op, kw, ins, device=DEV)
    with torch.backends.cudnn.flags(enabled=False):
        want = run_case(R, op, kw, ins, device=DEV)
    if kw["mode"] == "bicubic":  # ATen's bicubic kernel contracts its weight polynomials with FMAs of its own choosing
        torch.testing.assert_close(got, want, rtol=1e-5, atol=2e-6)
    else:
        assert torch.equal(got, want), float((got - want).abs().max())


GRAD_WARP = [n for op in ("warp_perspective_grad", "warp_affine_grad", "remap_grad") for n in WARP.names(op)]


@pytest.mark.parametrize("name", GRAD_WARP)
def test_warp_grads_match_reference(name):
    op, kw, ins, outs = WARP.case(name)
    got = run_case(K, op, kw, ins, device=DEV)
    for key, want in outs.items():
        g = got[key].cpu()
        if kw["mode"] == "nearest":
            if key.startswith("grad_M") or key.startswith("grad_map"):
                assert float(g.abs().max()) == 0.0  # nearest has no coordinate gradient
            else:
                _close_or_tieflip(g, want, frac=0.02)
            continue
        assert rel_l2(g, want) < 1e-4, (key, rel_l2(g, want))


@pytest.mark.parametrize("name", [n for n in GRAD_WARP[::3] if WARP.case(n)[1]["mode"] != "nearest"])  # nearest has no coordinate gradient
def test_warp_grads_fp64_match_oracle(name):
    op, kw, ins, _ = WARP.case(name)
    got = run_case(K, op, kw, ins, device=DEV, dtype=torch.float64)
    want = run_case(R, op, kw, ins, device=DEV, dtype=torch.float64)  # same device: same fp32 base grid
    for key in want:
        assert rel_l2(got[key], want[key]) < 1e-9, (key, rel_l2(got[key], want[key]))


FWD_FILT = FILT.names("filter2d") + FILT.names("filter2d_separable") + FILT.names("gaussian_blur2d")


@pytest.mark.parametrize("name", FWD_FILT)
def test_filter_forward_matches_reference(name):
    op, kw, ins, outs = FILT.case(name)
    got = run_case(K, op, kw, ins, device=DEV).cpu()
    assert got.is_contiguous()
    torch.testing.assert_close(got, outs["out"], **FP32)


GRAD_FILT = [n for op in ("filter2d_grad", "filter2d_separable_grad", "gaussian_blur2d_grad") for n in FILT.names(op)]


@pytest.mark.parametrize("name", GRAD_FILT)
def test_filter_grads_match_reference(name):
    op, kw, ins, outs = FILT.case(name)
    got = run_case(K, op, kw, ins, device=DEV)
    for key, want in outs.items():
        assert rel_l2(got[key].cpu(), want) < 1e-4, (key, rel_l2(got[key].cpu(), want))


@pytest.mark.parametrize("name", FWD_FILT[::5] + GRAD_FILT[::4])
def test_filter_fp64_matches_oracle(name):
    op, kw, ins, _ = FILT.case(name)
    got = run_case(K, op, kw, ins, device=DEV, dtype=torch.float64)
    want = run_case(R, op, kw, ins, dtype=torch.float64)
    if isinstance(want, dict):
        for key in want:
            assert rel_l2(got[key].cpu(), want[key]) < 1e-9, key
    else:
        torch.testing.assert_close(got.cpu(), want, rtol=1e-9, atol=1e-10)  # host fp64 BLAS varies at the 1e-11 level from box to box


# ------------------------------------------------------------------ gradcheck (reference: testing/base.py:158-206)
def _gradcheck(fn, inputs, **kw):
    # d/dsrc scatters with atomics: summation order (not value) varies run to run
    assert torch.autograd.gradcheck(fn, inputs, raise_exception=True, fast_mode=True, nondet_tol=1e-9, **kw)


def test_gradcheck_warp_affine():
    # tests/geometry/transform/test_imgwarp.py:295-299
    aff = torch.eye(2, 3, device=DEV, dtype=torch.float64)[None] + 1e-6
    img = torch.rand(1, 2, 3, 4, device=DEV, dtype=torch.float64)
    _gradcheck(lambda a, b: K.warp_affine(a, b, (3, 4)), (img.requires_grad_(), aff.requires_grad_()))


@pytest.mark.parametrize("mode", ["bilinear", "bicubic"])
@pytest.mark.parametrize("pad", ["zeros", "border", "reflection", "fill"])
def test_gradcheck_warp_perspective(mode, pad):
    g = torch.Generator().manual_seed(3)
    img = torch.rand(2, 3, 6, 7, generator=g, dtype=torch.float64).to(DEV).requires_grad_()
    M = (torch.eye(3, dtype=torch.float64)[None].repeat(2, 1, 1) + 0.03 * torch.randn(2, 3, 3, generator=g, dtype=torch.float64))
    M[:, 2, :2] *= 0.05
    M = M.to(DEV).requires_grad_()
    fv = torch.tensor([0.2, 0.4, 0.6], dtype=torch.float64, device=DEV)
    _gradcheck(lambda a, b: K.warp_perspective(a, b, (5, 6), mode=mode, padding_mode=pad, align_corners=False, fill_value=fv), (img, M))


def test_gradcheck_remap():
    g = torch.Generator().manual_seed(5)
    img = torch.rand(1, 2, 5, 6, generator=g, dtype=torch.float64).to(DEV).requires_grad_()
    mx = (torch.rand(1, 4, 5, generator=g, dtype=torch.float64) * 5).to(DEV).requires_grad_()
    my = (torch.rand(1, 4, 5, generator=g, dtype=torch.float64) * 4).to(DEV).requires_grad_()
    _gradcheck(lambda a, b, c: K.remap(a, b, c, align_corners=True), (img, mx, my))


def test_gradcheck_filter2d_and_gaussian():
    # tests/filters/test_filters.py:379-384, tests/filters/test_gaussian.py:266-274
    x = torch.rand(2, 3, 5, 6, device=DEV, dtype=torch.float64, requires_grad=True)
    k = torch.rand(1, 3, 3, device=DEV, dtype=torch.float64, requires_grad=True)
    _gradcheck(lambda a, b: K.filter2d(a, b), (x, k))
    _gradcheck(lambda a: K.gaussian_blur2d(a, (3, 5), (1.3, 0.8), "replicate"), (x,))
    sig = torch.tensor([[1.1, 0.7]], device=DEV, dtype=torch.float64, requires_grad=True)
    _gradcheck(lambda a, s: K.gaussian_blur2d(a, 3, s), (x, sig))


# ------------------------------------------------------------------ the tiled (TMA) kernel
def _bench_homographies(B, H, W, seed, sigma=8.0):
    import bench

    g = torch.Generator().manual_seed(seed)
    quad = torch.tensor([[0.0, 0.0], [W - 1.0, 0.0], [W - 1.0, H - 1.0], [0.0, H - 1.0]]).expand(B, 4, 2)
    return bench.perspective_from_quads(quad, quad + sigma * torch.randn(B, 4, 2, generator=g))


def _generic(fn, check_variant=True):
    """Run ``fn`` with the tiled kernels disabled (the C ABI then dispatches the generic kernels)."""
    from kornia_b200 import _lib

    with K.config.override(tma=0):
        out = fn()
        if check_variant:  # only kb200_warp_forward records the variant it dispatched to
            assert _lib.last_warp_variant() == "generic"
    return out


def _wild_matrices(H, W):
    """Homographies that stress the tile logic: rotations, zoom in/out, strong perspective,
    a horizon inside the image (denominator changes sign), fully out-of-view, singular-ish."""
    import math

    cx, cy = (W - 1) / 2, (H - 1) / 2
    mats = []
    for deg in (3.0, 30.0, 90.0, 180.0):
        c, s = math.cos(math.radians(deg)), math.sin(math.radians(deg))
        mats.append([[c, -s, cx - c * cx + s * cy], [s, c, cy - s * cx - c * cy], [0, 0, 1]])
    mats.append([[3.0, 0, -2 * cx], [0, 3.0, -2 * cy], [0, 0, 1]])       # zoom in
    mats.append([[0.25, 0, 0.4 * W], [0, 0.25, 0.3 * H], [0, 0, 1]])     # zoom out
    mats.append([[1, 0.2, 5], [0.1, 1, -7], [4e-4, 2e-4, 1]])            # strong perspective
    mats.append([[1, 0, 0], [0, 1, 0], [2.0 / W, 0, -1.0]])              # horizon through the image
    mats.append([[1, 0, 10.0 * W], [0, 1, 0], [0, 0, 1]])                # everything out of view
    mats.append([[1, 0, 0.5], [0, 1, 0.25], [0, 0, 1]])                  # sub-pixel shift
    return torch.tensor(mats, dtype=torch.float32)


def _shift_matrices(W):
    """Tiles wholly outside the image by 20-50 px ('reflection' folds them back as a whole: the box must follow the reflected corners)
    and a shift of more than one span (reflected twice: the exact path)."""
    return torch.tensor([[[0.96, -0.013, 13.1], [-0.016, 0.95, 32.0], [-1.5e-5, -1.1e-5, 1]],
                         [[1, 0, -50.0], [0, 1, -27.0], [0, 0, 1]],
                         [[1, 0, 1.6 * W], [0, 1, 0], [0, 0, 1]]], dtype=torch.float32)


_TILED_CASES = ([("bilinear", pad, C) for pad in ("zeros", "border", "reflection") for C in (1, 3, 4)] +
                [("bilinear", "fill", 3)] +
                [(mode, pad, 3) for mode in ("nearest", "bicubic") for pad in ("zeros", "border", "reflection", "fill")] +
                [("bicubic", "zeros", 1), ("nearest", "border", 1)])


@pytest.mark.parametrize("mode,pad,C", _TILED_CASES)
@pytest.mark.parametrize("ac", [True, False])
def test_tiled_kernel_bit_identical_to_generic(mode, pad, C, ac):
    """Every mode the tiled kernel serves must reproduce the generic kernel exactly, -0 and NaN included (the staged tile is
    only a cache): rotations, zoom, strong perspective, a horizon inside the image, everything out of view; on a random image
    and on one with NaN / Inf / -0 / subnormal texels at the tile seams."""
    from test_nonfinite_gpu import bits_equal, special_image

    H, W = 216, 384
    M = torch.cat([_wild_matrices(H, W), _shift_matrices(W), _bench_homographies(6, H, W, 5, sigma=4.0)]).to(DEV)
    fv = torch.tensor([0.2, 0.5, 0.8], device=DEV) if pad == "fill" else None
    from kornia_b200 import _lib

    same = bits_equal
    for src, dsize in ((torch.rand(M.shape[0], C, H, W, device=DEV), (H, W)), (torch.rand(M.shape[0], C, H, W, device=DEV), (150, 333)),
                       (special_image(M.shape[0], C, H, W, seed=C), (H, W)), (special_image(M.shape[0], C, H, W, seed=C), (150, 333))):
        a = K.warp_perspective(src, M, dsize, mode=mode, padding_mode=pad, align_corners=ac, fill_value=fv)
        assert _lib.last_warp_variant() == "tma_tile"
        b = _generic(lambda: K.warp_perspective(src, M, dsize, mode=mode, padding_mode=pad, align_corners=ac, fill_value=fv))
        assert same(a, b), (dsize, float((a - b).abs().nan_to_num().max()))
        A = M[:, :2, :].contiguous()
        fa = fv if C == 3 or fv is None else fv[:C]
        a = K.warp_affine(src, A, dsize, mode=mode, padding_mode=pad, align_corners=ac, fill_value=fa)
        assert _lib.last_warp_variant() == "tma_tile"
        b = _generic(lambda: K.warp_affine(src, A, dsize, mode=mode, padding_mode=pad, align_corners=ac, fill_value=fa))
        assert same(a, b), ("affine", dsize, float((a - b).abs().nan_to_num().max()))


def test_run_time_work_distribution_is_bit_identical():
    """warp_fwd_tma<DYN> (strips handed out at run time in chunks, switch dyn_sched) against the static deal at a batch large enough
    for the dispatcher to take it (B x ceil(h / 32) >= 8 x the SM count): the same tiles, the same results."""
    B, H, W = 40, 1080, 1920
    src = torch.rand(B, 3, H, W, device=DEV)
    M = torch.cat([_bench_homographies(B - 4, H, W, 3), _wild_matrices(H, W)[:4]]).to(DEV)
    fv = torch.tensor([0.2, 0.5, 0.8], device=DEV)
    for fn in (lambda: K.warp_perspective(src, M, (H, W)), lambda: K.warp_affine(src, M[:, :2].contiguous(), (H, W), align_corners=False),
               lambda: K.warp_perspective(src, M, (H, W), padding_mode="reflection"), lambda: K.warp_perspective(src, M, (H, W), padding_mode="border", align_corners=False),
               lambda: K.warp_affine(src, M[:, :2].contiguous(), (H, W), padding_mode="fill", fill_value=fv)):
        with K.config.override(dyn_sched=0):
            want = fn()
        with K.config.override(dyn_sched=1):
            got = fn()
        assert torch.equal(got, want), float((got - want).abs().max())
    # ... and inside a CUDA graph: the launch allocates its work counter in stream order (cudaMallocAsync), which a capture records
    many = torch.rand(400, 3, 96, 192, device=DEV)   # 1 200 strips of three tiles
    Mm = _bench_homographies(400, 96, 192, 5).to(DEV)
    with K.config.override(dyn_sched=0):
        want = K.warp_perspective(many, Mm, (96, 192))
    graphed = K.graphs.GraphedCall(lambda a, b: K.warp_perspective(a, b, (96, 192)), many, Mm)
    for _ in range(3):
        got = graphed(many, Mm)
    assert torch.equal(got, want)


def test_fast_division_is_ieee():
    """The shared-reciprocal division of the tiled kernel vs div.rn on 2^26 operand pairs in the ranges the
    normalised coordinates live in, plus wide-exponent pairs."""
    import ctypes

    from kornia_b200 import _lib

    lib = _lib.load()
    g = torch.Generator(device=DEV).manual_seed(1)
    n = 1 << 26
    for scale_n, scale_d in ((2.0, 2.0), (1e6, 1e-3), (1e-20, 1e10)):
        num = (torch.rand(n, device=DEV, generator=g) * 2 - 1) * scale_n
        den = (torch.rand(n, device=DEV, generator=g) * 2 - 1) * scale_d
        den[:1000] = torch.tensor([1.0, -1.0, 3.0, 0.1, 1e-18, -1e-18, 1e18, 7.0, 1.0000001, 0.99999994], device=DEV).repeat(100)
        cnt = torch.zeros(1, dtype=torch.int32, device=DEV)
        rc = lib.kb200_debug_fastdiv_mismatches(num.data_ptr(), den.data_ptr(), n, cnt.data_ptr(), None)
        assert rc == 0
        assert int(cnt.item()) == 0, f"{int(cnt.item())} mismatches at scales {scale_n}, {scale_d}"


def test_full_size_parity_1080p():
    """BASELINE.json configs[1] shape at reduced batch: tiled kernel vs (a) the generic kernel, bit exact;
    (b) the oracle on the SAME device, i.e. the reference's own CUDA path (ATen sampler, cuDNN off), to
    1e-6; (c) the CPU oracle on a band-limited image, 1e-4 norm-relative (north_star tolerance)."""
    H, W, B = 1080, 1920, 3
    M = _bench_homographies(B, H, W, 1000).to(DEV)
    g = torch.Generator().manual_seed(0)
    noise = torch.rand(B, 3, H, W, generator=g)
    yy = torch.linspace(0, 1, H)[:, None]
    xx = torch.linspace(0, 1, W)[None, :]
    smooth = torch.stack([torch.stack([0.5 + 0.25 * torch.sin(6.2831853 * ((c + 1) * xx + (b + 2) * yy)) +
                                       0.2 * torch.cos(6.2831853 * (5 * xx - 3 * yy + 0.1 * c)) for c in range(3)]) for b in range(B)])
    for img in (noise, smooth):
        ours = K.warp_perspective(img.to(DEV), M, (H, W))
        gen = _generic(lambda: K.warp_perspective(img.to(DEV), M, (H, W)))
        assert torch.equal(ours, gen)
        was = torch.backends.cudnn.enabled
        torch.backends.cudnn.enabled = False
        try:
            same_dev = R.warp_perspective(img.to(DEV), M, (H, W))
        finally:
            torch.backends.cudnn.enabled = was
        assert rel_l2(ours, same_dev) < 1e-6, rel_l2(ours, same_dev)
    cpu = R.warp_perspective(smooth, M.cpu(), (H, W))
    assert rel_l2(ours.cpu(), cpu) < 1e-4, rel_l2(ours.cpu(), cpu)


def test_batch_shards_equal_whole():
    """Sharding the batch (what the multi-GPU path does) cannot change any sample."""
    H, W, B = 270, 480, 8
    M = _bench_homographies(B, H, W, 3, sigma=3.0).to(DEV)
    src = torch.rand(B, 3, H, W, device=DEV)
    whole = K.warp_perspective(src, M, (H, W))
    parts = torch.cat([K.warp_perspective(src[i:i + 3], M[i:i + 3], (H, W)) for i in range(0, B, 3)])
    assert torch.equal(whole, parts)
    # linearity in the image (the warp is a linear operator for fixed M)
    other = torch.rand_like(src)
    lin = K.warp_perspective(src + other, M, (H, W))
    torch.testing.assert_close(lin, whole + K.warp_perspective(other, M, (H, W)), rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("dt", [torch.float32, torch.float64])
def test_fused_prelude_bit_identical(dt):
    """kb200_warp_prelude vs the reference's torch op sequence on the same device, over batch sizes (torch picks
    different GEMM kernels by size), image sizes and both matrix kinds."""
    from kornia_b200.geometry import _prelude as P

    g = torch.Generator().manual_seed(11)
    bad = {}
    for n in (2, 3, 4, 5, 7, 8, 16, 31, 64, 100, 256, 1000, 2048):
        for (H, W, h, w) in ((1080, 1920, 1080, 1920), (720, 1280, 360, 640), (37, 53, 29, 41), (64, 64, 64, 64)):
            M = torch.eye(3)[None].repeat(n, 1, 1) + 0.2 * torch.randn(n, 3, 3, generator=g)
            M[:, 2, :2] *= 0.001
            M = M.to(dt).to(DEV)
            want = P.inverse3x3(P.normalize_homography(M, (H, W), (h, w)))
            got = P.sampling_matrix(M, (H, W), (h, w), affine=False)
            A = M[:, :2].contiguous()
            want_a = P.inverse3x3(P.normalize_homography(P.affine_to_homography(A), (H, W), (h, w)))
            got_a = P.sampling_matrix(A, (H, W), (h, w), affine=True)
            nb = int((got != want).sum()) + int((got_a != want_a).sum())
            if nb:
                bad[(n, H, W)] = nb
    assert not bad, bad


def test_prelude_keeps_autograd_path():
    M = (torch.eye(3, device=DEV)[None].repeat(4, 1, 1) + 0.01).requires_grad_()
    src = torch.rand(4, 3, 32, 64, device=DEV, requires_grad=True)
    out = K.warp_perspective(src, M, (32, 64))
    gs, gm = torch.autograd.grad(out.sum(), [src, M])
    assert gs.shape == src.shape and gm.shape == M.shape and float(gm.abs().sum()) > 0


# ------------------------------------------------------------------ the tiled separable filter
@pytest.mark.parametrize("border", ["constant", "reflect", "replicate"])
@pytest.mark.parametrize("k", [3, 5, 7, 9, 11, 13, 15, 17])
def test_tiled_sepfilter_bit_identical_to_generic(k, border):
    """Per-sample taps exercise the b % Bk indexing; 37 x 3 x 200 x 520 has more strips than the persistent grid has CTAs.
    Each shape also runs on an image with NaN / Inf / -0 / subnormal texels at the tile seams (against the generic kernel,
    bit for bit with -0 != +0; tests/test_nonfinite_gpu.py checks it against the reference)."""
    from test_nonfinite_gpu import bits_equal, special_image

    g = torch.Generator().manual_seed(k)
    shapes = ((2, 3, 70, 200), (1, 1, 32, 128), (3, 2, 45, 132), (1, 3, 9 + k, 12 + 4 * (k // 4)), (3, 2, 33, 4), (1, 1, 6, 8),
              (2, 3, 1080, 1920), (37, 3, 200, 520))
    for (B, C, H, W) in shapes:
        if border != "constant" and min(H, W) <= k // 2:  # a fold needs an image larger than the half-width
            continue
        x = torch.rand(B, C, H, W, generator=g).to(DEV)
        kx = torch.randn(B, k, generator=g).to(DEV)
        ky = torch.randn(1, k, generator=g).to(DEV)
        for xx in (x, special_image(B, C, H, W, seed=k)) if B * C * H * W < 10 ** 6 else (x,):
            a = K.filter2d_separable(xx, kx, ky, border)
            with K.config.override(tiled_filter=0):
                b = K.filter2d_separable(xx, kx, ky, border)
            assert bits_equal(a, b), (B, C, H, W, float((a - b).abs().nan_to_num().max()))
        a = K.filter2d_separable(x, kx, ky, border)
        want = R.filter2d_separable(x.cpu(), kx.cpu(), ky.cpu(), border)
        torch.testing.assert_close(a.cpu(), want, rtol=1e-4, atol=1e-5)


def test_gaussian_blur_1080p_vs_oracle():
    """BASELINE.json configs[2] shape at reduced batch, against the CPU oracle (reference ops)."""
    g = torch.Generator().manual_seed(2)
    x = torch.rand(2, 3, 1080, 1920, generator=g)
    a = K.gaussian_blur2d(x.to(DEV), (11, 11), (2.0, 2.0)).cpu()
    want = R.gaussian_blur2d(x, (11, 11), (2.0, 2.0))
    assert rel_l2(a, want) < 1e-6, rel_l2(a, want)
    torch.testing.assert_close(a, want, rtol=1e-4, atol=1e-5)


# ------------------------------------------------------------------ the tiled backward kernel
@pytest.mark.parametrize("pad", ["zeros", "border"])
@pytest.mark.parametrize("ac", [True, False])
@pytest.mark.parametrize("C", [3, 1])
def test_tiled_backward_matches_generic_and_oracle(pad, ac, C):
    H, W = 120, 256
    M = torch.cat([_wild_matrices(H, W), _bench_homographies(6, H, W, 9, sigma=3.0)]).to(DEV)
    B = M.shape[0]
    g = torch.Generator().manual_seed(C)
    src = torch.rand(B, C, H, W, generator=g).to(DEV)
    for dsize in ((H, W), (96, 200)):
        cot = (torch.rand(B, C, *dsize, generator=g) - 0.5).to(DEV)

        def grads(kind):
            s = src.clone().requires_grad_(True)
            if kind == "persp":
                mm = M.clone().requires_grad_(True)
                out = K.warp_perspective(s, mm, dsize, padding_mode=pad, align_corners=ac)
            else:
                mm = M[:, :2].clone().requires_grad_(True)
                out = K.warp_affine(s, mm, dsize, padding_mode=pad, align_corners=ac)
            return torch.autograd.grad(out, [s, mm], grad_outputs=cot)

        for kind in ("persp", "affine"):
            gs, gm = grads(kind)
            gs_ref, gm_ref = _generic(lambda: grads(kind))
            assert rel_l2(gs, gs_ref) < 2e-6, (kind, dsize, rel_l2(gs, gs_ref))
            torch.testing.assert_close(gs, gs_ref, rtol=1e-4, atol=2e-5)
            # d/dM sums ~10^4 terms per entry: compare per sample in norm (a horizon-crossing sample has huge entries)
            for b in range(B):
                if not torch.isfinite(gm_ref[b]).all():
                    continue
                assert rel_l2(gm[b], gm_ref[b]) < 1e-4, (kind, dsize, b, rel_l2(gm[b], gm_ref[b]))
    # only one of the two gradients requested
    s = src.clone().requires_grad_(True)
    out = K.warp_perspective(s, M, (H, W), padding_mode=pad, align_corners=ac)
    (gs_only,) = torch.autograd.grad(out, [s], grad_outputs=torch.ones_like(out))
    mm = M.clone().requires_grad_(True)
    out = K.warp_perspective(src, mm, (H, W), padding_mode=pad, align_corners=ac)
    (gm_only,) = torch.autograd.grad(out, [mm], grad_outputs=torch.ones_like(out))
    s2, m2 = src.clone().requires_grad_(True), M.clone().requires_grad_(True)
    out = K.warp_perspective(s2, m2, (H, W), padding_mode=pad, align_corners=ac)
    gs_both, gm_both = torch.autograd.grad(out, [s2, m2], grad_outputs=torch.ones_like(out))
    assert rel_l2(gs_only, gs_both) < 2e-6
    for b in range(B):
        if torch.isfinite(gm_both[b]).all():
            assert rel_l2(gm_only[b], gm_both[b]) < 1e-5


def test_tiled_backward_720p_vs_cpu_oracle():
    """BASELINE.json configs[3] shape at reduced batch: d/dsrc and d/dH against the reference's autograd on CPU."""
    H, W, B = 720, 1280, 2
    M = _bench_homographies(B, H, W, 7).to(DEV)
    yy = torch.linspace(0, 1, H)[:, None]
    xx = torch.linspace(0, 1, W)[None, :]
    smooth = torch.stack([torch.stack([0.5 + 0.25 * torch.sin(6.2831853 * ((c + 1) * xx + (b + 2) * yy)) +
                                       0.2 * torch.cos(6.2831853 * (5 * xx - 3 * yy + 0.1 * c)) for c in range(3)]) for b in range(B)])
    target = smooth.flip(-1) * 0.5 + 0.25

    def run(mod, s, m, t):
        s = s.clone().requires_grad_(True)
        m = m.clone().requires_grad_(True)
        loss = ((mod.warp_perspective(s, m, (H, W)) - t) ** 2).mean()
        return torch.autograd.grad(loss, [s, m])

    gs, gm = run(K, smooth.to(DEV), M, target.to(DEV))
    gs_ref, gm_ref = run(R, smooth, M.cpu(), target)
    assert rel_l2(gs.cpu(), gs_ref) < 1e-4, rel_l2(gs.cpu(), gs_ref)
    # against the CPU run the bound is the reference's own CPU-vs-CUDA gap (base grid and bmm differ by an ulp between the
    # backends, SURVEY 7); the north_star tolerance is asserted against the SAME-DEVICE reference in the next test
    assert rel_l2(gm.cpu(), gm_ref) < 5e-4, rel_l2(gm.cpu(), gm_ref)


@pytest.mark.parametrize("images", ["bandlimited", "white"])
def test_gradients_match_the_same_device_reference_at_the_cfg4_shape(images):
    """north_star: within 1e-4 rel of the reference's own grid_sample path.  The reference composition (oracle/kornia_restated.py,
    the ATen calls the reference issues) runs on the SAME GPU, cuDNN off, at BASELINE.json configs[3]'s shape (reduced batch); d/dsrc
    and d/dH through both, for the well-conditioned band-limited loss and for a white-noise cotangent.  (tests/geometry/transform/
    test_imgwarp.py:548-555 skips d/dH altogether; measured here: ~5e-8 and ~1e-6.)"""
    import bench

    H, W, B = 720, 1280, 4
    M = _bench_homographies(B, H, W, 7).to(DEV)
    shape = (B, 3, H, W)
    if images == "white":
        src, cot = torch.rand(shape, device=DEV), torch.randn(shape, device=DEV)
        loss = lambda out: (out * cot).sum()  # noqa: E731
    else:
        src, target = bench.bandlimited(shape, DEV, 12), bench.bandlimited(shape, DEV, 13)
        loss = lambda out: ((out - target) ** 2).mean()  # noqa: E731

    def run(mod):
        s, m = src.clone().requires_grad_(True), M.clone().requires_grad_(True)
        out = mod.warp_perspective(s, m, (H, W))
        return (out.detach(),) + torch.autograd.grad(loss(out), [s, m])

    with torch.backends.cudnn.flags(enabled=False):
        want = run(R)
    got = run(K)
    assert torch.equal(got[0], want[0]), "the forward is bit-identical to the same-device reference"
    assert rel_l2(got[1], want[1]) < 1e-5, rel_l2(got[1], want[1])   # d/dsrc: only the order of the adds differs
    for b in range(B):
        assert rel_l2(got[2][b], want[2][b]) < 1e-4, (b, rel_l2(got[2][b], want[2][b]))  # d/dH per sample


@pytest.mark.parametrize("border", ["constant", "reflect", "replicate"])
@pytest.mark.parametrize("k", [3, 5, 7])
def test_tiled_filter2d_bit_identical_to_generic(k, border):
    """Also on an image with NaN / Inf / -0 / subnormal texels at the tile seams and a sample of -0 (against the generic kernel
    only).  The third kernel has only positive taps, like a blur: then a -0 sample filters to -0 or +0 depending on how the
    accumulator is seeded, which bits_equal sees and torch.equal does not."""
    from test_nonfinite_gpu import bits_equal, special_image

    g = torch.Generator().manual_seed(10 + k)
    for (B, C, H, W) in ((2, 3, 70, 200), (1, 1, 32, 128), (4, 2, 45, 132), (1, 3, 6 + k, 12)):
        x = torch.rand(B, C, H, W, generator=g).to(DEV)
        for kern in (torch.randn(1, k, k, generator=g), torch.randn(B, k, k, generator=g), torch.rand(1, k, k, generator=g)):
            kern = kern.to(DEV)
            for normalized, behaviour in ((False, "corr"), (True, "conv")):
                for xx in (x, special_image(B, C, H, W, seed=k)):
                    a = K.filter2d(xx, kern, border, normalized=normalized, behaviour=behaviour)
                    with K.config.override(tiled_filter=0):
                        b = K.filter2d(xx, kern, border, normalized=normalized, behaviour=behaviour)
                    assert bits_equal(a, b), (B, C, H, W, float((a - b).abs().nan_to_num().max()))
                a = K.filter2d(x, kern, border, normalized=normalized, behaviour=behaviour)
                want = R.filter2d(x.cpu(), kern.cpu(), border, normalized=normalized, behaviour=behaviour)
                torch.testing.assert_close(a.cpu(), want, rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("pad", ["zeros", "border", "reflection"])
@pytest.mark.parametrize("ac", [None, True])
@pytest.mark.parametrize("C", [3, 1])
def test_tiled_remap_bit_identical_to_generic(pad, ac, C):
    """Smooth maps (served from the staged box), a noisy map (mostly exact path), out-of-view and NaN entries; then special
    texels under the same maps, and maps with NaN / Inf / beyond-int / -0 / edge entries at the tile seams."""
    from test_nonfinite_gpu import _special_maps, bits_equal, special_image

    H, W, h, w = 96, 160, 80, 136
    g = torch.Generator().manual_seed(4)
    img = torch.rand(3, C, H, W, generator=g).to(DEV)
    ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float32), torch.arange(w, dtype=torch.float32), indexing="ij")
    smooth_x = xs * (W / w) + 3.0 * torch.sin(ys / 9.0) - 4.0
    smooth_y = ys * (H / h) + 2.5 * torch.cos(xs / 11.0) + 1.0
    noisy_x = smooth_x + 30.0 * torch.randn(h, w, generator=g)
    noisy_y = smooth_y + 30.0 * torch.randn(h, w, generator=g)
    far_x = smooth_x + 5000.0
    bad_x = smooth_x.clone()
    bad_x[::7, ::5] = float("nan")
    mx = torch.stack([smooth_x, noisy_x, bad_x]).to(DEV)
    my = torch.stack([smooth_y, noisy_y, smooth_y]).to(DEV)
    sx, sy = _special_maps(H, W, h, w, seed=C)
    special = special_image(3, C, H, W, seed=C)
    for (im, ax, ay) in ((img, mx, my), (img, far_x[None].to(DEV), smooth_y[None].to(DEV)), (img, smooth_x[None].to(DEV), smooth_y[None].to(DEV)),
                         (special, mx, my), (special, sx[None].to(DEV), sy[None].to(DEV))):
        a = K.remap(im, ax, ay, padding_mode=pad, align_corners=ac)
        b = _generic(lambda: K.remap(im, ax, ay, padding_mode=pad, align_corners=ac), check_variant=False)
        assert bits_equal(a, b), float((a - b).abs().nan_to_num().max())
    want = R.remap(img.cpu()[:1], smooth_x[None], smooth_y[None], padding_mode=pad, align_corners=ac)
    got = K.remap(img[:1], smooth_x[None].to(DEV), smooth_y[None].to(DEV), padding_mode=pad, align_corners=ac)
    torch.testing.assert_close(got.cpu(), want, rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("pad", ["zeros", "reflection"])
def test_tiled_remap_many_strips(pad):
    """A batch of many tiles with per-sample and shared maps and normalised coordinates: the tiled kernel against the generic
    kernel, bit for bit, in one launch."""
    B, H, W = 40, 200, 264   # 40 x 7 = 280 strips of 5 tiles
    g = torch.Generator().manual_seed(11)
    img = torch.rand(B, 3, H, W, generator=g).to(DEV)
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    amp = torch.linspace(0.0, 6.0, B)[:, None, None]
    mx = (xs[None] + amp * torch.sin(ys / 17.0)[None] - 2.0).contiguous().to(DEV)
    my = (ys[None] + amp * torch.cos(xs / 23.0)[None] + 1.5).contiguous().to(DEV)
    for (ax, ay, norm) in ((mx, my, False), (mx[:1], my[:1], False), (2 * mx / (W - 1) - 1, 2 * my / (H - 1) - 1, True)):
        want = _generic(lambda: K.remap(img, ax, ay, padding_mode=pad, align_corners=True, normalized_coordinates=norm), check_variant=False)
        n0 = K._ops.launch_count
        got = K.remap(img, ax, ay, padding_mode=pad, align_corners=True, normalized_coordinates=norm)
        assert K._ops.launch_count - n0 == 1
        assert torch.equal(got, want), float((got - want).abs().max())


# ------------------------------------------------------------------ contract details on the device
def test_noncontiguous_inputs_and_contiguous_outputs():
    # tests/geometry/transform/test_imgwarp.py:487-489, tests/filters/test_filters.py:359-366: stride-0 expanded inputs
    img = torch.rand(1, 1, 20, 24, device=DEV).expand(3, 3, -1, -1)
    M = torch.eye(3, device=DEV)[None].expand(3, -1, -1)
    out = K.warp_perspective(img, M, (20, 24))
    assert out.is_contiguous()
    torch.testing.assert_close(out, img.contiguous(), rtol=1e-4, atol=1e-4)
    blur = K.gaussian_blur2d(img, (3, 3), (1.0, 1.0))
    assert blur.is_contiguous() and blur.shape == img.shape
    f = K.filter2d(img.transpose(-1, -2), torch.ones(1, 3, 3, device=DEV), normalized=True)
    assert f.is_contiguous()
    torch.testing.assert_close(f, R.filter2d(img.transpose(-1, -2).cpu(), torch.ones(1, 3, 3), normalized=True).to(DEV), rtol=1e-4, atol=1e-5)


def test_empty_batch_and_huge_separable_kernel():
    e = K.warp_affine(torch.rand(0, 3, 8, 8, device=DEV), torch.zeros(0, 2, 3, device=DEV), (4, 4))
    assert e.shape == (0, 3, 4, 4)
    x = torch.rand(1, 1, 160, 160, device=DEV)
    kx = torch.rand(1, 151, device=DEV)
    ky = torch.rand(1, 151, device=DEV)
    got = K.filter2d_separable(x, kx, ky, "constant")  # too large for the one-pass tile: two 1-D passes inside the library
    want = R.filter2d_separable(x.cpu(), kx.cpu(), ky.cpu(), "constant")
    assert rel_l2(got.cpu(), want) < 1e-5


def test_last_visible_device():
    """Device placement follows the tensors, not the current device: runs on the LAST visible GPU (cuda:1.. on a multi-GPU box;
    on a single-GPU box that is cuda:0 addressed explicitly while the current device stays the default)."""
    d1 = torch.device("cuda", torch.cuda.device_count() - 1)
    x = torch.rand(2, 3, 64, 128, device=d1)
    M = torch.eye(3, device=d1)[None].repeat(2, 1, 1)
    M[:, 0, 2] = 2.0
    a = K.warp_perspective(x, M, (64, 128))
    b = K.gaussian_blur2d(x, (5, 5), (1.0, 1.0))
    assert a.device == d1 and b.device == d1
    torch.testing.assert_close(a.cpu(), R.warp_perspective(x.cpu(), M.cpu(), (64, 128)), rtol=1e-4, atol=1e-5)


def test_tiled_backward_shared_affine_matrix():
    """warp_affine with one (1,2,3) matrix for the whole batch: d/dM sums over the batch (imgwarp.py:282-283)."""
    H, W, B = 64, 128, 5
    g = torch.Generator().manual_seed(3)
    src = torch.rand(B, 3, H, W, generator=g).to(DEV)
    A = torch.tensor([[[0.98, 0.05, 1.5], [-0.04, 1.01, -2.0]]], device=DEV)
    cot = (torch.rand(B, 3, H, W, generator=g) - 0.5).to(DEV)

    def grads():
        s, a = src.clone().requires_grad_(True), A.clone().requires_grad_(True)
        return torch.autograd.grad(K.warp_affine(s, a, (H, W)), [s, a], grad_outputs=cot)

    gs, ga = grads()
    gs_ref, ga_ref = _generic(grads)
    assert ga.shape == (1, 2, 3)
    assert rel_l2(gs, gs_ref) < 2e-6 and rel_l2(ga, ga_ref) < 1e-4
    s, a = src.cpu().requires_grad_(True), A.cpu().requires_grad_(True)
    gs_cpu, ga_cpu = torch.autograd.grad(R.warp_affine(s, a, (H, W)), [s, a], grad_outputs=cot.cpu())
    assert rel_l2(gs.cpu(), gs_cpu) < 1e-4 and rel_l2(ga.cpu(), ga_cpu) < 5e-4  # vs CPU: bounded by the reference's own CPU-vs-CUDA gap
