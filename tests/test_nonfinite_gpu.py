"""Non-finite texels, signed zeros, subnormals and degenerate geometry through the CUDA kernels.

Every other parity test feeds ``torch.rand`` images: finite, in [0, 1).  Depth maps and flow fields with NaN or Inf holes,
random augmentation that draws a scale of 0, and matrices that leave the int range go through the same kernels, and the code
that decides what happens to such pixels (the tile classes and box fitting of the tiled warp, the index guard, the exact
division fallback) is exactly what the fast kernels rewrite.  So here:

* the tiled kernels are compared with the generic ones with ``bits_equal`` (-0 and +0 differ, any NaN equals any NaN);
* both are compared with the reference composition (``oracle/kornia_restated.py``) run on the SAME GPU with cuDNN off --
  bit for bit where the finite tests already claim it, otherwise with ``classes_equal`` (NaN / +Inf / -Inf in the same
  places, finite entries within the existing tolerances);
* outputs written through the C ABI land in a buffer prefilled with a NaN of a payload no kernel produces, so a pixel
  that no kernel writes is told apart from a NaN the image or the geometry legitimately produces.

The CPU oracle is not the judge of non-finite coordinates: ATen's CPU and CUDA samplers clamp a NaN coordinate differently
(the CUDA one's ``fminf`` / ``fmaxf`` send it to texel 0 under 'border'); this library follows the CUDA behaviour, so every
comparison here runs the reference on the device."""
import math

import pytest
import torch
import torch.nn.functional as F

import kornia_b200 as K
from kornia_b200 import _lib
from kornia_b200.geometry import _prelude as P
from oracle import kornia_restated as R
from test_parity_gpu import _bench_homographies, _shift_matrices, _wild_matrices

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAN, INF = float("nan"), float("inf")
SPECIALS = (NAN, INF, -INF, -0.0, 1e-40, -1e-41, 1e-38, 3e38)
SENTINEL = {torch.float32: 0x7FC0DEAD, torch.float64: 0x7FF80000DEADBEEF}   # quiet NaNs with a payload no kernel writes
FP32 = dict(rtol=1e-4, atol=1e-5)
FP64 = dict(rtol=1e-12, atol=1e-13)


# ------------------------------------------------------------------------------------------ comparators
def _bits(t):
    return t.contiguous().view(torch.int64 if t.dtype == torch.float64 else torch.int32)


def bits_equal(a, b):
    """Same shape, dtype and bit pattern in every entry: -0 != +0; any NaN equals any NaN (the device writes one canonical
    NaN, the reference may carry the input's)."""
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    nan_a, nan_b = torch.isnan(a), torch.isnan(b)
    return bool(torch.equal(nan_a, nan_b) and ((_bits(a) == _bits(b)) | nan_a).all())


def classes_equal(a, b, rtol=0.0, atol=0.0):
    """NaN, +Inf and -Inf in exactly the same places; the finite entries within ``atol + rtol * |b|``."""
    if a.shape != b.shape:
        return False
    for cls in (torch.isnan, torch.isposinf, torch.isneginf):
        if not torch.equal(cls(a), cls(b)):
            return False
    fin = torch.isfinite(a)
    x, y = a[fin].double(), b[fin].double()
    return bool(((x - y).abs() <= atol + rtol * y.abs()).all())


def diff(a, b):
    """What differs, for an assertion message: counts per class and the first entry whose bits differ."""
    if a.shape != b.shape:
        return f"shapes {tuple(a.shape)} vs {tuple(b.shape)}"
    kinds = {n: int((f(a) != f(b)).sum()) for n, f in (("nan", torch.isnan), ("+inf", torch.isposinf), ("-inf", torch.isneginf))}
    both_nan = torch.isnan(a) & torch.isnan(b)
    bad = ((_bits(a) != _bits(b)) & ~both_nan).flatten().nonzero()
    if not len(bad):
        return f"class mismatches {kinds}"
    i = int(bad[0])
    return f"{len(bad)} of {a.numel()} differ (class mismatches {kinds}); first at {i}: {a.flatten()[i].item()!r} vs {b.flatten()[i].item()!r}"


def sentinel_like(shape, dtype=torch.float32):
    return torch.full(shape, SENTINEL[dtype], dtype=torch.int64 if dtype == torch.float64 else torch.int32, device=DEV).view(dtype)


def unwritten(out):
    return int((_bits(out) == SENTINEL[out.dtype]).sum())


# ------------------------------------------------------------------------------------------ special texels
def seam_rows(H):
    """Rows where tiles meet: the first and last row of the image and of every 32-row strip."""
    return sorted({r for k in range(0, H + 32, 32) for r in (k - 1, k)} & set(range(H)) | {0, H - 1})


def seam_cols(W):
    """Columns where tiles and boxes meet: 0, W-1, k*32 - 1, k*32, k*64 and k*128 +- 1."""
    cols = {0, W - 1}
    for k in range(0, W // 32 + 2):
        cols |= {32 * k - 1, 32 * k, 64 * k, 128 * k - 1, 128 * k + 1}
    return sorted(cols & set(range(W)))


def special_image(B, C, H, W, seed=0, dtype=torch.float32, whole=True, huge=True):
    """``torch.rand`` with {NaN, +-Inf, -0, subnormals, 1e-38, 3e38} scattered (~0.2 %) and placed along the tile seams
    (every 29th texel of each seam row and column, at a random phase); with ``whole`` and B >= 4 the last three samples are
    all -0, all NaN and all subnormal.  ``huge=False`` leaves out 3e38: where two computations sum the same terms in a
    different order, whether a partial sum of such texels overflows to Inf depends on that order, not on the kernel."""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(B, C, H, W, generator=g, dtype=torch.float64)
    sp = torch.tensor([v for v in SPECIALS if huge or v != 3e38], dtype=torch.float64)

    def draw(*shape):
        return sp[torch.randint(len(sp), shape, generator=g)]

    flat = x.view(-1)
    n = max(1, flat.numel() // 500)
    flat[torch.randint(flat.numel(), (n,), generator=g)] = draw(n)
    for r in seam_rows(H):
        idx = torch.arange(int(torch.randint(29, (1,), generator=g)) % W, W, 29)
        x[:, :, r, idx] = draw(B, C, len(idx))
    for c in seam_cols(W):
        idx = torch.arange(int(torch.randint(29, (1,), generator=g)) % H, H, 29)
        x[:, :, idx, c] = draw(B, C, len(idx))
    if whole and B >= 4:
        x[B - 3] = -0.0
        x[B - 2] = NAN
        x[B - 1] = torch.rand(C, H, W, generator=g, dtype=torch.float64) * (1e-39 if dtype == torch.float32 else 1e-310)
    return x.to(dtype).to(DEV)   # the double -> float cast keeps 1e-40 etc. subnormal and the signs of zeros


def degenerate_matrices(W):
    """The zero matrix, an exactly rank-2 M, a NaN and an Inf entry, translations beyond the int range and of 1e30, scales of
    1e-30 and 1e7, and a denominator that is negative everywhere."""
    eye = [[1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0]]

    def put(i, j, v):
        m = [row[:] for row in eye]
        m[i][j] = v
        return m

    mats = [[[0.0] * 3] * 3,
            [[1.0, 2.0, 5.0], [2.0, 4.0, 10.0], [0.0, 0.0, 1.0]],       # rank 2 (also as an affine map)
            put(0, 1, NAN), put(1, 2, INF),
            [[1.0, 0.0, 3e9], [0.0, 1.0, -3e9], [0.0, 0.0, 1.0]], put(0, 2, -3e9), put(1, 2, 1e30),
            [[1e-30, 0.0, 0.0], [0.0, 1e-30, 0.0], [0.0, 0.0, 1.0]], [[1e7, 0.0, 0.0], [0.0, 1e7, 0.0], [0.0, 0.0, 1.0]],
            [[-1.0, 0.02, 3.0], [0.01, -1.0, -2.0], [1e-4, -2e-4, -1.0]]]   # w < 0 over the whole image
    return torch.tensor(mats, dtype=torch.float32)


def all_matrices(H, W):
    return torch.cat([_wild_matrices(H, W), _shift_matrices(W), _bench_homographies(4, H, W, 5, sigma=4.0), degenerate_matrices(W)]).to(DEV)


# ------------------------------------------------------------------------------------------ calls through the C ABI
def forward_abi(src, m, bx, by, h, w, projective, mode, pad, align, fill=None, tiled=True):
    """kb200_warp_forward into a sentinel-filled buffer; returns (out, variant)."""
    n, C, Hs, Ws = src.shape
    out = sentinel_like((n, C, h, w), src.dtype)
    dt = _lib.F32 if src.dtype == torch.float32 else _lib.F64
    with K.config.override(tma=int(tiled)):
        _lib.call("kb200_warp_forward", src.data_ptr(), m.data_ptr(), bx.data_ptr(), by.data_ptr(),
                  None if fill is None else fill.data_ptr(), out.data_ptr(), n, C, Hs, Ws, h, w, m.shape[0], int(projective),
                  _lib.INTERP[mode], _lib.PADDING[pad], int(align), dt, torch.cuda.current_stream().cuda_stream)
        variant = _lib.last_warp_variant()
    torch.cuda.synchronize()
    return out, variant


def warp_abi(src, M, dsize, projective, mode, pad, align, fill=None, tiled=True):
    h, w = dsize
    m = P.sampling_matrix(M, src.shape[-2:], dsize, affine=not projective).contiguous()
    if projective:
        bx, by = P.meshgrid_axes(h, w, src.device, src.dtype)
    else:
        bx, by = P.affine_axes(h, w, align, src.device, src.dtype)
    return forward_abi(src, m, bx.contiguous(), by.contiguous(), h, w, projective, mode, pad, align, fill, tiled)


def remap_abi(img, mx, my, mode, pad, align, normalized=False, tiled=True):
    B, C, H, W = img.shape
    _, h, w = mx.shape
    out = sentinel_like((B, C, h, w), img.dtype)
    dt = _lib.F32 if img.dtype == torch.float32 else _lib.F64
    with K.config.override(tma=int(tiled)):
        _lib.call("kb200_remap_forward", img.data_ptr(), mx.data_ptr(), my.data_ptr(), out.data_ptr(), B, C, H, W, h, w, mx.shape[0],
                  int(normalized), _lib.INTERP[mode], _lib.PADDING[pad], int(align), dt, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return out


def reference(fn):
    with torch.backends.cudnn.flags(enabled=False):
        return fn()


def check_against_reference(got, want, mode, what):
    """Bilinear and nearest replicate ATen's sampler op for op (bit for bit, as for finite inputs); ATen's bicubic contracts its
    weight polynomials with FMAs of its own choosing (the finite tolerance, 1e-5 / 2e-6)."""
    if mode == "bicubic":
        assert classes_equal(got, want, rtol=1e-5, atol=2e-6), (what, diff(got, want))
    else:
        assert bits_equal(got, want), (what, diff(got, want))


# ------------------------------------------------------------------------------------------ warps, forward
# the tiled kernel serves C 1..4 under bilinear, C 1 and 3 under nearest and bicubic
_FWD_CASES = [(mode, pad, C) for mode in ("bilinear", "nearest", "bicubic") for pad in ("zeros", "border", "reflection")
              for C in ((1, 3, 4) if mode == "bilinear" else (1, 3))]
_FWD_CASES += [(mode, "fill", 3) for mode in ("bilinear", "nearest", "bicubic")]


@pytest.mark.parametrize("mode,pad,C", _FWD_CASES)
@pytest.mark.parametrize("ac", [True, False])
def test_warp_forward_special_texels_and_degenerate_matrices(mode, pad, C, ac):
    """Special texels under rotations, zooms, horizons, out-of-view and shifted samples, the bench homographies and degenerate
    matrices (singular, NaN / Inf entries, beyond the int range, scales of 1e-30 and 1e7, negative denominator): (a) the
    tiled kernel bits_equal the generic one, (b) both match the same-device reference, (c) every pixel is written."""
    H, W = 216, 384
    M = all_matrices(H, W)
    # bicubic: no 3e38 texels -- ATen contracts its weight polynomials with FMAs of its own choosing, so whether 16 weighted
    # texels near FLT_MAX overflow depends on that choice
    src = special_image(M.shape[0], C, H, W, seed=C, huge=mode != "bicubic")
    fill = torch.tensor([0.2, 0.5, 0.8], device=DEV) if pad == "fill" else None
    for projective in (True, False):
        Mk = M if projective else M[:, :2].contiguous()
        for dsize in ((H, W), (150, 333)):
            what = (projective, dsize)
            tiled, variant = warp_abi(src, Mk, dsize, projective, mode, pad, ac, fill)
            assert variant == "tma_tile", what
            gen, variant = warp_abi(src, Mk, dsize, projective, mode, pad, ac, fill, tiled=False)
            assert variant == "generic", what
            assert unwritten(tiled) == 0 and unwritten(gen) == 0, (what, unwritten(tiled), unwritten(gen))
            assert bits_equal(tiled, gen), (what, "tiled vs generic", diff(tiled, gen))
            if projective:
                want = reference(lambda: R.warp_perspective(src, Mk, dsize, mode=mode, padding_mode=pad, align_corners=ac, fill_value=fill))
            else:
                want = reference(lambda: R.warp_affine(src, Mk, dsize, mode=mode, padding_mode=pad, align_corners=ac, fill_value=fill))
            check_against_reference(tiled, want, mode, what)


def test_warp_forward_special_texels_in_the_run_time_sweep():
    """A 1080p batch large enough for the run-time sweep (warp_fwd_tma<DYN>) with special texels and degenerate samples."""
    H, W = 1080, 1920
    M = torch.cat([_bench_homographies(32 - 10 - 10, H, W, 3), _wild_matrices(H, W), degenerate_matrices(W)]).to(DEV)
    src = special_image(M.shape[0], 3, H, W, seed=40)
    assert K.config.get("dyn_sched") == 1
    for pad in ("zeros", "reflection"):
        tiled, variant = warp_abi(src, M, (H, W), True, "bilinear", pad, True)
        assert variant == "tma_tile"
        gen, _ = warp_abi(src, M, (H, W), True, "bilinear", pad, True, tiled=False)
        assert unwritten(tiled) == 0, unwritten(tiled)
        assert bits_equal(tiled, gen), (pad, diff(tiled, gen))
        want = reference(lambda: R.warp_perspective(src, M, (H, W), padding_mode=pad))
        assert bits_equal(tiled, want), (pad, diff(tiled, want))


def _hand_built(kind, B):
    """Normalised sampling matrices (dst -> src) the prelude would not produce: a denominator exactly 0 on the middle output
    column (m20 = 1, m21 = m22 = 0), and one of ~1e-20, below the 2^-60 window of the shared-reciprocal division."""
    m = torch.eye(3).repeat(B, 1, 1)
    if kind == "zero_column":
        m[:, 2] = torch.tensor([1.0, 0.0, 0.0])
        m[1:, 0, 2] = torch.linspace(-0.5, 0.5, B - 1)
    elif kind == "tiny":
        m[:, 2, 2] = 1e-20
        m[1:, :2, :] *= 1e-20   # numerators of the same size: coordinates inside the image through the exact division
        m[2:, 0, 1] = 3e-21
    return m.to(DEV).contiguous()


@pytest.mark.parametrize("kind", ["zero_column", "tiny"])
@pytest.mark.parametrize("mode,pad", [(mode, pad) for mode in ("bilinear", "nearest", "bicubic") for pad in ("zeros", "border", "reflection", "fill")])
def test_warp_forward_degenerate_denominators_through_the_abi(kind, mode, pad):
    H, W, h, w = 96, 160, 67, 131   # odd w: the middle column's base coordinate is exactly 0
    B = 4
    src = special_image(B, 3, H, W, seed=9, whole=False)
    m = _hand_built(kind, B)
    bx, by = P.meshgrid_axes(h, w, DEV, torch.float32)
    bx, by = bx.contiguous(), by.contiguous()
    assert float(bx[w // 2]) == 0.0 and not torch.signbit(bx[w // 2])
    fill = torch.tensor([0.2, 0.5, 0.8], device=DEV) if pad == "fill" else None
    for ac in (True, False):
        tiled, variant = forward_abi(src, m, bx, by, h, w, True, mode, pad, ac, fill)
        assert variant == "tma_tile"
        gen, _ = forward_abi(src, m, bx, by, h, w, True, mode, pad, ac, fill, tiled=False)
        assert unwritten(tiled) == 0 and unwritten(gen) == 0
        assert bits_equal(tiled, gen), (ac, diff(tiled, gen))

        def ref():
            grid = R.perspective_grid(m, bx, by)
            if pad == "fill":
                return R.fill_and_sample(src, grid, mode, ac, fill)
            return F.grid_sample(src, grid, mode=mode, padding_mode=pad, align_corners=ac)

        check_against_reference(tiled, reference(ref), mode, ac)


def _special_maps(H, W, h, w, seed):
    """Smooth pixel maps with NaN, +-Inf, +-2^31, +-3e9, -0, -1, W-1 and W (H-1, H for y) at the tile seams and scattered."""
    g = torch.Generator().manual_seed(seed)
    ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float32), torch.arange(w, dtype=torch.float32), indexing="ij")
    mx = xs * (W / w) + 3.0 * torch.sin(ys / 9.0) - 2.0
    my = ys * (H / h) + 2.5 * torch.cos(xs / 11.0) + 1.0
    vx = torch.tensor([NAN, INF, -INF, 2.0 ** 31, -(2.0 ** 31), 3e9, -3e9, -0.0, -1.0, W - 1.0, float(W)])
    vy = torch.tensor([NAN, INF, -INF, 2.0 ** 31, -(2.0 ** 31), 3e9, -3e9, -0.0, -1.0, H - 1.0, float(H)])
    for mm, v in ((mx, vx), (my, vy)):
        flat = mm.view(-1)
        n = flat.numel() // 200
        flat[torch.randint(flat.numel(), (n,), generator=g)] = v[torch.randint(len(v), (n,), generator=g)]
        for r in seam_rows(h):
            idx = torch.arange(int(torch.randint(13, (1,), generator=g)) % w, w, 13)
            mm[r, idx] = v[torch.randint(len(v), (len(idx),), generator=g)]
        for c in seam_cols(w):
            idx = torch.arange(int(torch.randint(13, (1,), generator=g)) % h, h, 13)
            mm[idx, c] = v[torch.randint(len(v), (len(idx),), generator=g)]
    return mx, my


@pytest.mark.parametrize("mode", ["bilinear", "nearest", "bicubic"])
@pytest.mark.parametrize("pad", ["zeros", "border", "reflection"])
@pytest.mark.parametrize("C", [1, 3])
def test_remap_special_maps_and_texels(mode, pad, C):
    """remap with special map entries (pixel maps, and normalised maps holding exactly +-1) over special texels: the tiled kernel
    (bilinear) bits_equal the generic one; both match the same-device reference; every pixel is written."""
    H, W, h, w = 96, 160, 80, 136
    img = special_image(4, C, H, W, seed=11 + C)
    mx, my = _special_maps(H, W, h, w, seed=C)
    ys, xs = torch.meshgrid(torch.linspace(-1, 1, h), torch.linspace(-1, 1, w), indexing="ij")
    nx, ny = xs.clone(), ys.clone()
    nx[:, ::3], ny[::4, :] = 1.0, -1.0
    nx[::5, 1::3] = -1.0
    cases = [(mx[None], my[None], False), (torch.stack([mx, mx.flip(-1), mx, mx]), torch.stack([my, my, my.flip(0), my]), False),
             (nx[None], ny[None], True)]
    for ac in (True, False):
        for ax, ay, norm in cases:
            ax, ay = ax.to(DEV).contiguous(), ay.to(DEV).contiguous()
            got = remap_abi(img, ax, ay, mode, pad, ac, norm)
            gen = remap_abi(img, ax, ay, mode, pad, ac, norm, tiled=False)
            assert unwritten(got) == 0 and unwritten(gen) == 0
            assert bits_equal(got, gen), (ac, norm, diff(got, gen))
            want = reference(lambda: R.remap(img, ax, ay, mode=mode, padding_mode=pad, align_corners=ac, normalized_coordinates=norm))
            check_against_reference(got, want, mode, (ac, norm))


@pytest.mark.parametrize("mode,pad", [("bilinear", "zeros"), ("bilinear", "border"), ("bilinear", "reflection"), ("bilinear", "fill"),
                                      ("nearest", "zeros"), ("bicubic", "border")])
def test_fp64_special_texels_and_degenerate_matrices(mode, pad):
    """fp64 (generic kernel) against the fp64 reference on the same device: the same non-finite classes, finite entries
    within 1e-12.  (Same device: the reference builds its base grid in fp32 even for fp64 input.)"""
    H, W = 64, 96
    M = torch.cat([_wild_matrices(H, W), degenerate_matrices(W)]).to(DEV, torch.float64)
    src = special_image(M.shape[0], 3, H, W, seed=64, dtype=torch.float64, huge=mode != "bicubic")
    fill = torch.tensor([0.2, 0.5, 0.8], device=DEV, dtype=torch.float64) if pad == "fill" else None
    for ac in (True, False):
        for dsize in ((H, W), (50, 77)):
            got, variant = warp_abi(src, M, dsize, True, mode, pad, ac, fill)
            assert variant == "generic" and unwritten(got) == 0
            want = reference(lambda: R.warp_perspective(src, M, dsize, mode=mode, padding_mode=pad, align_corners=ac, fill_value=fill))
            if mode == "nearest":
                assert bits_equal(got, want), (ac, dsize, diff(got, want))
            else:
                assert classes_equal(got, want, **FP64), (ac, dsize, diff(got, want))
            A = M[:, :2].contiguous()
            got = K.warp_affine(src, A, dsize, mode=mode, padding_mode=pad, align_corners=ac, fill_value=fill)
            want = reference(lambda: R.warp_affine(src, A, dsize, mode=mode, padding_mode=pad, align_corners=ac, fill_value=fill))
            assert classes_equal(got, want, **FP64), ("affine", ac, dsize, diff(got, want))
    mx, my = _special_maps(H, W, 40, 72, seed=5)
    mx, my = mx[None].to(DEV, torch.float64), my[None].to(DEV, torch.float64)
    img = src[:1]
    got = remap_abi(img, mx, my, mode, "zeros" if pad == "fill" else pad, True)
    want = reference(lambda: R.remap(img, mx, my, mode=mode, padding_mode="zeros" if pad == "fill" else pad, align_corners=True))
    assert unwritten(got) == 0 and classes_equal(got, want, **FP64), ("remap", diff(got, want))


# ------------------------------------------------------------------------------------------ warps, backward
def _rel_l2_finite(a, b):
    fin = torch.isfinite(b)
    x, y = a[fin].double(), b[fin].double()
    return float((x - y).norm() / y.norm().clamp_min(1e-30))


def _check_grads(got, want, what, gm_samples, nan_superset=False):
    """d/dsrc: the same classes, finite entries within 1e-5 in norm (atomic order moves values, not classes); d/dM: the same
    classes, and per sample in ``gm_samples`` the finite entries within 1e-4 in norm.  ``nan_superset``: d/dM may be NaN where
    the reference's is finite (see test_warp_backward_specials), never the other way round."""
    gs, gm = got
    gs_ref, gm_ref = want
    assert classes_equal(gs, gs_ref, atol=INF), (what, "d/dsrc", diff(gs, gs_ref))
    assert _rel_l2_finite(gs, gs_ref) < 1e-5, (what, "d/dsrc", _rel_l2_finite(gs, gs_ref))
    if nan_superset:
        fin = torch.isfinite(gm)
        assert torch.equal(fin & ~torch.isfinite(gm_ref), torch.zeros_like(fin)), (what, "d/dM", diff(gm, gm_ref))
        gm_ref = torch.where(fin, gm_ref, gm)
    assert classes_equal(gm, gm_ref, atol=INF), (what, "d/dM", diff(gm, gm_ref))
    for b in gm_samples:
        assert _rel_l2_finite(gm[b], gm_ref[b]) < 1e-4, (what, b, _rel_l2_finite(gm[b], gm_ref[b]))


def _backward_inputs(kind, B, C, H, W, dsize, seed):
    g = torch.Generator().manual_seed(seed)
    M = torch.cat([_wild_matrices(H, W), _bench_homographies(B - 10, H, W, 9, sigma=3.0)]).to(DEV)
    src = torch.rand(M.shape[0], C, H, W, generator=g).to(DEV)
    cot = (torch.rand(M.shape[0], C, *dsize, generator=g) - 0.5).to(DEV)
    if kind == "texels":
        src = special_image(M.shape[0], C, H, W, seed=seed, whole=False, huge=False)
    elif kind == "cotangent":
        cot = special_image(M.shape[0], C, *dsize, seed=seed, whole=False, huge=False) - 0.5
    else:
        M = torch.cat([M[:4], degenerate_matrices(W).to(DEV)])
        src, cot = src[:M.shape[0]], cot[:M.shape[0]]
    return src, M, cot


@pytest.mark.parametrize("kind", ["texels", "cotangent", "matrices"])
@pytest.mark.parametrize("stride1", [0, 1])
@pytest.mark.parametrize("pad", ["zeros", "border"])
@pytest.mark.parametrize("C", [1, 3])
def test_warp_backward_specials(kind, stride1, pad, C):
    """warp_bwd_tma2 (both lane layouts) against the generic backward, and against autograd of the reference on the same device:
    special texels, NaN / Inf in the upstream gradient, degenerate matrices.

    d/dM per sample is compared in norm only where it is a well-conditioned sum: not for the horizon sample (terms grow as
    1 / den^2 next to den = 0, as in test_tiled_backward_matches_generic) nor for the degenerate matrices (every pixel on a
    handful of texels, or no pixel in view), whose classes are still compared.

    Documented exception, NaN / Inf upstream gradient against the reference: ATen's sampler backward skips the taps of a pixel
    that lie outside the image, so an upstream NaN at a pixel whose taps are all out of view never reaches its coordinate
    gradient; this library's backward multiplies it by the zero value of such taps, so d/dM of that sample is NaN here and
    finite there.  Checked: NaN here wherever the reference is not finite, the same classes and values everywhere else."""
    H, W, dsize = 120, 256, (96, 200)
    src, M, cot = _backward_inputs(kind, 16, C, H, W, dsize, seed=C + 3 * stride1)
    well_conditioned = [b for b in range(4 if kind == "matrices" else M.shape[0]) if b != 7]

    def grads(mod, projective):
        s = src.clone().requires_grad_(True)
        mm = (M if projective else M[:, :2]).clone().requires_grad_(True)
        fn = mod.warp_perspective if projective else mod.warp_affine
        out = fn(s, mm, dsize, padding_mode=pad, align_corners=True)
        return torch.autograd.grad(out, [s, mm], grad_outputs=cot)

    K.config.set("bwd_stride1", stride1)
    for projective in (True, False):
        got = grads(K, projective)
        with K.config.override(tma=0):
            gen = grads(K, projective)
        _check_grads(got, gen, (projective, "tiled vs generic"), well_conditioned)
        want = reference(lambda: grads(R, projective))
        _check_grads(got, want, (projective, "vs reference"), well_conditioned, nan_superset=kind == "cotangent")


@pytest.mark.parametrize("kind", ["texels", "cotangent", "maps"])
def test_remap_backward_specials(kind):
    """d/dimage and d/dmap of remap (bilinear, zeros and border) against autograd of the reference on the same device.  d/dmap may
    be NaN where the reference's is finite, for the reason given in test_warp_backward_specials (never the other way round)."""
    H, W, h, w = 96, 160, 80, 136
    g = torch.Generator().manual_seed(21)
    img = (special_image(2, 3, H, W, seed=21, whole=False, huge=False) if kind == "texels" else torch.rand(2, 3, H, W, generator=g).to(DEV))
    cot = torch.rand(2, 3, h, w, generator=g).to(DEV) - 0.5
    if kind == "cotangent":
        cot = special_image(2, 3, h, w, seed=22, whole=False, huge=False) - 0.5
    if kind == "maps":
        mx, my = _special_maps(H, W, h, w, seed=3)
    else:
        ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float32), torch.arange(w, dtype=torch.float32), indexing="ij")
        mx, my = xs * (W / w) + 0.3 * torch.sin(ys) - 1.0, ys * (H / h) + 0.4 * torch.cos(xs) + 0.5
    mx, my = torch.stack([mx, mx + 0.25]).to(DEV), torch.stack([my, my - 0.5]).to(DEV)
    for pad in ("zeros", "border"):
        def grads(mod):
            i, ax, ay = img.clone().requires_grad_(True), mx.clone().requires_grad_(True), my.clone().requires_grad_(True)
            out = mod.remap(i, ax, ay, padding_mode=pad, align_corners=True)
            return torch.autograd.grad(out, [i, ax, ay], grad_outputs=cot)

        got = grads(K)
        want = reference(lambda: grads(R))
        assert classes_equal(got[0], want[0], atol=INF) and _rel_l2_finite(got[0], want[0]) < 1e-5, (pad, "d/dimage", diff(got[0], want[0]))
        for k in (1, 2):   # one coordinate, four taps per pixel: fp32 rounding apart
            fin = torch.isfinite(got[k])
            assert not (fin & ~torch.isfinite(want[k])).any(), (pad, "d/dmap", k, diff(got[k], want[k]))
            assert classes_equal(got[k], torch.where(fin, want[k], got[k]), rtol=1e-4, atol=1e-4), (pad, "d/dmap", k, diff(got[k], want[k]))


# ------------------------------------------------------------------------------------------ filters and fused kernels
# Against the reference the images carry no 3e38 texels: the generic kernels and ATen's convolution sum the taps in different
# orders, and whether a partial sum of texels near FLT_MAX overflows depends on that order (the tiled kernels are held to the
# generic ones bit for bit WITH such texels in the bit-identity tests of test_parity_gpu.py / test_variants_gpu.py).
BORDERS = ["constant", "reflect", "replicate", "circular"]
FILTER_SHAPES = [(4, 3, 70, 200), (5, 1, 45, 132)]


def _filter_check(got, want, what):
    assert got.shape == want.shape, what
    assert classes_equal(got, want, **FP32), (what, diff(got, want))


@pytest.mark.parametrize("border", BORDERS)
def test_filter2d_special_texels(border):
    """filter2d at K 3 / 5 / 7 (tiled kernel, generic under 'circular'), an even and a non-square kernel and 'valid' padding
    (generic), shared and per-sample kernels, against the same-device reference."""
    g = torch.Generator().manual_seed(3)
    for shape in FILTER_SHAPES:
        x = special_image(*shape, seed=shape[0], huge=False)
        B = shape[0]
        for kh, kw in ((3, 3), (5, 5), (7, 7), (4, 4), (3, 5)):
            for kern in (torch.randn(1, kh, kw, generator=g), torch.randn(B, kh, kw, generator=g)):
                kern = kern.to(DEV)
                for padding in ("same", "valid"):
                    got = K.filter2d(x, kern, border, padding=padding)
                    want = reference(lambda: R.filter2d(x, kern, border, padding=padding))
                    _filter_check(got, want, (shape, kh, kw, padding))


@pytest.mark.parametrize("border", BORDERS)
def test_separable_and_gaussian_special_texels(border):
    g = torch.Generator().manual_seed(5)
    for shape in FILTER_SHAPES:
        x = special_image(*shape, seed=10 + shape[0], huge=False)
        for k in range(3, 18, 2):
            kx, ky = torch.randn(shape[0], k, generator=g).to(DEV), torch.randn(1, k, generator=g).to(DEV)
            got = K.filter2d_separable(x, kx, ky, border)
            want = reference(lambda: R.filter2d_separable(x, kx, ky, border))
            _filter_check(got, want, ("separable", shape, k))
            got = K.gaussian_blur2d(x, (k, k), (1.7, 0.9), border)
            want = reference(lambda: R.gaussian_blur2d(x, (k, k), (1.7, 0.9), border))
            _filter_check(got, want, ("gaussian", shape, k))


@pytest.mark.parametrize("border", BORDERS)
def test_filter_family_special_texels(border):
    """box_blur, laplacian and unsharp_mask (blur + lerp in the blur kernel's epilogue) with every border."""
    for shape in FILTER_SHAPES:
        x = special_image(*shape, seed=20 + shape[0], huge=False)
        for ks in (3, 5):
            _filter_check(K.filters.box_blur(x, (ks, ks), border), reference(lambda: R.box_blur(x, (ks, ks), border)), ("box", shape, ks))
            _filter_check(K.filters.laplacian(x, ks, border), reference(lambda: R.laplacian(x, ks, border)), ("laplacian", shape, ks))
        for ks in (3, 5, 7, 11):
            got = K.filters.unsharp_mask(x, (ks, ks), (1.3, 1.7), border)
            want = reference(lambda: R.unsharp_mask(x, (ks, ks), (1.3, 1.7), border))
            _filter_check(got, want, ("unsharp", shape, ks))


def test_gradients_pyramid_ssim_undistort_special_texels():
    """spatial_gradient (sobel / diff, order 1 / 2) and the sobel magnitude, pyrdown (the fused 5x5 + 2x decimation), ssim and
    ssim_loss (the band-walking kernel), and the fused undistort_image."""
    for shape in ((4, 3, 70, 200), (5, 1, 64, 132)):
        x = special_image(*shape, seed=30 + shape[0], huge=False)
        for mode in ("sobel", "diff"):
            for order in (1, 2):
                for normalized in (True, False):
                    got = K.filters.spatial_gradient(x, mode, order, normalized)
                    want = reference(lambda: R.spatial_gradient(x, mode, order, normalized))
                    _filter_check(got, want, ("spatial_gradient", shape, mode, order, normalized))
        _filter_check(K.filters.sobel(x), reference(lambda: R.sobel(x)), ("sobel", shape))
        for border in ("reflect", "replicate", "constant"):
            _filter_check(K.geometry.transform.pyrdown(x, border), reference(lambda: R.pyrdown(x, border)), ("pyrdown", shape, border))
        y = special_image(*shape, seed=40 + shape[0], huge=False)
        for window in (3, 7, 11):
            _filter_check(K.metrics.ssim(x, y, window), reference(lambda: R.ssim(x, y, window)), ("ssim", shape, window))
            got = K.losses.ssim_loss(x, y, window, reduction="none")
            _filter_check(got, reference(lambda: R.ssim_loss(x, y, window, reduction="none")), ("ssim_loss", shape, window))
        B, C, H, W = shape
        cam = torch.tensor([[0.8 * W, 0.0, 0.5 * W - 3.0], [0.0, 0.75 * W, 0.5 * H + 2.0], [0.0, 0.0, 1.0]], device=DEV).expand(B, 3, 3).contiguous()
        dist = torch.tensor([-0.2, 0.05, 0.001, -0.002, 0.01], device=DEV).expand(B, 5).contiguous()
        before = K._ops.launch_count
        got = K.geometry.calibration.undistort_image(x, cam, dist)
        assert K._ops.launch_count == before + 1, "the fused kernel did not run"
        _filter_check(got, reference(lambda: R.undistort_image(x, cam, dist)), ("undistort", shape))


def test_comparators():
    """The comparators themselves: -0 != +0 for bits_equal, any NaN equals any NaN, classes before tolerance."""
    z = torch.zeros(4, device=DEV)
    assert not bits_equal(z, -z) and torch.equal(z, -z)
    odd_nan = torch.tensor([SENTINEL[torch.float32]], dtype=torch.int32, device=DEV).view(torch.float32)
    assert bits_equal(odd_nan, torch.tensor([NAN], device=DEV))
    assert classes_equal(torch.tensor([1.0, INF, NAN], device=DEV), torch.tensor([1.0 + 1e-7, INF, NAN], device=DEV), rtol=1e-6)
    assert not classes_equal(torch.tensor([INF], device=DEV), torch.tensor([NAN], device=DEV), atol=INF)
    assert not classes_equal(torch.tensor([3e38], device=DEV), torch.tensor([INF], device=DEV), atol=INF)
    assert unwritten(sentinel_like((3,))) == 3 and math.isnan(float(sentinel_like((1,))[0]))
