"""Gradients of the warp and remap kernels against float64, element by element, at real image sizes.

The ops are called below the prelude (``_ops.warp(src, m, bx, by, ...)`` with ``m`` an autograd leaf, ``_ops.remap`` with the
maps as leaves), so d/dm is the warp kernel's own output.

Coordinate replica.  ``replica`` recomputes, in the op's dtype and in the kernels' op order, the sampling coordinate of every
output pixel: ``nx = (m00 bx + m01 by) + m02`` (likewise ``ny``, ``den``), ``gx = nx / den`` (IEEE), the unnormalisation
(``warp_tma.cuh:unnorm``, ``sampler.cuh:unnormalize``; with align_corners=False ``(g + 1) size - 1`` is ONE FMA), the padded
coordinate with its derivative factor (``pad_coord_grad``: border clamp, reflection sign) and, for remap, ``coord_of``'s
``fx = 2 / max(W - 1, 1e-8)`` chain.  A float64 coordinate would differ from the kernel's by about u |ix| and pick another
floor cell now and then; taking the replica's values as exact leaves only the kernels' rounding to bound.  Every GPU test
first checks the replica: the float64 forward built from it must match the kernel's forward within ``FWD_ROUNDINGS u
sum|w v|`` element by element (one ulp of coordinate at |ix| ~ 1000 misses that by orders of magnitude).

Reference and bound, float64 from the replica's values: ``ref`` is d/dsrc by ``index_add_`` of ``w g`` and d/dm by
``ax = gix ux px / den``, ``az = -(ax gx + ay gy)`` and the nine products with ``bx`` / ``by``; ``A`` is the same with every
operand replaced by its absolute value and every difference by a sum; ``n_t`` counts the (pixel, tap) contributions landing on
element t.  The criteria (u = 2^-24; fp64: u = 2^-53 and twice the bound, since the reference rounds as often as the kernel):

  bilinear d/dsrc  |got - ref| <= (C_W + n_t) u A_t + tiny
  d/dm             |got - ref| <= u |ref| + (c_pix + L) u A + tiny      (Bm = 1: A summed over the batch)
  nearest          d/dsrc <= n_t u sum|g|; d/dm and d/dmap exactly 0
  remap d/dmap     |got - ref| <= c_pix u A_p + tiny  (+ the batch sum when Bmap = 1 < B)
  bicubic          the same, plus the a-priori error of the fp32 weight polynomials (``CUBIC_ROUNDINGS u P_abs(t)``)

with the constants derived below next to their definitions.  Entries whose float64 ``ref`` is not finite are skipped
(non-finite classes are tests/test_nonfinite_gpu.py's).  The report printed at teardown gives, per group, the largest
|got - ref| / (u (A + CUBIC_ROUNDINGS E)), E being the weight-polynomial term (0 except for bicubic).

Cost: on an H100 80GB HBM3 (700 W power limit) the GPU tests of this file take about 60 s; the longest is the run-time deal
at 400x3x96x192 (about 4 s, most of it the per-sample float64 reference loop), 48x3x720x1280 takes about 1 s.
"""
import math

import pytest
import torch
import torch.nn.functional as F

import kornia_b200 as K
from kornia_b200 import _lib, _ops
from kornia_b200.geometry import _prelude as P
from oracle import kornia_restated as R
from test_grad_bounds_gpu import REPORT, _assert_within, _report, _tiny, _unit, check_composed  # noqa: F401 (_report: teardown)
from test_parity_gpu import _bench_homographies, _shift_matrices, _wild_matrices

U64 = 2.0 ** -53
gpu = pytest.mark.gpu

# d/dsrc of a bilinear tap: wx = (x0 + 1) - ix and ix - x0 are exact unless |ix| < 1 (one rounding each axis), then
# w = wx wy and w g: 2 + 2 roundings before the value enters the accumulation chain of its element.
C_W = 4
# the forward: the same weights (4 roundings) and a chain of four FMAs (4); bicubic adds its weight error below
FWD_ROUNDINGS = 8
# fp32 cubic_weights / cubic_weights_grad at t in [0, 1): three Horner steps, each a multiply and an add when nvcc does not
# contract them (6; one FMA each when it does, 3), plus the rounded argument (t + 1, 1 - t, ...; and t = ix - floor(ix) itself
# below |ix| < 1): two relative errors in x, amplified by at most the degree (3) -> 6.  12 u P_abs(t) in all, where P_abs is
# the polynomial evaluated on absolute coefficients.
CUBIC_ROUNDINGS = 12
BWD_DYN_CHUNK = 10  # warp_bwd_tma.cuh: tiles per chunk of the run-time deal
GEN_BY = 8          # warp_generic.cuh: rows of a generic block, summed in fp32 after the warp shuffle


def c_pix(interp, C):
    """Roundings on the longest per-pixel chain from the taps to one of the nine d/dm products (or to d/dmap).

    bilinear, tiled fast path: s_tap = C FMAs over the channels; s_ne - s_nw, times wy1, plus the other row: 3; the weight wy
    itself when |iy| < 1: 1; times ux: 1; times rden, whose refined reciprocal is within 1 ulp of 1/den: 1 + 2; times bx / by: 1;
    az = -(ax gx + ay gy) adds a product and a sum: 2.  -> C + 11.  The exact path (bwd_pixel_global) and the generic kernel
    form gix per channel (v - fill: 1, difference, product, sum: 3, times go: 1, accumulated over channels: C) -> C + 5 before
    ux, the same tail (1 + 3 + 1 + 2) -> C + 12.  Remap: the same gix, then ux, fx and fx's own rounding -> C + 8.  So C + 12.
    bicubic (generic): each term (v - fill) dx_j cy_i go: 1 + 3; accumulated over 16 C taps; then ux, rden (IEEE: 1 + 1), bx,
    az (2) -> 16 C + 10; 16 C + 12 with the rounded t."""
    return 16 * C + 12 if interp == "bicubic" else C + 12


def run_length(w):
    """L: the longest fp32 run of d/dm partials before the double stage.  Tiled kernel, static deal: a lane sums its two
    columns of four rows of every tile of a strip segment, 8 ceil(w / 64) terms, then a 5-step shuffle tree; run-time deal:
    8 BWD_DYN_CHUNK + 5; generic kernel: the 5-step warp shuffle, then GEN_BY row partials.  The largest of the three."""
    return max(8 * math.ceil(w / 64), 8 * BWD_DYN_CHUNK) + 5


# ---------------------------------------------------------------------------------------------------------------------
# the coordinate replica (op's dtype, the kernels' op order)
# ---------------------------------------------------------------------------------------------------------------------
def _fma(a, b, c):
    """fl(a b + c) with one rounding, a a tensor, b and c small integers."""
    if a.dtype == torch.float32:
        return (a.double() * b + c).float()  # exact in fp64 while the product fits 53 bits; then one rounding
    # fp64: error-free product (Veltkamp split) and sum, then one final rounding
    p = a * b
    sp = 134217729.0
    t = sp * a
    ah = t - (t - a)
    al = a - ah
    e = ((ah * b - p) + al * b)
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)
    return s + (err + e)


def unnorm(g, size, align):
    if align:
        return ((g + 1) * 0.5) * (size - 1)
    return _fma(g + 1, size, -1) * 0.5


def _reflect(c, size, align):
    """reflect_coord (sampler.cuh) in c's dtype: (coordinate, sign of d out / d in)."""
    tl, th = (0, 2 * (size - 1)) if align else (-1, 2 * size - 1)
    if tl == th:
        return torch.zeros_like(c), torch.zeros_like(c)
    lo, span = tl * 0.5, (th - tl) * 0.5
    c = c - lo
    sgn = torch.where(c < 0, -1.0, 1.0).to(c.dtype)
    c = c.abs()
    extra = torch.fmod(c, span)
    # static_cast<int>(floor(c / span)): the conversion saturates at INT_MAX (odd) and takes NaN to 0 (even)
    # a tensor divisor: ATen's CUDA division by a Python scalar multiplies by its reciprocal, which is not R::div
    flips = torch.floor(c / torch.full_like(c, span)).double().clamp(max=2147483647.0)
    even = (torch.remainder(flips, 2) == 0) | torch.isnan(flips)
    out = torch.where(even, extra + lo, (span - extra) + lo)
    return out, torch.where(even, sgn, -sgn)


def pad_grad(c, size, align, pad):
    """pad_coord_grad: the padded coordinate and d(padded)/d(coordinate), then guard_index."""
    g = torch.ones_like(c)
    if pad == "reflection":
        c, g = _reflect(c, size, align)
    if pad in ("border", "reflection"):
        lo, hi = c <= 0, c >= size - 1
        g = torch.where(lo | hi, 0.0, g).to(c.dtype)
        c = torch.where(lo, 0.0, torch.where(hi, float(size - 1), c)).to(c.dtype)
    return _guard(c), g


def pad_plain(c, size, align, pad):
    """pad_coord: the clip of 'border', reflect + clip of 'reflection', then guard_index."""
    if pad == "reflection":
        c, _ = _reflect(c, size, align)
    if pad in ("border", "reflection"):
        c = torch.fmin(torch.fmax(c, torch.zeros_like(c)), torch.full_like(c, size - 1))  # fmax(NaN, 0) = 0, as clip_coord
    return _guard(c)


def _guard(c):
    return torch.where(c.abs() <= 2147483648.0, c, torch.full_like(c, -100.0))


def replica(m, bx, by, H, W, projective, align, fma=True):
    """(gx, gy, den, ix, iy) of one sample in m's dtype: (h, w) each.  ``fma=False`` rounds the unnormalisation's product
    separately (a deliberately wrong replica for the self-tests)."""
    X, Y = bx[None, :], by[:, None]
    nx = (m[0] * X + m[1] * Y) + m[2]
    ny = (m[3] * X + m[4] * Y) + m[5]
    if projective:
        den = (m[6] * X + m[7] * Y) + m[8]
        gx, gy = nx / den, ny / den
    else:
        den = torch.ones_like(nx)
        gx, gy = nx, ny
    if fma or align:
        ix, iy = unnorm(gx, W, align), unnorm(gy, H, align)
    else:
        ix, iy = ((gx + 1) * W - 1) * 0.5, ((gy + 1) * H - 1) * 0.5
    return gx, gy, den, ix, iy


def remap_replica(mx, my, H, W, normalized):
    """coord_of<KIND_REMAP>: (gx, gy, fx, fy) in the maps' dtype."""
    dt = mx.dtype
    if normalized:
        return mx, my, 1.0, 1.0
    fx = float(torch.tensor(2.0, dtype=dt) / torch.clamp(torch.tensor(float(W - 1), dtype=dt), min=torch.tensor(1e-8, dtype=dt)))
    fy = float(torch.tensor(2.0, dtype=dt) / torch.clamp(torch.tensor(float(H - 1), dtype=dt), min=torch.tensor(1e-8, dtype=dt)))
    return mx * torch.tensor(fx, dtype=dt, device=mx.device) - 1, my * torch.tensor(fy, dtype=dt, device=my.device) - 1, fx, fy


# ---------------------------------------------------------------------------------------------------------------------
# float64 reference and bound of one sample
# ---------------------------------------------------------------------------------------------------------------------
def _cubic(t):
    """cubic_weights and cubic_weights_grad in fp64 (exact polynomials) and their P_abs."""
    A = -0.75
    x0, u, x3 = t + 1, 1 - t, 2 - t
    w = [((A * x0 - 5 * A) * x0 + 8 * A) * x0 - 4 * A, ((A + 2) * t - (A + 3)) * t * t + 1,
         ((A + 2) * u - (A + 3)) * u * u + 1, ((A * x3 - 5 * A) * x3 + 8 * A) * x3 - 4 * A]
    wa = [((0.75 * x0 + 3.75) * x0 + 6) * x0 + 3, (1.25 * t + 2.25) * t * t + 1, (1.25 * u + 2.25) * u * u + 1,
          ((0.75 * x3 + 3.75) * x3 + 6) * x3 + 3]
    xs = [-1 - t, -t, 1 - t, 2 - t]
    d = [(-3 * A * xs[0] - 10 * A) * xs[0] - 8 * A, (-3 * (A + 2) * xs[1] - 2 * (A + 3)) * xs[1],
         (3 * (A + 2) * xs[2] - 2 * (A + 3)) * xs[2], (3 * A * xs[3] - 10 * A) * xs[3] + 8 * A]
    da = [(2.25 * xs[0].abs() + 7.5) * xs[0].abs() + 6, (3.75 * xs[1].abs() + 4.5) * xs[1].abs(),
          (3.75 * xs[2].abs() + 4.5) * xs[2].abs(), (2.25 * xs[3].abs() + 7.5) * xs[3].abs() + 6]
    return w, wa, d, da


def _taps(ix, iy, H, W, interp, pad, align, forward=False):
    """Taps of every pixel: list of (flat index, valid, (wx, wy), (wa_x, wa_y), (dx, dy), (da_x, da_y)) in fp64, and the
    padding factors (px, py) of the bilinear coordinate.  ``forward``: the bicubic column taps as the forward spells them."""
    one = torch.ones_like(ix, dtype=torch.float64)
    zero = torch.zeros_like(one)
    if interp == "bilinear":
        spad = "zeros" if pad == "fill" else pad
        cx, px = pad_grad(ix, W, align, spad)
        cy, py = pad_grad(iy, H, align, spad)
        cx, cy = cx.double(), cy.double()
        x0, y0 = torch.floor(cx), torch.floor(cy)
        fx, fy = cx - x0, cy - y0
        taps = []
        for dy, wy, sy in ((0, 1 - fy, -1.0), (1, fy, 1.0)):
            for dx, wx, sx in ((0, 1 - fx, -1.0), (1, fx, 1.0)):
                xi, yi = x0 + dx, y0 + dy
                ok = (xi >= 0) & (xi < W) & (yi >= 0) & (yi < H)
                idx = (yi.clamp(0, H - 1) * W + xi.clamp(0, W - 1)).long()
                # d w / d ix = sx wy, d w / d iy = sy wx; no weight polynomial error
                taps.append((idx, ok, (wx, wy), (zero, zero), (sx * one, sy * one), (zero, zero)))
        return taps, px.double(), py.double()
    if interp == "nearest":
        spad = "zeros" if pad == "fill" else pad
        cx, cy = pad_plain(ix, W, align, spad), pad_plain(iy, H, align, spad)
        xi, yi = torch.round(cx).double(), torch.round(cy).double()  # rint: half to even
        ok = (xi >= 0) & (xi < W) & (yi >= 0) & (yi < H)
        idx = (yi.clamp(0, H - 1) * W + xi.clamp(0, W - 1)).long()
        return [(idx, ok, (one, one), (zero, zero), (zero, zero), (zero, zero))], zero, zero
    # bicubic: the coordinate stays un-padded, every tap is padded on its own
    spad = "zeros" if pad == "fill" else pad
    fx, fy = torch.floor(ix), torch.floor(iy)
    tx, ty = (ix - fx).double(), (iy - fy).double()
    wxs, waxs, dxs, daxs = _cubic(tx)
    wys, ways, dys, days = _cubic(ty)
    # The tap columns as PixelSampler::prepare spells them, fx + (i - 1), or as warp_bwd_generic does, (fx - 1) + i: the same
    # values below 2^24, not above.  The padded tap is then truncated to int.  Under 'reflection' with align_corners=False it
    # need not be an integer: fx - 1 + i - (-0.5) rounds for |fx| >= 2^23, and the fold returns a half-integer.
    xi = [torch.trunc(pad_plain(fx + (i - 1) if forward else (fx - 1) + i, W, align, spad)).double() for i in range(4)]
    yi = [torch.trunc(pad_plain((fy - 1) + i, H, align, spad)).double() for i in range(4)]
    taps = []
    for i in range(4):
        for j in range(4):
            ok = (xi[j] >= 0) & (xi[j] < W) & (yi[i] >= 0) & (yi[i] < H)
            idx = (yi[i].clamp(0, H - 1) * W + xi[j].clamp(0, W - 1)).long()
            taps.append((idx, ok, (wxs[j], wys[i]), (waxs[j], ways[i]), (dxs[j], dys[i]), (daxs[j], days[i])))
    return taps, one, one


def sample_reference(src, go, coords, interp, pad, align, fill, dtype):
    """float64 reference of one sample: src (C, H, W), go (C, h, w) (or None), coords = (gx, gy, den, ix, iy) from the replica.

    Returns a dict: fwd / fwd_A (the forward and sum|w v|, plus the weight-error bound), gsrc / gsrc_A / gsrc_E / n (C, H, W),
    and per pixel gix, giy with their abs-chain A and weight-error E, and the padding factors."""
    C, H, W = src.shape
    gx, gy, den, ix, iy = coords
    taps, px, py = _taps(ix, iy, H, W, interp, pad, align)
    ftaps = _taps(ix, iy, H, W, interp, pad, align, forward=True)[0] if interp == "bicubic" else taps
    s = src.detach().double().reshape(C, H * W)
    f = fill.detach().double().reshape(C, 1, 1) if (pad == "fill" and fill is not None) else torch.zeros(C, 1, 1, dtype=torch.float64, device=s.device)
    h, w = ix.shape
    q = CUBIC_ROUNDINGS * _unit(dtype)  # relative size of the second-order term of two erroneous cubic weights
    out = {"px": px, "py": py}
    fwd = torch.zeros(C, h, w, dtype=torch.float64, device=s.device)
    fwd_A = torch.zeros_like(fwd)
    cover = torch.zeros(h, w, dtype=torch.float64, device=s.device)
    cover_A = torch.zeros_like(cover)
    for idx, ok, (wx, wy), (wax, way), _, _ in ftaps:
        v = torch.where(ok, s[:, idx], 0.0)
        wt = wx * wy
        werr = CUBIC_ROUNDINGS * (wax * wy.abs() + wx.abs() * way + q * wax * way) if interp == "bicubic" else 0.0  # in units of u
        fwd += wt * v
        fwd_A += (wt.abs() + werr / FWD_ROUNDINGS) * v.abs()
        cover += torch.where(ok, wt, 0.0)
        cover_A += torch.where(ok, wt.abs() + werr / FWD_ROUNDINGS, 0.0)
    if pad == "fill":
        fwd += (1 - cover) * f
        fwd_A += (1 + cover_A) * f.abs() * 2
    # a non-finite coordinate is padded differently by the forward (fmin / fmax) and the backward (comparisons): a
    # non-finite class, left to test_nonfinite_gpu.py
    fwd = torch.where(torch.isfinite(ix) & torch.isfinite(iy), fwd, math.nan)
    out["fwd"], out["fwd_A"] = fwd, fwd_A
    if go is None:
        return out
    g = go.detach().double()
    gsrc = torch.zeros(C, H * W, dtype=torch.float64, device=s.device)
    gA, gE = torch.zeros_like(gsrc), torch.zeros_like(gsrc)
    n = torch.zeros(H * W, dtype=torch.float64, device=s.device)
    gix, giy = torch.zeros(h, w, dtype=torch.float64, device=s.device), torch.zeros(h, w, dtype=torch.float64, device=s.device)
    Ax, Ay, Ex, Ey = (torch.zeros_like(gix) for _ in range(4))
    for idx, ok, (wx, wy), (wax, way), (dx, dy), (dax, day) in taps:
        sel = ok.flatten()
        fi = idx.flatten()[sel]
        wt = (wx * wy).flatten()[sel]
        gf = g.reshape(C, -1)[:, sel]
        gsrc.index_add_(1, fi, wt * gf)
        gA.index_add_(1, fi, wt.abs() * gf.abs())
        n.index_add_(0, fi, torch.ones_like(wt))
        if interp == "bicubic":
            gE.index_add_(1, fi, ((wax * wy.abs() + wx.abs() * way + q * wax * way).flatten()[sel]) * gf.abs())
        if interp == "nearest":
            continue
        v = torch.where(ok, s[:, idx] - f, 0.0)
        va = torch.where(ok, s[:, idx].abs() + f.abs(), 0.0)
        # d out / d ix of this tap: dx * wy (bilinear: dx = +-1; bicubic: the cubic derivative, with the minus sign of the
        # generic kernel's `gix -= v dx cy go` folded into the -t argument convention of cubic_weights_grad)
        sgn = -1.0 if interp == "bicubic" else 1.0
        gix += sgn * (g * v * (dx * wy)).sum(0)
        giy += sgn * (g * v * (dy * wx)).sum(0)
        Ax += (g.abs() * va * (dx.abs() * wy.abs())).sum(0)
        Ay += (g.abs() * va * (dy.abs() * wx.abs())).sum(0)
        if interp == "bicubic":
            Ex += (g.abs() * va * (dax * wy.abs() + dx.abs() * way + q * dax * way)).sum(0)
            Ey += (g.abs() * va * (day * wx.abs() + dy.abs() * wax + q * day * wax)).sum(0)
    out.update(gsrc=gsrc.reshape(C, H, W), gsrc_A=gA.reshape(C, H, W), gsrc_E=gE.reshape(C, H, W), n=n.reshape(1, H, W),
               gix=gix, giy=giy, Ax=Ax, Ay=Ay, Ex=Ex, Ey=Ey)
    return out


def dm_terms(r, coords, bx, by, H, W, align, projective):
    """The nine d/dm entries of one sample (fp64): (ref, A, E) each (9,)."""
    gx, gy, den, _, _ = (t.double() for t in coords)
    ux = (W - 1) * 0.5 if align else W * 0.5
    uy = (H - 1) * 0.5 if align else H * 0.5
    rden = 1.0 / den if projective else torch.ones_like(den)
    X, Y = bx.double()[None, :].expand_as(gx), by.double()[:, None].expand_as(gx)
    res = []
    for gxk, gyk, absolute in ((r["gix"], r["giy"], False), (r["Ax"], r["Ay"], True), (r["Ex"], r["Ey"], True)):
        pxk, pyk, rd, gxx, gyy, XX, YY = r["px"], r["py"], rden, gx, gy, X, Y
        if absolute:
            pxk, pyk, rd, gxx, gyy, XX, YY = (t.abs() for t in (pxk, pyk, rd, gxx, gyy, XX, YY))
        ax, ay = gxk * ux * pxk * rd, gyk * uy * pyk * rd
        if projective:
            az = (ax * gxx + ay * gyy) if absolute else -(ax * gxx + ay * gyy)
        else:
            az = torch.zeros_like(ax)
        res.append(torch.stack([(ax * XX).sum(), (ax * YY).sum(), ax.sum(), (ay * XX).sum(), (ay * YY).sum(), ay.sum(),
                                (az * XX).sum(), (az * YY).sum(), az.sum()]))
    return res


# ---------------------------------------------------------------------------------------------------------------------
# criteria
# ---------------------------------------------------------------------------------------------------------------------
def _finite(ref, *others):
    keep = torch.isfinite(ref)
    return [torch.where(keep, t.double() if t.dtype != torch.float64 else t, 0.0) for t in (ref,) + others]


def check_forward(group, what, got, r, dtype):
    """The replica self-check: the kernel's forward against the float64 forward from the replica's coordinates."""
    u = _unit(dtype)
    k = 2 if dtype == torch.float64 else 1
    ref, got_, A = _finite(r["fwd"], got, r["fwd_A"])
    _assert_within(f"{group} forward (replica check)", what + " forward", got_, ref, k * FWD_ROUNDINGS * u * A + _tiny(dtype), u, A)


def check_gsrc(group, what, got, r, interp, dtype):
    u = _unit(dtype)
    k = 2 if dtype == torch.float64 else 1
    ref, got_, A, E, n = _finite(r["gsrc"], got, r["gsrc_A"], r["gsrc_E"], r["n"].expand_as(r["gsrc"]))
    cw = 0 if interp == "nearest" else C_W
    allowed = k * ((cw + n) * u * A + CUBIC_ROUNDINGS * u * E) + n * U64 * A + _tiny(dtype)
    _assert_within(f"{group} d/dsrc {dtype}", what + " d/dsrc", got_, ref, allowed, u, A + CUBIC_ROUNDINGS * E)


def check_dm(group, what, got, ref, A, E, interp, C, w, dtype):
    """|got - ref| <= u |ref| + (c_pix + L) u A (+ the cubic weight error) + tiny; nearest: exactly 0."""
    u = _unit(dtype)
    k = 2 if dtype == torch.float64 else 1
    ref, got_, A, E = _finite(ref, got, A, E)
    if interp == "nearest":
        allowed = torch.zeros_like(ref)
    else:
        allowed = k * (u * ref.abs() + (c_pix(interp, C) + run_length(w)) * u * A + CUBIC_ROUNDINGS * u * E) + _tiny(dtype)
    _assert_within(f"{group} d/dm {dtype}", what + " d/dm", got_, ref, allowed, u, A + CUBIC_ROUNDINGS * E)


# ---------------------------------------------------------------------------------------------------------------------
# the warp below the prelude
# ---------------------------------------------------------------------------------------------------------------------
def sampling(M, src_hw, dsize, projective, align, dtype):
    """(m, bx, by) as imgwarp.py builds them."""
    h, w = dsize
    Mm = M if projective else M[:, :2, :].contiguous()
    m = P.sampling_matrix(Mm.to(dtype), src_hw, dsize, affine=not projective).contiguous()
    if projective:
        bx, by = P.meshgrid_axes(h, w, M.device, dtype)
    else:
        bx, by = P.affine_axes(h, w, align, M.device, dtype)
    return m.detach(), bx.contiguous(), by.contiguous()


INTERP_CODE = {"bilinear": _lib.BILINEAR, "nearest": _lib.NEAREST, "bicubic": _lib.BICUBIC}


def run_warp(src, m, bx, by, fill, dsize, projective, interp, pad, align, need, go):
    """Forward and the requested gradients of _ops.warp (need: 'both', 'src' or 'm')."""
    h, w = dsize
    s = src.detach().clone().requires_grad_(need in ("both", "src"))
    mm = m.detach().clone().requires_grad_(need in ("both", "m"))
    out = _ops.warp(s, mm, bx, by, fill, h, w, projective, INTERP_CODE[interp], _lib.PADDING[pad], align)
    leaves = [t for t in (s, mm) if t.requires_grad]
    grads = torch.autograd.grad(out, leaves, go)
    gs = grads[0] if s.requires_grad else None
    gm = grads[-1] if mm.requires_grad else None
    return out.detach(), gs, gm


def warp_references(src, m, bx, by, fill, go, dsize, projective, interp, pad, align):
    """Per-sample float64 references (looped per sample to bound memory).  m (Bm, 3, 3); Bm = 1 sums d/dm over the batch."""
    B, C, H, W = src.shape
    dtype = src.dtype
    Bm = m.shape[0]
    fwd, gsrc = [], []
    dm = torch.zeros(Bm, 3, 9, dtype=torch.float64, device=src.device)
    for b in range(B):
        mb = m[b if Bm > 1 else 0].reshape(9)
        coords = replica(mb, bx, by, H, W, projective, align)
        r = sample_reference(src[b], go[b], coords, interp, pad, align, fill, dtype)
        fwd.append(r)
        gsrc.append({k: r[k] for k in ("gsrc", "gsrc_A", "gsrc_E", "n")})
        for k, t in enumerate(dm_terms(r, coords, bx, by, H, W, align, projective)):
            dm[b if Bm > 1 else 0, k] += t
        for key in ("gsrc", "gsrc_A", "gsrc_E", "n", "gix", "giy", "Ax", "Ay", "Ex", "Ey"):
            r.pop(key, None)
    return fwd, gsrc, dm


def check_warp(group, src, M, dsize, projective, interp, pad, align, needs=("both", "src", "m"), fill=None, options=({},),
               shared=False, seed=0):
    """Every gradient the kernel selected by each ``options`` override computes, against the float64 bounds."""
    B, C, H, W = src.shape
    dtype = src.dtype
    m, bx, by = sampling(M, (H, W), dsize, projective, align, dtype)
    if shared:
        m = m[:1].contiguous()
    g = torch.Generator(device=src.device).manual_seed(seed)
    go = (torch.rand(B, C, *dsize, generator=g, device=src.device, dtype=dtype) * 2 - 1)
    fwd, gs_ref, dm = warp_references(src, m, bx, by, fill, go, dsize, projective, interp, pad, align)
    what = f"{group} {interp} {pad} {'proj' if projective else 'affine'} align={align} {tuple(src.shape)}->{dsize} {dtype}"
    for opt in options:
        with K.config.override(**opt):
            for need in needs:
                out, gs, gm = run_warp(src, m, bx, by, fill, dsize, projective, interp, pad, align, need, go)
                tag = f"{what} {opt} need={need}"
                for b in range(B):
                    if need == "both":  # the replica's self-check, once per kernel
                        check_forward(group, f"{tag} sample {b}", out[b], fwd[b], dtype)
                    if gs is not None:
                        check_gsrc(group, f"{tag} sample {b}", gs[b], gs_ref[b], interp, dtype)
                if gm is not None:
                    check_dm(group, tag, gm.reshape(-1, 9), dm[:, 0], dm[:, 1], dm[:, 2], interp, C, dsize[1], dtype)


# ---------------------------------------------------------------------------------------------------------------------
# 1. CPU self-tests: a torch fp32 restatement of the kernel arithmetic passes; five mutations of it are rejected
# ---------------------------------------------------------------------------------------------------------------------
def _fma32(a, b, c):
    return (a.double() * b.double() + c.double()).float()


def restated_warp(src, go, m, bx, by, dsize, projective, pad, align, mutation=None, ctx=None):
    """warp_bwd_tma2's arithmetic in fp32 torch ops (bilinear, zeros / border): forward, d/dsrc and d/dm, d/dm summed in fp32
    over runs of 8 ceil(w / 64) consecutive pixel terms, then in double (the static deal's records)."""
    B, C, H, W = src.shape
    h, w = dsize
    ctx = {} if ctx is None else ctx
    out = torch.zeros(B, C, h, w)
    gsrc = torch.zeros(B, C, H * W)
    run = 8 * math.ceil(w / 64)
    nrun = math.ceil(h * w / run)
    runs = torch.zeros(B, nrun, 9)
    for b in range(B):
        gx, gy, den, ix, iy = replica(m[b].reshape(9), bx, by, H, W, projective, align)
        px, py = torch.ones_like(ix), torch.ones_like(iy)
        if pad == "border":
            ix, px = pad_grad(ix, W, align, "border")
            iy, py = pad_grad(iy, H, align, "border")
        ix, iy = _guard(ix), _guard(iy)
        if mutation == "px" and b == 0:
            px = px.clone()
            px.view(-1)[ctx["px_pixel"]] = 1.0
        x0f, y0f = torch.floor(ix), torch.floor(iy)
        wx1, wx0, wy1, wy0 = (x0f + 1) - ix, ix - x0f, (y0f + 1) - iy, iy - y0f
        x0, y0 = x0f.long(), y0f.long()
        s = src[b].reshape(C, -1)
        taps = {}
        for name, dy, dx, wt in (("nw", 0, 0, wx1 * wy1), ("ne", 0, 1, wx0 * wy1), ("sw", 1, 0, wx1 * wy0), ("se", 1, 1, wx0 * wy0)):
            yy, xx = y0 + dy, x0 + dx
            ok = (xx >= 0) & (xx < W) & (yy >= 0) & (yy < H)
            idx = (yy.clamp(0, H - 1) * W + xx.clamp(0, W - 1))
            taps[name] = (idx, ok, wt, torch.where(ok, s[:, idx], 0.0))
        acc = torch.zeros(C, h, w)
        for name in ("nw", "ne", "sw", "se"):
            _, ok, wt, v = taps[name]
            acc = torch.where(ok, _fma32(v, wt.expand_as(v), acc), acc)
        out[b] = acc
        for name in ("nw", "ne", "sw", "se"):
            idx, ok, wt, _ = taps[name]
            if mutation == "ne" and b == 0 and name == "ne":
                ok = ok.clone()
                ok.view(-1)[ctx["ne_pixel"]] = False
            sel = ok.flatten()
            gsrc[b].index_add_(1, idx.flatten()[sel], (wt * go[b]).reshape(C, -1)[:, sel])
        st = {}
        for name in ("nw", "ne", "sw", "se"):
            acc = torch.zeros(h, w)
            for c in range(C):
                acc = _fma32(go[b, c], taps[name][3][c], acc)
            st[name] = acc
        w1, w0 = wy1, wy0
        if mutation == "wy" and b == 0:
            r = ctx["wy_row"]
            w1, w0 = wy1.clone(), wy0.clone()
            w1[r], w0[r] = wy0[r], wy1[r]
        gix = (st["ne"] - st["nw"]) * w1 + (st["se"] - st["sw"]) * w0
        giy = (st["sw"] - st["nw"]) * wx1 + (st["se"] - st["ne"]) * wx0
        ux = (W - 1) * 0.5 if align else W * 0.5
        uy = (H - 1) * 0.5 if align else H * 0.5
        rden = 1 / den if projective else torch.ones_like(den)
        ax, ay = ((gix * ux) * px) * rden, ((giy * uy) * py) * rden
        X, Y = bx[None, :].expand(h, w), by[:, None].expand(h, w)
        az = -(ax * gx + ay * gy) if projective else torch.zeros_like(ax)
        terms = torch.stack([ax * X, ax * Y, ax, ay * X, ay * Y, ay, az * X, az * Y, az], -1).reshape(-1, 9)
        terms = torch.cat([terms, torch.zeros(nrun * run - h * w, 9)]).reshape(nrun, run, 9)
        part = torch.zeros(nrun, 9)
        for k in range(run):  # fp32, in order
            part = part + terms[:, k]
        runs[b] = part
    if mutation == "record":
        b0, r0 = ctx["record"]
        runs[b0 + 1, r0] += runs[b0, r0]
        runs[b0, r0] = 0
    gm = runs.double().sum(1).float().reshape(B, 3, 3)
    return out, gsrc.reshape(B, C, H, W), gm


def _cpu_case(seed=0, pad="border", align=False, projective=True):
    B, C, H, W, dsize = 2, 3, 40, 600, (24, 136)
    g = torch.Generator().manual_seed(seed)
    src = torch.rand(B, C, H, W, generator=g)
    go = torch.rand(B, C, *dsize, generator=g) * 2 - 1
    # sample 0 reaches past the left edge (border clamps), sample 1 stays inside
    M = torch.tensor([[[0.9, -0.2, 40.0], [0.15, 1.1, -6.0], [-3e-5, 2e-4, 1.0]],
                      [[1.03, 0.08, -9.0], [-0.05, 0.97, 3.0], [2e-5, -1e-4, 1.0]]])
    m, bx, by = sampling(M, (H, W), dsize, projective, align, torch.float32)
    return src, go, m, bx, by, dsize, projective, pad, align


def _check_restated(args, mutation=None, ctx=None, replica_fma=True):
    src, go, m, bx, by, dsize, projective, pad, align = args
    B, C, H, W = src.shape
    out, gs, gm = restated_warp(src, go, m, bx, by, dsize, projective, pad, align, mutation, ctx)
    dm = torch.zeros(B, 3, 9, dtype=torch.float64)
    for b in range(B):
        coords = replica(m[b].reshape(9), bx, by, H, W, projective, align, fma=replica_fma)
        r = sample_reference(src[b], go[b], coords, "bilinear", pad, align, None, torch.float32)
        check_forward("self-test", f"sample {b}", out[b], r, torch.float32)
        check_gsrc("self-test", f"sample {b}", gs[b], r, "bilinear", torch.float32)
        for k, t in enumerate(dm_terms(r, coords, bx, by, H, W, align, projective)):
            dm[b, k] = t
    check_dm("self-test", "restated", gm.reshape(-1, 9), dm[:, 0], dm[:, 1], dm[:, 2], "bilinear", C, dsize[1], torch.float32)
    return dm


@pytest.mark.parametrize("align", [True, False])
@pytest.mark.parametrize("pad", ["zeros", "border"])
@pytest.mark.parametrize("projective", [True, False], ids=["proj", "affine"])
def test_restated_kernel_arithmetic_passes(projective, pad, align):
    _check_restated(_cpu_case(1, pad, align, projective))


def _pixel_data(args):
    """Per-pixel coordinates of sample 0 of a self-test case (for choosing where to mutate)."""
    src, go, m, bx, by, dsize, projective, pad, align = args
    H, W = src.shape[-2:]
    gx, gy, den, ix, iy = replica(m[0].reshape(9), bx, by, H, W, projective, align)
    cx, px = pad_grad(ix, W, align, pad)
    cy, py = pad_grad(iy, H, align, pad)
    return cx, cy, px, py


def test_mutation_dropped_edge_tap_is_rejected():
    args = _cpu_case(2, "zeros")
    src, go = args[0], args[1]
    cx, cy, _, _ = _pixel_data(args)
    W, H = src.shape[-1], src.shape[-2]
    x0, y0 = torch.floor(cx), torch.floor(cy)
    fx = (cx - x0)
    # a pixel of the last output column whose NE tap lies in the image, with the largest NE weight times |g|
    ok = (x0 + 1 < W) & (x0 + 1 >= 0) & (y0 >= 0) & (y0 < H)
    score = torch.where(ok, fx * (1 - (cy - y0)) * go[0].abs().sum(0), -1.0)
    score[:, :-1] = -1.0
    pixel = int(score.flatten().argmax())
    assert float(score.flatten()[pixel]) > 0.05
    with pytest.raises(AssertionError, match="d/dsrc"):
        _check_restated(args, "ne", {"ne_pixel": pixel})


def test_mutation_swapped_row_weights_are_rejected():
    args = _cpu_case(3, "zeros")
    with pytest.raises(AssertionError, match="d/dm"):
        _check_restated(args, "wy", {"wy_row": 7})


def test_mutation_ignored_border_factor_is_rejected():
    args = _cpu_case(4, "border")
    src = args[0]
    cx, cy, px, py = _pixel_data(args)
    # a clamped pixel (px = 0) whose coordinate gradient would be large
    cand = (px == 0) & (py != 0)
    assert bool(cand.any())
    score = torch.where(cand, torch.rand(cand.shape, generator=torch.Generator().manual_seed(0)) + 1, 0.0)
    pixel = int(score.flatten().argmax())
    with pytest.raises(AssertionError, match="d/dm"):
        _check_restated(args, "px", {"px_pixel": pixel})


def test_mutation_record_booked_to_the_neighbouring_sample_is_rejected():
    args = _cpu_case(5, "zeros")
    src, go, m, bx, by, dsize, projective, pad, align = args
    # the run with the largest partial of sample 0
    run = 8 * math.ceil(dsize[1] / 64)
    H, W = src.shape[-2:]
    coords = replica(m[0].reshape(9), bx, by, H, W, projective, align)
    r = sample_reference(src[0], go[0], coords, "bilinear", pad, align, None, torch.float32)
    ux = (W - 1) * 0.5 if align else W * 0.5
    ax = (r["gix"] * ux * r["px"] / coords[2].double()).flatten()
    nrun = math.ceil(ax.numel() / run)
    part = torch.cat([ax, ax.new_zeros(nrun * run - ax.numel())]).reshape(nrun, run).sum(1)
    r0 = int(part.abs().argmax())
    with pytest.raises(AssertionError, match="d/dm"):
        _check_restated(args, "record", {"record": (0, r0)})


def test_mutation_replica_without_the_fma_is_caught_by_the_forward_check():
    args = _cpu_case(6, "zeros", align=False)
    _check_restated(args)
    with pytest.raises(AssertionError, match="forward"):
        _check_restated(args, replica_fma=False)


def test_fp64_fma_emulation():
    g = torch.Generator().manual_seed(0)
    a = (torch.rand(100000, generator=g, dtype=torch.float64) * 2 - 1) * torch.pow(2.0, torch.randint(-40, 3, (100000,), generator=g)).double()
    from fractions import Fraction
    got = _fma(a, 1279, -1)
    for i in range(0, 100000, 997):
        exact = Fraction(float(a[i])) * 1279 - 1
        assert float(got[i]) == float(exact), (float(a[i]), float(got[i]), float(exact))


# ---------------------------------------------------------------------------------------------------------------------
# 2. on the device
# ---------------------------------------------------------------------------------------------------------------------
DEV = "cuda"


def _matrices(H, W, B=None, seed=0):
    M = torch.cat([_wild_matrices(H, W), _shift_matrices(W), _bench_homographies(4, H, W, seed, sigma=6.0)])
    if B is not None:
        M = M[torch.arange(B) % M.shape[0]]
    return M.to(DEV)


def _src(shape, seed, dtype=torch.float32):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.rand(shape, generator=g, device=DEV, dtype=dtype)


TILED_SHAPES = {"120x256->96x200": (18, 120, 256, (96, 200)), "720p": (4, 720, 1280, (720, 1280))}


@gpu
@pytest.mark.parametrize("shape", list(TILED_SHAPES))
@pytest.mark.parametrize("align", [True, False])
@pytest.mark.parametrize("projective", [True, False], ids=["proj", "affine"])
@pytest.mark.parametrize("pad", ["zeros", "border"])
@pytest.mark.parametrize("C", [1, 3])
def test_tiled_backward(C, pad, projective, align, shape):
    B, H, W, dsize = TILED_SHAPES[shape]
    M = _matrices(H, W)
    if B < M.shape[0]:
        M = M[torch.tensor([1, 7, 14, 15])]  # 30 degrees, the horizon, two bench homographies
    src = _src((M.shape[0], C, H, W), C)
    _assert_tiled_backward(src, dsize, pad)
    check_warp("tiled", src, M, dsize, projective, "bilinear", pad, align,
               options=({"bwd_stride1": 1}, {"bwd_stride1": 0}))


def _assert_tiled_backward(src, dsize, pad):
    """warp_tma_backward's conditions (warp_bwd_tma.cu), so that a case meant for warp_bwd_tma2 cannot silently be served by
    the generic kernel: the tiled kernels on, fp32, bilinear (the callers' mode), zeros or border, C = 1 or 3, W and w
    multiples of 4, 16-byte aligned planes."""
    B, C, H, W = src.shape
    h, w = dsize
    assert K.config.get("tma") == 1, "the tiled kernels are switched off"
    assert src.dtype == torch.float32 and pad in ("zeros", "border") and C in (1, 3), (src.dtype, pad, C)
    assert W % 4 == 0 and w % 4 == 0, f"W = {W}, w = {w}: the tiled backward needs multiples of 4"
    assert src.data_ptr() % 16 == 0 and B * C < 2 ** 31, "the tiled backward needs 16-byte aligned planes"


def _assert_dynamic_deal(B, h):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    strips = B * math.ceil(h / 32)
    assert strips >= 8 * sms, f"{B}x{h}: {strips} strips < 8 x {sms} SMs: the run-time deal would not be taken"


@gpu
@pytest.mark.parametrize("B,H,W", [(400, 96, 192), (48, 720, 1280)], ids=["400x3x96x192", "48x3x720x1280"])
@pytest.mark.parametrize("projective", [True, False], ids=["proj", "affine"])
def test_run_time_deal(B, H, W, projective):
    """One chunk per strip (w = 192: 3 tiles) and two chunks per strip (w = 1280: 20 tiles), against the static deal."""
    _assert_dynamic_deal(B, H)
    M = _matrices(H, W, B, seed=B)
    src = _src((B, 3, H, W), B)
    _assert_tiled_backward(src, (H, W), "zeros")
    check_warp("run-time deal", src, M, (H, W), projective, "bilinear", "zeros", True, needs=("both",),
               options=({"dyn_sched": 1, "bwd_stride1": 1}, {"dyn_sched": 0}))


@gpu
@pytest.mark.parametrize("kernel", ["static", "run-time", "generic"])
def test_shared_affine_matrix(kernel):
    """One (1, 2, 3) matrix for the whole batch: d/dM is summed over the batch."""
    B, H, W = (400, 96, 192) if kernel == "run-time" else (6, 120, 256)
    if kernel == "run-time":
        _assert_dynamic_deal(B, H)
    opt = {"static": {"dyn_sched": 0}, "run-time": {"dyn_sched": 1, "bwd_stride1": 1}, "generic": {"tma": 0}}[kernel]
    M = _matrices(H, W)[1:2]
    src = _src((B, 3, H, W), 9)
    if kernel != "generic":
        _assert_tiled_backward(src, (H, W), "zeros")
    check_warp(f"shared matrix {kernel}", src, M.expand(B, 3, 3), (H, W), False, "bilinear", "zeros", True, options=(opt,), shared=True)


GENERIC = ({"tma": 0},)


@gpu
@pytest.mark.parametrize("align", [True, False])
@pytest.mark.parametrize("projective", [True, False], ids=["proj", "affine"])
@pytest.mark.parametrize("pad", ["zeros", "border", "reflection", "fill"])
def test_generic_bilinear(pad, projective, align):
    H, W, dsize = 120, 256, (96, 200)
    M = _matrices(H, W)
    src = _src((M.shape[0], 3, H, W), 3)
    fill = torch.tensor([0.2, -0.5, 0.8], device=DEV) if pad == "fill" else None
    check_warp("generic bilinear", src, M, dsize, projective, "bilinear", pad, align, fill=fill, options=GENERIC)


@gpu
def test_generic_bilinear_720p():
    M = _matrices(720, 1280)[torch.tensor([1, 7, 14, 15])]
    check_warp("generic bilinear", _src((4, 3, 720, 1280), 5), M, (720, 1280), True, "bilinear", "zeros", False, options=GENERIC)


@gpu
@pytest.mark.parametrize("align", [True, False])
@pytest.mark.parametrize("pad", ["zeros", "border", "reflection", "fill"])
@pytest.mark.parametrize("interp", ["bicubic", "nearest"])
def test_generic_bicubic_and_nearest(interp, pad, align):
    H, W, dsize = 120, 256, (96, 200)
    M = _matrices(H, W)
    src = _src((M.shape[0], 3, H, W), 4)
    fill = torch.tensor([0.2, -0.5, 0.8], device=DEV) if pad == "fill" else None
    for projective in (True, False):
        check_warp(f"generic {interp}", src, M, dsize, projective, interp, pad, align, fill=fill, options=GENERIC)


@gpu
@pytest.mark.parametrize("C,W", [(2, 256), (4, 256), (3, 250), (1, 131)])
def test_shapes_the_tiled_kernel_declines(C, W):
    H, dsize = 120, (96, 198)
    M = _matrices(H, W)
    src = _src((M.shape[0], C, H, W), C + W)
    for projective in (True, False):
        for pad in ("zeros", "border"):
            check_warp("declined shapes", src, M, dsize, projective, "bilinear", pad, True)


@gpu
@pytest.mark.parametrize("interp,pad", [("bilinear", "zeros"), ("bilinear", "border"), ("bilinear", "reflection"), ("bilinear", "fill"),
                                        ("bicubic", "zeros"), ("bicubic", "reflection"), ("nearest", "border")])
def test_generic_fp64(interp, pad):
    H, W, dsize = 40, 52, (30, 44)
    M = _matrices(H, W).double()
    src = _src((M.shape[0], 3, H, W), 8, torch.float64)
    fill = torch.tensor([0.2, -0.5, 0.8], device=DEV, dtype=torch.float64) if pad == "fill" else None
    for projective in (True, False):
        for align in (True, False):
            check_warp("fp64", src, M, dsize, projective, interp, pad, align, fill=fill)


# ---- remap ------------------------------------------------------------------------------------------------------------
def _maps(Bmap, h, w, H, W, normalized, seed, dtype=torch.float32):
    g = torch.Generator(device=DEV).manual_seed(seed)
    ys, xs = torch.meshgrid(torch.arange(h, device=DEV, dtype=torch.float64), torch.arange(w, device=DEV, dtype=torch.float64), indexing="ij")
    mx = torch.stack([(xs * (W / max(w, 1)) * (1 + 0.05 * b) + 6 * torch.sin(ys / 17 + b) - 3) for b in range(Bmap)])
    my = torch.stack([(ys * (H / max(h, 1)) * (1 - 0.04 * b) + 5 * torch.cos(xs / 23 - b) - 2) for b in range(Bmap)])
    mx = mx + 0.3 * torch.rand(mx.shape, generator=g, device=DEV, dtype=torch.float64)
    my = my + 0.3 * torch.rand(my.shape, generator=g, device=DEV, dtype=torch.float64)
    if normalized:
        mx, my = mx * (2 / (W - 1)) - 1, my * (2 / (H - 1)) - 1
    return mx.to(dtype).contiguous(), my.to(dtype).contiguous()


def check_remap(group, img, mx, my, interp, pad, align, normalized, seed=0):
    B, C, H, W = img.shape
    Bmap, h, w = mx.shape
    dtype = img.dtype
    u = _unit(dtype)
    k = 2 if dtype == torch.float64 else 1
    g = torch.Generator(device=DEV).manual_seed(seed)
    go = torch.rand(B, C, h, w, generator=g, device=DEV, dtype=dtype) * 2 - 1
    il, xl, yl = (t.detach().clone().requires_grad_(True) for t in (img, mx, my))
    out = _ops.remap(il, xl, yl, normalized, INTERP_CODE[interp], _lib.PADDING[pad], align)
    gi, gmx, gmy = torch.autograd.grad(out, (il, xl, yl), go)
    what = f"{group} {interp} {pad} align={align} normalized={normalized} {tuple(img.shape)} maps {tuple(mx.shape)} {dtype}"
    ref_x = torch.zeros(Bmap, h, w, dtype=torch.float64, device=DEV)
    ref_y, A_x, A_y, E_x, E_y = (torch.zeros_like(ref_x) for _ in range(5))
    ux = (W - 1) * 0.5 if align else W * 0.5
    uy = (H - 1) * 0.5 if align else H * 0.5
    for b in range(B):
        bm = b if Bmap > 1 else 0
        gx, gy, fx, fy = remap_replica(mx[bm], my[bm], H, W, normalized)
        ix, iy = unnorm(gx, W, align), unnorm(gy, H, align)
        r = sample_reference(img[b], go[b], (gx, gy, None, ix, iy), interp, pad, align, None, dtype)
        check_forward(group, f"{what} sample {b}", out[b].detach(), r, dtype)
        check_gsrc(group, f"{what} sample {b}", gi[b], r, interp, dtype)
        ref_x[bm] += r["gix"] * ux * r["px"] * fx
        ref_y[bm] += r["giy"] * uy * r["py"] * fy
        A_x[bm] += r["Ax"] * ux * r["px"].abs() * abs(fx)
        A_y[bm] += r["Ay"] * uy * r["py"].abs() * abs(fy)
        E_x[bm] += r["Ex"] * ux * abs(fx)
        E_y[bm] += r["Ey"] * uy * abs(fy)
    # Bmap = 1 < B: the per-sample map gradients are summed over the batch in the op's dtype (B - 1 more roundings)
    extra = B - 1 if Bmap == 1 else 0
    for name, got, ref, A, E in (("d/dmap_x", gmx, ref_x, A_x, E_x), ("d/dmap_y", gmy, ref_y, A_y, E_y)):
        ref, got_, A, E = _finite(ref, got, A, E)
        if interp == "nearest":
            allowed = torch.zeros_like(ref)
        else:
            allowed = k * ((c_pix(interp, C) + extra) * u * A + CUBIC_ROUNDINGS * u * E) + _tiny(dtype)
        _assert_within(f"remap {name} {interp} {dtype}", f"{what} {name}", got_, ref, allowed, u, A + CUBIC_ROUNDINGS * E)


@gpu
@pytest.mark.parametrize("Bmap", [1, 2])
@pytest.mark.parametrize("normalized", [False, True], ids=["pixel", "normalized"])
@pytest.mark.parametrize("pad", ["zeros", "border", "reflection"])
@pytest.mark.parametrize("interp", ["bilinear", "bicubic", "nearest"])
def test_remap(interp, pad, normalized, Bmap):
    img = _src((2, 3, 360, 640), 11)
    for align in (False, True):
        mx, my = _maps(Bmap, 360, 640, 360, 640, normalized, Bmap)
        check_remap("remap", img, mx, my, interp, pad, align, normalized)
        mx, my = _maps(Bmap, 50, 1, 360, 640, normalized, Bmap + 1)  # a one-pixel-wide map
        check_remap("remap", img, mx, my, interp, pad, align, normalized)


@gpu
@pytest.mark.parametrize("interp", ["bilinear", "bicubic", "nearest"])
def test_remap_fp64(interp):
    img = _src((2, 3, 40, 52), 12, torch.float64)
    for pad in ("zeros", "border", "reflection"):
        for normalized in (False, True):
            mx, my = _maps(2, 30, 44, 40, 52, normalized, 3, torch.float64)
            check_remap("remap", img, mx, my, interp, pad, False, normalized)


# ---- end to end, through the prelude backward ------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("op", ["warp_perspective", "warp_affine"])
@pytest.mark.parametrize("align", [True, False])
@pytest.mark.parametrize("pad", ["zeros", "border"])
def test_end_to_end_matrix_gradient(op, pad, align):
    """d/dM through warp_perspective / warp_affine (prelude backward included) against the same-device oracle in fp32 and
    fp64: ours must be as close to fp64 as the oracle's own fp32 composition."""
    H, W, dsize = 120, 256, (96, 200)
    M = _matrices(H, W)
    if op == "warp_affine":
        M = M[:, :2, :].contiguous()
    src = _src((M.shape[0], 3, H, W), 13)
    g = torch.Generator(device=DEV).manual_seed(1)
    cot = torch.rand(M.shape[0], 3, *dsize, generator=g, device=DEV) * 2 - 1
    ours_fn = getattr(K, op) if hasattr(K, op) else getattr(K.geometry.transform, op)
    ref_fn = getattr(R, op)

    def grads(fn, dtype):
        s, mm = src.to(dtype), M.to(dtype).requires_grad_(True)
        out = fn(s, mm, dsize, padding_mode=pad, align_corners=align)
        return torch.autograd.grad((out * cot.to(dtype)).sum(), mm)[0]

    ours = grads(ours_fn, torch.float32)
    with torch.backends.cudnn.flags(enabled=False):
        r32, r64 = grads(ref_fn, torch.float32), grads(ref_fn, torch.float64)
    check_composed(f"end-to-end {op}", f"{op} {pad} align={align} d/dM", ours, r32, r64, 0)


# ---- fairness: the same-device oracle's own fp32 gradients meet the same bounds ---------------------------------------
@gpu
@pytest.mark.parametrize("align", [True, False])
@pytest.mark.parametrize("projective", [True, False], ids=["proj", "affine"])
@pytest.mark.parametrize("pad", ["zeros", "border"])
def test_oracle_fp32_meets_the_bounds(pad, projective, align):
    H, W, dsize = 120, 256, (96, 200)
    M = _matrices(H, W)
    B = M.shape[0]
    src = _src((B, 3, H, W), 21)
    m, bx, by = sampling(M, (H, W), dsize, projective, align, torch.float32)
    g = torch.Generator(device=DEV).manual_seed(2)
    go = torch.rand(B, 3, *dsize, generator=g, device=DEV) * 2 - 1
    s, mm = src.clone().requires_grad_(True), m.clone().requires_grad_(True)
    with torch.backends.cudnn.flags(enabled=False):
        grid = R.perspective_grid(mm, bx, by) if projective else R.affine_grid(mm, bx, by)
        out = F.grid_sample(s, grid, mode="bilinear", padding_mode=pad, align_corners=align)
        gs, gm = torch.autograd.grad(out, (s, mm), go)
    _, gs_ref, dm = warp_references(src, m, bx, by, None, go, dsize, projective, "bilinear", pad, align)
    what = f"oracle fp32 {pad} {'proj' if projective else 'affine'} align={align}"
    for b in range(B):
        check_gsrc("oracle fp32", f"{what} sample {b}", gs[b], gs_ref[b], "bilinear", torch.float32)
    check_dm("oracle fp32", what, gm.reshape(-1, 9), dm[:, 0], dm[:, 1], dm[:, 2], "bilinear", 3, dsize[1], torch.float32)
