"""extract_patches_from_pyramid / extract_patches_simple on the GPU: the fused kernel (csrc/laf_patches.cuh) and the
library composition against a float64 replica of the reference's coordinate chain, with per-element bounds derived
below; the exact parts (level choice, zero patches of unbuilt levels, non-finite LAFs) against the same-device
composition; the goldens; CUDA graphs, torch.compile, opcheck, gradcheck, the launch list; and the SIFT / orientation
chains that consume the patches."""
import importlib
import os
import subprocess
import sys

import pytest
import torch

from conftest import golden

pytestmark = pytest.mark.gpu

F = importlib.import_module("kornia_b200.feature")
LAF = importlib.import_module("kornia_b200.feature.laf")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

U = 2.0 ** -24  # fp32 unit roundoff
# The sampling coordinate (pixels of the level) is a chain of about eight fp32 roundings: nlaf = coef * laf (1), theta =
# coef_l * nlaf (1), bx * t0 (1), the fma with by * t1 (1), + t2 (1), * 2 and * 1 / (w_l - 1) (1, plus 1 in the reciprocal),
# - 1 (1), and unnormalize's fma (1).  Each is at most u relative to the magnitude it produces; X_p bounds those magnitudes
# in pixels (below), so the coordinate is off by at most K_COORD * u * X_p, and the bilinear value by that times D_p, the
# largest adjacent-texel difference around the sample (linear interpolation is D_p-Lipschitz per axis; two axes).
K_COORD = 10
# The blend: each weight is one rounded product of exact differences (1), and four fmas accumulate (<= 4, relative to the
# running sum of |w v|), so FWD_ROUNDINGS * u * sum |w v| bounds it.
FWD_ROUNDINGS = 6


def _lafs(B, N, h, w, PS, gen, device):
    """Rotated, sheared, anisotropic pixel LAFs with log-uniform scales from one level below level 0 to two above the last
    level the pyramid builds (the clamp allows far more at large images; beyond the built levels every patch is zero)."""
    top = LAF._built_levels(h, w, PS) - 1
    u = torch.rand(B, N, generator=gen) * (top + 3.0) - 1.0
    s = torch.pow(2.0, u) * PS / 2.0
    ang = torch.rand(B, N, generator=gen) * 6.283185307
    r = torch.exp(torch.randn(B, N, generator=gen) * 0.3)
    sh = torch.randn(B, N, generator=gen) * 0.2
    c, si = torch.cos(ang), torch.sin(ang)
    A = torch.stack([torch.stack([c * r.sqrt(), c * sh - si / r.sqrt()], -1),
                     torch.stack([si * r.sqrt(), si * sh + c / r.sqrt()], -1)], -2) * s[..., None, None]
    cx = (torch.rand(B, N, generator=gen) * 1.3 - 0.15) * (w - 1)
    cy = (torch.rand(B, N, generator=gen) * 1.3 - 0.15) * (h - 1)
    return torch.cat([A, torch.stack([cx, cy], -1)[..., None]], -1).to(device)


def _image(B, C, h, w, gen, kind):
    if kind == "noise":
        return torch.rand(B, C, h, w, generator=gen).cuda()
    yy, xx = torch.linspace(0, 1, h)[:, None], torch.linspace(0, 1, w)[None, :]
    img = torch.zeros(B, C, h, w)
    for _ in range(6):
        f = torch.randint(0, 9, (2, B, C, 1, 1), generator=gen).float()
        img = img + torch.sin(6.2831853 * (f[0] * xx + f[1] * yy) + torch.rand(B, C, 1, 1, generator=gen) * 6.28)
    return (img / 12 + 0.5).cuda()


def _levels(img, PS):
    levels = [img]
    for _ in range(LAF._built_levels(img.shape[-2], img.shape[-1], PS) - 1):
        levels.append(LAF.pyrdown(levels[-1]))
    return levels


def _composed_levels(img, laf, PS, normalize=True):
    """The composition's fp32 level of every patch (B, N) on this device."""
    nlaf = LAF.normalize_laf(laf, img) if normalize else laf
    scale = 2.0 * LAF.get_laf_scale(LAF.denormalize_laf(nlaf, img)) / float(PS)
    top = min(img.shape[-2:]) // PS
    return scale.log2().clamp(min=0.0, max=max(0, top - 1)).long().view(laf.shape[:2])


def _replica(levels, laf, PS, idx, normalize=True):
    """float64 patches of the reference's chain at the levels ``idx``, with the bound of each element."""
    B, N = laf.shape[:2]
    C = levels[0].shape[1]
    h0, w0 = levels[0].shape[-2:]
    L = laf.double()
    if normalize:
        L = L * torch.tensor([[1 / min(h0 - 1, w0 - 1)] * 2 + [1 / (w0 - 1)], [1 / min(h0 - 1, w0 - 1)] * 2 + [1 / (h0 - 1)]],
                             dtype=torch.float64, device=L.device)
    ref = torch.zeros(B, N, C, PS, PS, dtype=torch.float64, device=L.device)
    bound = torch.zeros_like(ref)
    j = torch.arange(PS, device=L.device, dtype=torch.float64)
    base = (2 * j - (PS - 1)) / PS if PS > 1 else torch.zeros(1, dtype=torch.float64, device=L.device)
    bx, by = base.view(1, PS), base.view(PS, 1)
    for lv, img in enumerate(levels):
        sel = (idx == lv).nonzero()
        if sel.numel() == 0:
            continue
        b, n = sel[:, 0], sel[:, 1]
        h, w = img.shape[-2:]
        m = float(min(h - 1, w - 1))
        T = L[b, n] * torch.tensor([[m, m, w - 1], [m, m, h - 1]], dtype=torch.float64, device=L.device)
        t = [T[:, r, c].view(-1, 1, 1) for r in range(2) for c in range(3)]
        G, H = bx * t[0] + by * t[1] + t[2], bx * t[3] + by * t[4] + t[5]
        mag_x = (bx * t[0]).abs() + (by * t[1]).abs() + t[2].abs()
        mag_y = (bx * t[3]).abs() + (by * t[4]).abs() + t[5].abs()
        ix = ((2 * G / (w - 1) - 1) + 1) * w / 2 - 0.5
        iy = ((2 * H / (h - 1) - 1) + 1) * h / 2 - 0.5
        X = torch.maximum(mag_x * w / max(w - 1, 1) + w / 2 + ix.abs(), mag_y * h / max(h - 1, 1) + h / 2 + iy.abs())
        ix, iy = ix.clamp(0, w - 1), iy.clamp(0, h - 1)
        x0, y0 = ix.floor().long(), iy.floor().long()
        fx, fy = ix - x0, iy - y0
        flat = img.double().reshape(-1)  # the level's texels, gathered by global index (no per-patch image copies)
        plane = ((b.view(-1, 1, 1, 1) * C + torch.arange(C, device=L.device).view(1, C, 1, 1)) * (h * w))

        def tex(yy, xx):
            yy, xx = yy.clamp(0, h - 1), xx.clamp(0, w - 1)
            return flat[plane + (yy * w + xx).unsqueeze(1)]

        v00, v01, v10, v11 = tex(y0, x0), tex(y0, x0 + 1), tex(y0 + 1, x0), tex(y0 + 1, x0 + 1)
        fx, fy = fx.unsqueeze(1), fy.unsqueeze(1)
        val = (1 - fx) * (1 - fy) * v00 + fx * (1 - fy) * v01 + (1 - fx) * fy * v10 + fx * fy * v11
        D = torch.zeros_like(val)
        for dy in (-1, 0, 1, 2):  # adjacent-texel differences of the 4 x 4 texels around the sample, along both axes
            for dx in (-1, 0, 1, 2):
                a = tex(y0 + dy, x0 + dx)
                if dx < 2:
                    D = torch.maximum(D, (tex(y0 + dy, x0 + dx + 1) - a).abs())
                if dy < 2:
                    D = torch.maximum(D, (tex(y0 + dy + 1, x0 + dx) - a).abs())
        absw = (1 - fx) * (1 - fy) * v00.abs() + fx * (1 - fy) * v01.abs() + (1 - fx) * fy * v10.abs() + fx * fy * v11.abs()
        ref[b, n] = val
        bound[b, n] = 2 * K_COORD * U * X.unsqueeze(1) * D + FWD_ROUNDINGS * U * absw + 1e-30
    return ref, bound


WORKLOADS = [(1, 1, 1080, 1920, 8000, 19), (1, 1, 1080, 1920, 8000, 41), (8, 3, 480, 640, 2000, 32)]


@pytest.mark.parametrize("B,C,h,w,N,PS", WORKLOADS)
def test_kernel_and_composition_within_the_fp64_bound(B, C, h, w, N, PS):
    gen = torch.Generator().manual_seed(B * 1000 + PS)
    img = _image(B, C, h, w, gen, "noise")
    laf = _lafs(B, N, h, w, PS, gen, "cuda")
    with torch.no_grad():
        got = F.extract_patches_from_pyramid(img, laf, PS)
        comp = LAF._composed_extract_pyramid(img, laf, PS, True)
        idx = _composed_levels(img, laf, PS)
        n_built = LAF._built_levels(h, w, PS)
        ref, bound = _replica(_levels(img, PS), laf, PS, idx)
    built = (idx < n_built).view(B, N, 1, 1, 1).expand_as(got)
    for name, out in (("kernel", got), ("composition", comp)):
        err = (out.double() - ref).abs()
        bad = (err > bound) & built
        assert not bad.any(), (name, int(bad.sum()), float(err[bad].max()), float(bound[bad].min()))
    # the level is the composition's: patches of unbuilt levels are exactly zero in both, and every other patch is within
    # the bound of the replica at the composition's level (a neighbouring level of a noise image is far outside it)
    assert torch.equal(got[~built], torch.zeros_like(got[~built])) and torch.equal(comp[~built], got[~built])
    print(f"{B}x{C}x{h}x{w} N={N} PS={PS}: max |kernel - composition| {float((got - comp).abs().max()):.3g}, "
          f"levels {torch.bincount(idx.view(-1)).tolist()}")


def test_simple_variant_within_the_fp64_bound():
    gen = torch.Generator().manual_seed(7)
    img = _image(2, 3, 240, 320, gen, "smooth")
    laf = _lafs(2, 500, 240, 320, 32, gen, "cuda")
    with torch.no_grad():
        got = F.extract_patches_simple(img, laf, 32)
        comp = LAF._composed_extract_simple(img, laf, 32, True)
        ref, bound = _replica([img], laf, 32, torch.zeros(2, 500, dtype=torch.long, device="cuda"))
    for out in (got, comp):
        assert not ((out.double() - ref).abs() > bound).any()


def test_nonfinite_lafs_equal_the_composition():
    gen = torch.Generator().manual_seed(11)
    img = _image(1, 3, 300, 400, gen, "noise")
    laf = _lafs(1, 64, 300, 400, 32, gen, "cuda")
    vals = [float("nan"), float("inf"), float("-inf")]
    for k in range(48):
        laf[0, k, (k // 6) % 2, k % 3] = vals[k % 3]
    with torch.no_grad():
        for fn, comp in ((F.extract_patches_from_pyramid, LAF._composed_extract_pyramid), (F.extract_patches_simple, LAF._composed_extract_simple)):
            got, want = fn(img, laf, 32), comp(img, laf, 32, True)
            # the same level, the same zero patches and the same NaNs; a coordinate that stays finite may differ by the ulps of
            # the fixed versus cuBLAS's order of affine_grid's sum, as for finite LAFs
            a, b = got[:, :48], want[:, :48]
            assert torch.equal(a.isnan(), b.isnan())
            assert torch.equal(a.flatten(2).eq(0).all(-1), b.flatten(2).eq(0).all(-1))
            assert float((a.nan_to_num() - b.nan_to_num()).abs().max()) <= 1e-5


GOLD = golden("patches")


@pytest.mark.parametrize("name", GOLD.names("patches"))
def test_goldens_on_the_kernel(name):
    _, kw, ins, outs = GOLD.case(name)
    fn = {"pyramid": F.extract_patches_from_pyramid, "simple": F.extract_patches_simple}[kw["fn"]]
    with torch.no_grad():
        got = fn(ins["img"].cuda(), ins["laf"].cuda(), kw["PS"], kw["normalize"]).cpu()
    want = outs["out"]
    assert torch.equal(got.isnan(), want.isnan())
    ok = ~want.isnan()
    # the goldens come from the CPU reference (exact division, another bmm order, the reference's pyrdown): within the sum
    # of both sides' bounds, which for images in [0, 1] at these sizes stays below 1e-4
    torch.testing.assert_close(got[ok], want[ok], rtol=0, atol=1e-4)


def test_a_strided_level0_and_extra_images():
    gen = torch.Generator().manual_seed(3)
    big = _image(3, 2, 200, 300, gen, "noise")
    view = big[:, :, 10:170, 20:260]
    laf = _lafs(2, 100, 160, 240, 19, gen, "cuda")
    with torch.no_grad():
        got = F.extract_patches_from_pyramid(view, laf, 19)
        want = F.extract_patches_from_pyramid(view.contiguous()[:2], laf, 19)
    assert torch.equal(got, want)


def test_cuda_graph_replay():
    gen = torch.Generator().manual_seed(5)
    img = _image(1, 1, 480, 640, gen, "noise")
    laf = _lafs(1, 300, 480, 640, 32, gen, "cuda")
    with torch.no_grad():
        want = F.extract_patches_from_pyramid(img, laf, 32)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            F.extract_patches_from_pyramid(img, laf, 32)
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = F.extract_patches_from_pyramid(img, laf, 32)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, want)
        laf.mul_(1.0)
        img.copy_(img.flip(-1))
        g.replay()
        assert torch.equal(out, F.extract_patches_from_pyramid(img, laf, 32))


@pytest.mark.parametrize("dynamic", [False, True])
def test_torch_compile_equals_eager(dynamic):
    torch._dynamo.reset()
    gen = torch.Generator().manual_seed(6)
    img = _image(1, 1, 240, 320, gen, "noise")
    laf = _lafs(1, 200, 240, 320, 19, gen, "cuda")
    # dynamic shapes are traced with aot_eager: the traced graph is the same one graph, without inductor's code generation
    fn = torch.compile(lambda i, l: F.extract_patches_from_pyramid(i, l, 19), fullgraph=True, dynamic=dynamic,
                       backend="aot_eager" if dynamic else "inductor")
    with torch.no_grad():
        got, want = fn(img, laf), F.extract_patches_from_pyramid(img, laf, 19)
    # under compilation pyrdown runs its composition (bit-identical to its fused kernel), the extraction the same kernel
    assert torch.equal(got, want)


def test_opcheck():
    gen = torch.Generator().manual_seed(8)
    img = _image(2, 3, 100, 120, gen, "noise")
    laf = _lafs(2, 20, 100, 120, 32, gen, "cuda")
    levels = _levels(img, 32)
    torch.library.opcheck(torch.ops.kornia_b200.extract_patches_fwd.default, (levels, laf, 32, True, True))
    torch.library.opcheck(torch.ops.kornia_b200.extract_patches_fwd.default, ([img], laf, 19, False, False))


def test_gradcheck_through_the_composition():
    gen = torch.Generator().manual_seed(9)
    img = _image(1, 2, 40, 50, gen, "smooth").double().requires_grad_(True)
    laf = _lafs(1, 3, 40, 50, 8, gen, "cuda").double().requires_grad_(True)
    assert torch.autograd.gradcheck(lambda i, l: F.extract_patches_from_pyramid(i, l, 8), (img, laf), eps=1e-6, atol=1e-5)
    img32, laf32 = img.detach().float().requires_grad_(True), laf.detach().float()
    out = F.extract_patches_from_pyramid(img32, laf32, 8)
    assert out.requires_grad  # grad mode with an input that requires grad: the differentiable composition


_PROFILE = r"""
import torch, kornia_b200.feature as F, kornia_b200.feature.laf as LAF
img = torch.rand(1, 1, 1080, 1920, device="cuda"); laf = torch.zeros(1, 500, 2, 3, device="cuda")
laf[..., 0, 0] = 30.0; laf[..., 1, 1] = 30.0; laf[..., 0, 2] = 900.0; laf[..., 1, 2] = 500.0
def names(fn):
    fn(); torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as p:
        fn(); torch.cuda.synchronize()
    return sorted(e.name for e in p.events() if e.device_type == torch.autograd.DeviceType.CUDA and "emcpy" not in e.name and "emset" not in e.name)
with torch.no_grad():
    fused = names(lambda: F.extract_patches_from_pyramid(img, laf, 41))
    def build():
        x = img
        for _ in range(LAF._built_levels(1080, 1920, 41) - 1):
            x = LAF.pyrdown(x)
    chain = names(build)
    f64 = names(lambda: F.extract_patches_from_pyramid(img.double(), laf.double(), 41))
print("FUSED", fused); print("CHAIN", chain); print("F64", f64)
"""


def test_launch_list_in_a_fresh_interpreter():
    run = subprocess.run([sys.executable, "-c", _PROFILE], capture_output=True, text=True, cwd=ROOT, timeout=300)
    assert run.returncode == 0, run.stdout[-2000:] + run.stderr[-4000:]
    out = {ln.split(" ", 1)[0]: eval(ln.split(" ", 1)[1]) for ln in run.stdout.splitlines() if ln.split(" ", 1)[0] in ("FUSED", "CHAIN", "F64")}
    fused, chain, f64 = out["FUSED"], out["CHAIN"], out["F64"]
    extra = list(fused)
    for n in chain:
        extra.remove(n)
    assert len(extra) == 1 and "laf_patches_kernel" in extra[0], (fused, chain)
    assert not any("laf_patches_kernel" in n for n in f64) and any("grid_sampler" in n for n in f64), f64


def test_end_to_end_orientation_and_sift():
    gen = torch.Generator().manual_seed(12)
    img = _image(1, 1, 1080, 1920, gen, "smooth")
    laf = _lafs(1, 8000, 1080, 1920, 41, gen, "cuda")
    ori, sift = F.PatchDominantGradientOrientation(19).cuda(), F.SIFTDescriptor(41).cuda()
    with torch.no_grad():
        p19, c19 = F.extract_patches_from_pyramid(img, laf, 19), LAF._composed_extract_pyramid(img, laf, 19, True)
        p41, c41 = F.extract_patches_from_pyramid(img, laf, 41), LAF._composed_extract_pyramid(img, laf, 41, True)
        a, ac = ori(p19.view(-1, 1, 19, 19)), ori(c19.view(-1, 1, 19, 19))
        d, dc = sift(p41.view(-1, 1, 41, 41)), sift(c41.view(-1, 1, 41, 41))
    dang = (a - ac).abs()
    dang = torch.minimum(dang, 2 * torch.pi - dang)
    print(f"orientation: max {float(dang.max()):.3g}, > 1e-4: {int((dang > 1e-4).sum())}; sift max {float((d - dc).abs().max()):.3g}")
    assert float((d - dc).abs().max()) <= 1e-4
    assert int((dang > 1e-4).sum()) <= 8  # near-ties of the two top bins may flip with one-ulp patch differences
