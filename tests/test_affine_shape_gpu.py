"""PatchAffineShapeEstimator and LAFAffineShapeEstimator on the GPU: the fused kernels (csrc/affine_shape.cuh) against the
float64 evaluation of the composition on the same device, with the fp32 composition as the yardstick; the level and
degenerate decisions; the circular shapes and NaN patterns of the composition; the goldens; CUDA graphs, torch.compile,
opcheck, gradcheck, the launch list; and the orientation chain that consumes the LAFs."""
import importlib
import os
import subprocess
import sys

import pytest
import torch

from conftest import golden

pytestmark = pytest.mark.gpu

F = importlib.import_module("kornia_b200.feature")
AS = importlib.import_module("kornia_b200.feature.affine_shape")
LAF = importlib.import_module("kornia_b200.feature.laf")
KF = importlib.import_module("kornia_b200.filters")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

U = 2.0 ** -24  # fp32 unit roundoff
# The floor of the accuracy bound, relative to S = the largest |entry| of the keypoint's float64 output linear part.  The
# kernel's moments are correctly rounded (fp64 sums, one rounding); what remains is its fp32 tail: the max normalisation
# (1 rounding), two square roots and the clamp (2), a21 and the closed-form inverse (4), get_laf_scale and the rescale
# coefficient (5), the rescale products (1), and with preserve_orientation two atan2 (2 ulp each), two rad2deg (2 each), the
# difference (1, relative to 360 degrees), deg2rad (2), cos / sin (1 ulp each) and the 2 x 2 product (2).  A rotation error
# of d radians moves every entry by at most d * S, and the angle's rounding is relative to its magnitude (at most 360
# degrees, 2 pi radians), so each term is at most a few u * S; their sum stays below 48 u * S.  The bound is the fp32
# composition's largest error times two, plus this floor.
FLOOR = 48 * U
REL = 1e-5


def _image(B, h, w, gen, kind):
    if kind == "noise":
        return torch.rand(B, 1, h, w, generator=gen).cuda()
    yy, xx = torch.linspace(0, 1, h)[:, None], torch.linspace(0, 1, w)[None, :]
    img = torch.zeros(B, 1, h, w)
    for _ in range(6):
        f = torch.randint(0, 9, (2, B, 1, 1, 1), generator=gen).float()
        img = img + torch.sin(6.2831853 * (f[0] * xx + f[1] * yy) + torch.rand(B, 1, 1, 1, generator=gen) * 6.28)
    return (img / 12 + 0.5).cuda()


def _lafs(B, N, h, w, PS, gen, outside=0.15):
    """Rotated, sheared, anisotropic pixel LAFs with log-uniform scales from one level below level 0 to two above the last
    level the pyramid builds (those keypoints get zero patches and circular shapes), some centred outside the image."""
    top = LAF._built_levels(h, w, PS) - 1
    u = torch.rand(B, N, generator=gen) * (top + 3.0) - 1.0
    s = torch.pow(2.0, u) * PS / 2.0
    ang = torch.rand(B, N, generator=gen) * 6.283185307
    r = torch.exp(torch.randn(B, N, generator=gen) * 0.3)
    sh = torch.randn(B, N, generator=gen) * 0.2
    c, si = torch.cos(ang), torch.sin(ang)
    A = torch.stack([torch.stack([c * r.sqrt(), c * sh - si / r.sqrt()], -1),
                     torch.stack([si * r.sqrt(), si * sh + c / r.sqrt()], -1)], -2) * s[..., None, None]
    cx = (torch.rand(B, N, generator=gen) * (1 + 2 * outside) - outside) * (w - 1)
    cy = (torch.rand(B, N, generator=gen) * (1 + 2 * outside) - outside) * (h - 1)
    return torch.cat([A, torch.stack([cx, cy], -1)[..., None]], -1).cuda()


def _composed(m, laf, img):
    """The composition with every stage on its composed path (autograd tracks the LAFs, so the extraction and the patch
    estimator run their compositions too)."""
    with torch.enable_grad():
        return AS._composed_laf_affine_shape(m, laf.detach().clone().requires_grad_(True), img).detach()


def _decisions(m, laf, img):
    """Per keypoint: the level, whether the level and moments clear their margins (log2(scale) >= 1e-3 from an integer,
    every moment >= 1e-3 relative from eps), whether the shape is degenerate, and whether the level is built."""
    PS, det = m.patch_size, m.affine_shape_detector
    B, N = laf.shape[:2]
    with torch.no_grad():
        up = LAF.make_upright(laf)
        scale = 2.0 * LAF.get_laf_scale(LAF.denormalize_laf(LAF.normalize_laf(up, img), img)) / float(PS)
        lg = scale.log2().view(B, N)
        top = min(img.shape[-2:]) // PS
        level = lg.clamp(min=0.0, max=max(0, top - 1)).long()
        built = level < LAF._built_levels(img.shape[-2], img.shape[-1], PS)
        patches = LAF._composed_extract_pyramid(img, up, PS, True).view(-1, 1, PS, PS)
        g = KF.spatial_gradient(patches, "sobel") * det.weighting.to(patches)
        gx, gy = g[:, :, 0], g[:, :, 1]
        mom = torch.stack([(gx * gx).mean((-2, -1)), (gx * gy).mean((-2, -1)), (gy * gy).mean((-2, -1))], -1).view(B, N, 3)
    frac = (lg - lg.round()).abs()
    level_ok = ~lg.isfinite() | (frac >= 1e-3) | (lg <= -1e-3) | (lg >= top - 1 + 1e-3)
    mom_ok = ((mom - det.eps).abs() >= 1e-3 * det.eps).all(-1)
    degenerate = (mom < det.eps).sum(-1) >= 2
    return level, level_ok & mom_ok, degenerate, built


def _rel_err(out, ref):
    """(B, N, 2, 2) |out - ref| of the linear parts over S, the largest |entry| of the reference's linear part."""
    S = ref[..., :2, :2].abs().amax((-2, -1), keepdim=True)
    return (out.double()[..., :2, :2] - ref[..., :2, :2]).abs() / S


WORKLOADS = [(1, 1080, 1920, 8000, 32, "noise"), (1, 1080, 1920, 8000, 19, "smooth"), (8, 480, 640, 2000, 41, "noise"),
             (8, 480, 640, 2000, 41, "smooth")]


@pytest.mark.parametrize("B,h,w,N,PS,kind", WORKLOADS)
@pytest.mark.parametrize("preserve", [True, False])
def test_kernel_within_twice_the_compositions_fp64_error(B, h, w, N, PS, kind, preserve):
    gen = torch.Generator().manual_seed(B * 1000 + PS + (kind == "smooth"))
    img = _image(B, h, w, gen, kind)
    laf = _lafs(B, N, h, w, PS, gen)
    m = F.LAFAffineShapeEstimator(PS, preserve_orientation=preserve).cuda()
    with torch.no_grad():
        got = m(laf, img)
    comp = _composed(m, laf, img)
    ref = _composed(m, laf.double(), img.double())
    _, ok, _, _ = _decisions(m, laf.double(), img.double())
    assert torch.equal(got[..., 2], laf[..., 2])  # the centres are copied
    ek, ec = _rel_err(got, ref)[ok], _rel_err(comp, ref)[ok]
    for i in range(2):
        for j in range(2):
            mk, mc = float(ek[:, i, j].max()), float(ec[:, i, j].max())
            assert mk <= 2 * mc + FLOOR, (i, j, mk, mc)
    nk, nc = int((ek > REL).sum()), int((ec > REL).sum())
    assert nk <= nc, (nk, nc)
    print(f"{B}x{h}x{w} N={N} PS={PS} {kind} preserve={preserve}: kernel max {float(ek.max()):.3g} (>1e-5: {nk}), "
          f"composition max {float(ec.max()):.3g} (>1e-5: {nc}), {int(ok.sum())} of {ok.numel()} keypoints clear the margins")


@pytest.mark.parametrize("B,h,w,N,PS,kind", WORKLOADS[:3])
def test_level_and_degenerate_decisions(B, h, w, N, PS, kind):
    gen = torch.Generator().manual_seed(77 + PS)
    img = _image(B, h, w, gen, kind)
    laf = _lafs(B, N, h, w, PS, gen)
    m = F.LAFAffineShapeEstimator(PS).cuda()
    with torch.no_grad():
        got = m(laf, img)
    comp = _composed(m, laf, img)
    ref = _composed(m, laf.double(), img.double())
    _, ok, _, _ = _decisions(m, laf.double(), img.double())
    # where the margins hold, the same level and degenerate decision as the composition: any other level or shape is far
    # outside 1e-3 of S on these images
    assert float(_rel_err(got, comp.double())[ok].max()) <= 1e-3
    # elsewhere, no more flips against float64 than the composition
    flips_k = int((_rel_err(got, ref).amax((-2, -1)) > 1e-2)[~ok].sum())
    flips_c = int((_rel_err(comp, ref).amax((-2, -1)) > 1e-2)[~ok].sum())
    assert flips_k <= flips_c, (flips_k, flips_c)


@pytest.mark.parametrize("kind", ["unbuilt", "constant", "stripes"])
def test_circular_shapes_equal_the_composition(kind):
    gen = torch.Generator().manual_seed(21)
    h, w, PS = 300, 400, 32
    img = _image(1, h, w, gen, "noise")
    laf = _lafs(1, 500, h, w, PS, gen)
    if kind == "constant":
        img = torch.full_like(img, 0.375)
    if kind == "stripes":  # no vertical gradient once the LAF is upright
        img = ((torch.arange(w, device="cuda") // 4) % 2).float().view(1, 1, 1, w).expand(1, 1, h, w).contiguous()
    for preserve in (True, False):
        m = F.LAFAffineShapeEstimator(PS, preserve_orientation=preserve).cuda()
        with torch.no_grad():
            got, want = m(laf, img), AS._composed_laf_affine_shape(m, laf, img)
        _, _, degenerate, built = _decisions(m, laf, img)
        sel = ~built if kind == "unbuilt" else degenerate
        assert sel.sum() > 20 and (kind != "unbuilt" or bool(degenerate[~built].all()))
        assert torch.equal(got[sel], want[sel])


def test_nonfinite_pixels_and_lafs_give_the_compositions_nans():
    gen = torch.Generator().manual_seed(13)
    img = _image(1, 300, 400, gen, "noise")
    img[0, 0, 100:104, 200:230] = float("nan")
    img[0, 0, 50, 50] = float("inf")
    laf = _lafs(1, 600, 300, 400, 19, gen)
    vals = [float("nan"), float("inf"), float("-inf")]
    for k in range(60):
        laf[0, k, (k // 6) % 2, k % 3] = vals[k % 3]
    m = F.LAFAffineShapeEstimator(19).cuda()
    with torch.no_grad():
        got, want = m(laf, img), AS._composed_laf_affine_shape(m, laf, img)
    assert want.isnan().any() and torch.equal(got.isnan(), want.isnan())
    fin = want.isfinite().all(-1).all(-1)
    assert float(_rel_err(got[fin], want[fin].double()).max()) <= 1e-3


@pytest.mark.parametrize("N", [8000, 65536])
@pytest.mark.parametrize("P", [19, 32])
def test_patch_estimator_within_twice_the_compositions_fp64_error(N, P):
    gen = torch.Generator().manual_seed(N + P)
    x = torch.rand(N, 1, P, P, generator=gen).cuda()
    x[: N // 4] = _image(1, P, P * (N // 4), gen, "smooth").view(1, P, N // 4, P).permute(2, 0, 1, 3)
    x[N // 4: N // 4 + 50] = 0.5  # flat patches
    det = F.PatchAffineShapeEstimator(P).cuda()
    with torch.no_grad():
        got = det(x)
    with torch.enable_grad():
        comp = AS._composed_patch_affine_shape(det, x.clone().requires_grad_(True)).detach()
        det.weighting = det.weighting.double()
        ref = AS._composed_patch_affine_shape(det, x.double())
        det.weighting = det.weighting.float()
    assert torch.equal(got[N // 4: N // 4 + 50], comp[N // 4: N // 4 + 50])  # the circle, exactly
    ek, ec = (got.double() - ref).abs(), (comp.double() - ref).abs()
    for k in range(3):
        assert float(ek[..., k].max()) <= 2 * float(ec[..., k].max()) + 8 * U, k
    assert int((ek > REL).sum()) <= int((ec > REL).sum())


GOLD = golden("affine_shape")


@pytest.mark.parametrize("name", GOLD.names("laf") + GOLD.names("patch"))
def test_goldens_on_the_kernels(name):
    op, kw, ins, outs = GOLD.case(name)
    with torch.no_grad():
        if op == "laf":
            m = F.LAFAffineShapeEstimator(kw["PS"], F.PatchAffineShapeEstimator(kw["PS"], eps=kw["eps"]), kw["preserve_orientation"]).cuda()
            got = m(ins["laf"].cuda(), ins["img"].cuda()).cpu()
        else:
            got = F.PatchAffineShapeEstimator(kw["patch_size"], kw["eps"]).cuda()(ins["patch"].cuda()).cpu()
    want = outs["out"]
    assert torch.equal(got.isnan(), want.isnan())
    ok = ~want.isnan()
    # the goldens come from the CPU reference (pairwise fp32 means, exact division, LAPACK's inverse, the reference's pyrdown)
    torch.testing.assert_close(got[ok], want[ok], rtol=1e-4, atol=1e-4)


def test_cuda_graph_replay():
    gen = torch.Generator().manual_seed(5)
    img = _image(1, 480, 640, gen, "noise")
    laf = _lafs(1, 300, 480, 640, 32, gen)
    m = F.LAFAffineShapeEstimator(32).cuda()
    with torch.no_grad():
        want = m(laf, img)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            m(laf, img)
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = m(laf, img)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, want)
        img.copy_(img.flip(-1))
        g.replay()
        assert torch.equal(out, m(laf, img))


@pytest.mark.parametrize("dynamic", [False, True])
def test_torch_compile_equals_eager(dynamic):
    torch._dynamo.reset()
    gen = torch.Generator().manual_seed(6)
    img = _image(1, 240, 320, gen, "noise")
    laf = _lafs(1, 200, 240, 320, 19, gen)
    m = F.LAFAffineShapeEstimator(19).cuda()
    det = F.PatchAffineShapeEstimator(19).cuda()
    patches = torch.rand(64, 1, 19, 19, generator=gen).cuda()
    with torch.no_grad():
        want, want_p = m(laf, img), det(patches)
    # dynamic shapes are traced with aot_eager: the same one graph, without inductor's code generation
    fn = torch.compile(lambda i, l, p: (m(l, i), det(p)), fullgraph=True, dynamic=dynamic, backend="aot_eager" if dynamic else "inductor")
    with torch.no_grad():
        got, got_p = fn(img, laf, patches)
    assert torch.equal(got, want) and torch.equal(got_p, want_p)


def test_opcheck():
    gen = torch.Generator().manual_seed(8)
    img = _image(2, 100, 120, gen, "noise")
    laf = _lafs(2, 20, 100, 120, 32, gen)
    levels = [img, LAF.pyrdown(img)]
    w = F.PatchAffineShapeEstimator(32).weighting.cuda()
    torch.library.opcheck(torch.ops.kornia_b200.laf_affine_shape_fwd.default, (levels, laf, w, 32, 1e-10, True))
    torch.library.opcheck(torch.ops.kornia_b200.laf_affine_shape_fwd.default, ([img], laf, w, 32, 1e-10, False))
    torch.library.opcheck(torch.ops.kornia_b200.patch_affine_shape_fwd.default, (torch.rand(30, 1, 32, 32, device="cuda"), w, 1e-10))


def test_gradcheck_through_the_composition():
    gen = torch.Generator().manual_seed(9)
    img = _image(1, 40, 50, gen, "smooth").double().requires_grad_(True)
    laf = _lafs(1, 3, 40, 50, 8, gen, outside=-0.2).double()
    laf[..., :2, :2] *= 0.6
    laf.requires_grad_(True)
    m = F.LAFAffineShapeEstimator(8)
    assert torch.autograd.gradcheck(lambda i, l: m(l, i), (img, laf), eps=1e-6, atol=1e-4)
    out = m(laf.detach().float(), img.detach().float().requires_grad_(True))
    assert out.requires_grad  # grad mode with an input that requires grad: the differentiable composition


_PROFILE = r"""
import torch, kornia_b200.feature as F, kornia_b200.feature.laf as LAF
img = torch.rand(1, 1, 1080, 1920, device="cuda"); laf = torch.zeros(1, 500, 2, 3, device="cuda")
laf[..., 0, 0] = 30.0; laf[..., 1, 1] = 20.0; laf[..., 1, 0] = 5.0; laf[..., 0, 2] = 900.0; laf[..., 1, 2] = 500.0
m = F.LAFAffineShapeEstimator(32).cuda()
def names(fn):
    fn(); torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as p:
        fn(); torch.cuda.synchronize()
    return sorted(e.name for e in p.events() if e.device_type == torch.autograd.DeviceType.CUDA and "emcpy" not in e.name and "emset" not in e.name)
with torch.no_grad():
    fused = names(lambda: m(laf, img))
    def build():
        x = img
        for _ in range(LAF._built_levels(1080, 1920, 32) - 1):
            x = LAF.pyrdown(x)
    chain = names(build)
    f64 = names(lambda: m(laf.double(), img.double()))
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
    # the pyrdowns and one kernel: no patch stack, no cuBLAS / cuSOLVER inverse
    assert len(extra) == 1 and "laf_affine_shape_kernel" in extra[0], (fused, chain)
    assert not any("affine_shape_kernel" in n for n in f64) and any("grid_sampler" in n for n in f64), f64
    print(f"fused: {len(fused)} kernels; float64 composition: {len(f64)} kernels")


def test_chain_with_orientation_equals_the_composed_chain():
    gen = torch.Generator().manual_seed(12)
    img = _image(1, 1080, 1920, gen, "smooth")
    laf = _lafs(1, 8000, 1080, 1920, 32, gen)
    aff, ori = F.LAFAffineShapeEstimator(32).cuda(), F.PatchDominantGradientOrientation(19).cuda()
    with torch.no_grad():
        la = aff(laf, img)
        a = ori(F.extract_patches_from_pyramid(img, la, 19).view(-1, 1, 19, 19))
    lc = _composed(aff, laf, img)
    with torch.enable_grad():
        pc = LAF._composed_extract_pyramid(img, lc, 19, True).view(-1, 1, 19, 19)
        ac = ori(pc.requires_grad_(True)).detach()
    assert float(_rel_err(la, lc.double()).max()) <= 1e-3
    dang = (a - ac).abs()
    dang = torch.minimum(dang, 2 * torch.pi - dang)
    print(f"LAF max rel {float(_rel_err(la, lc.double()).max()):.3g}; orientation max {float(dang.max()):.3g}, > 1e-3: {int((dang > 1e-3).sum())}")
    assert int((dang > 1e-3).sum()) <= 16  # near-ties of the two top bins may flip with ulp-level LAF differences
