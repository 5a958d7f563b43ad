"""Gradients of the filter family against float64, element by element, at real image sizes.

The input and kernel gradients of filter2d, filter2d_separable and spatial_gradient are linear maps.  For each of them
``ref`` is the float64 autograd gradient of the oracle (oracle/kornia_restated.py) on the fp32 operands widened exactly,
on the same device with cuDNN off, and ``bound`` is the same autograd with every operand (input, taps, cotangent) replaced
by its absolute value: border folds only select elements, so ``bound`` is exactly the sum of |terms| of each output
element.  The kernels are then held to a rounding-error bound per element:

  input gradients   |got - ref| <= 2 n u bound + tiny, n = longest FMA chain of the path (u = 2^-24, or 2^-53 in fp64)
  kernel gradients  |got - ref| <= u (|ref| + sum_p |ref_p|) + (n 2^-53 + 2 u^2) bound + tiny

The kernel-gradient form is what the two-stage reduction promises: each plane p is summed in double and rounded once
(ref_p is that plane's exact contribution), the planes are summed in double and rounded once.  With zero-mean data it is
far tighter than ``2 u bound``, so a reduction that accumulates in fp32 misses it.

The fused ops (SSIM, the corner responses, ScalePyramid) are not linear; their gradients are held to the same-device
oracle run in fp32 (ref32) and fp64 (ref64), separately on the border frame and on the interior.
"""
import math

import pytest
import torch
import torch.nn.functional as F

import kornia_b200 as K
import responses_restated as RR
import scale_pyramid_restated as SR
from oracle import kornia_restated as R

U32 = 2.0 ** -24
U64 = 2.0 ** -53
gpu = pytest.mark.gpu

# group -> largest |got - ref| / (u bound) seen (linear maps), or largest err / allowance (fused ops); printed at teardown
REPORT: dict = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if REPORT:
        print("\nlargest observed error per group:")
        for k in sorted(REPORT):
            print(f"  {k:40s} {REPORT[k]:.3g}")


def _unit(dtype):
    return U32 if dtype == torch.float32 else U64


def _tiny(dtype):
    return torch.finfo(dtype).tiny


# ---------------------------------------------------------------------------------------------------------------------
# the comparator
# ---------------------------------------------------------------------------------------------------------------------
def fold_count(n: int, front: int, rear: int, border: str) -> int:
    """Largest number of padded positions in [-front, n-1+rear] that a border fold maps onto one source index."""
    q = torch.arange(-front, n + rear)
    if border == "constant":
        s = q[(q >= 0) & (q < n)]
    elif border == "replicate":
        s = q.clamp(0, n - 1)
    elif border == "reflect":
        s = torch.where(q < 0, -q, torch.where(q >= n, 2 * (n - 1) - q, q))
    else:
        s = torch.where(q < 0, q + n, torch.where(q >= n, q - n, q))
    return int(torch.bincount(s, minlength=n).max())


def pads(k: int, same: bool):
    return ((k - 1) // 2, (k - 1) - (k - 1) // 2) if same else (0, 0)


def grads64(fn, operands, cot, wrt, absolute=False):
    """float64 autograd of ``fn(*operands)`` contracted with ``cot``, w.r.t. the operands indexed by ``wrt``; with
    ``absolute`` every operand and the cotangent enter as their absolute values."""
    f = (lambda t: t.detach().to(torch.float64).abs()) if absolute else (lambda t: t.detach().to(torch.float64))
    leaves = [f(t).requires_grad_(i in wrt) for i, t in enumerate(operands)]
    with torch.backends.cudnn.flags(enabled=False):
        out = fn(*leaves)
        return torch.autograd.grad(out, [leaves[i] for i in wrt], f(cot).expand(out.shape))


def _record(group, ratio):
    REPORT[group] = max(REPORT.get(group, 0.0), ratio)


def _assert_within(group, what, got, ref, allowed, u, bound):
    """Element-wise |got - ref| <= allowed; records the largest |got - ref| / (u bound) of the group."""
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    err = (got.detach().to(torch.float64) - ref).abs()
    err = torch.where(torch.isnan(err), torch.full_like(err, math.inf), err)
    _record(group, float((err / (u * bound).clamp_min(torch.finfo(torch.float64).tiny)).max()))
    bad = err > allowed
    if bool(bad.any()):
        i = int(torch.argmax((err / allowed.clamp_min(1e-300)).flatten()))
        idx = tuple(int(v) for v in torch.unravel_index(torch.tensor(i), err.shape))
        raise AssertionError(f"{what}: {int(bad.sum())} of {err.numel()} elements out of bound; worst at {idx}: got "
                             f"{float(got.flatten()[i])!r} ref {float(ref.flatten()[i])!r} err {float(err.flatten()[i]):.3e} "
                             f"allowed {float(allowed.flatten()[i]):.3e} (= {float(err.flatten()[i] / (u * bound.flatten()[i])):.3g} u bound)")


def check_input_grad(group, what, got, ref, bound, n, dtype):
    """A chain of n roundings on each of ours and (at most) the reference's: 2 n u times the sum of |terms|."""
    u = _unit(dtype)
    _assert_within(group, what, got, ref, 2 * n * u * bound + _tiny(dtype), u, bound)


def check_kernel_grad(group, what, got, ref, bound, abs_planes, n_double, dtype, folds=0):
    """Two roundings to ``dtype`` of double sums: u |ref| for the total, u |ref_p| for each plane (``abs_planes`` =
    sum_p |ref_p| per tap), ``n_double`` terms summed in double by either side, and 2 u |ref_p| more per plane chunk
    folded in ``dtype`` (``folds``)."""
    u = _unit(dtype)
    allowed = u * (ref.abs() + (1 + 2 * folds) * abs_planes) + (n_double * U64 + 2 * u * u) * bound + _tiny(dtype)
    _assert_within(group, what, got, ref, allowed, u, bound)


def filter2d_bounds(x, k, cot, border, same, wrt_kernel=True):
    """(ref_x, ref_k, bound_x, bound_k, sum_p |ref_p|) of R.filter2d(x, k) contracted with ``cot``."""
    padding = "same" if same else "valid"
    fn = lambda a, b: R.filter2d(a, b, border, padding=padding)  # noqa: E731
    wrt = [0, 1] if wrt_kernel else [0]
    ref = grads64(fn, (x, k), cot, wrt)
    bound = grads64(fn, (x, k), cot, wrt, absolute=True)
    if not wrt_kernel:
        return ref[0], None, bound[0], None, None
    B, C, H, W = x.shape
    Bk = k.shape[0]
    # per-plane contributions: every plane (b, c) filtered with its own copy of kernel b mod Bk
    kp = k[torch.arange(B, device=k.device) % Bk].repeat_interleave(C, 0)
    (ref_p,) = grads64(fn, (x.reshape(B * C, 1, H, W), kp), cot.expand(B, C, *cot.shape[2:]).reshape(B * C, 1, *cot.shape[2:]), [1])
    per_sample = ref_p.abs().reshape(B, C, *k.shape[1:]).sum(1)
    abs_planes = torch.zeros(k.shape, dtype=torch.float64, device=k.device).index_add_(0, torch.arange(B, device=k.device) % Bk, per_sample)
    return ref[0], ref[1], bound[0], bound[1], abs_planes


def plane_folds(B, C):
    """Plane chunks beyond the first whose per-sample kernel gradients are folded with index_add_ (_ops._plane_chunks)."""
    if B * C <= 65535:
        return 0
    return math.ceil(B / (65535 // C))


# ---------------------------------------------------------------------------------------------------------------------
# 1. comparator self-tests (CPU)
# ---------------------------------------------------------------------------------------------------------------------
BORDERS = ["constant", "reflect", "replicate", "circular"]


def _operands(shape, kshape, seed, dtype=torch.float32, device="cpu"):
    g = torch.Generator(device=device).manual_seed(seed)
    x = torch.rand(shape, generator=g, device=device, dtype=dtype) * 2 - 1
    k = torch.rand(kshape, generator=g, device=device, dtype=dtype) * 2 - 1
    return x, k, g


def _oracle_fp32(x, k, cot, border, same):
    xl, kl = x.clone().requires_grad_(True), k.clone().requires_grad_(True)
    out = R.filter2d(xl, kl, border, padding="same" if same else "valid")
    return torch.autograd.grad(out, [xl, kl], cot)


@pytest.mark.parametrize("border", BORDERS)
@pytest.mark.parametrize("K", [3, 11, 15])
def test_comparator_passes_the_oracles_fp32_gradients(border, K):
    x, k, g = _operands((2, 3, 23, 29), (2, K, K), K)
    cot = torch.rand(2, 3, 23, 29, generator=g) * 2 - 1
    got_x, got_k = _oracle_fp32(x, k, cot, border, True)
    ref_x, ref_k, bx, bk, ap = filter2d_bounds(x, k, cot, border, True)
    f = pads(K, True)
    n = K * K * fold_count(23, *f, border) * fold_count(29, *f, border)
    check_input_grad("self-test oracle d/dx", "oracle d/dx", got_x, ref_x, bx, n, torch.float32)
    # The CPU oracle does not sum its kernel gradient in double (it misses check_kernel_grad's cancellation-aware form by
    # 4-40x here); it is held to the looser (2 u + n 2^-53) bound, which it meets at about 0.3 u bound.
    allowed = (2 * U32 + 2 * 3 * 23 * 29 * U64) * bk + _tiny(torch.float32)
    _assert_within("self-test oracle d/dk", "oracle d/dk", got_k, ref_k, allowed, U32, bk)


@pytest.mark.parametrize("border", BORDERS)
def test_comparator_catches_a_border_element_off_by_a_thousandth_of_its_bound(border):
    x, k, g = _operands((1, 2, 20, 24), (1, 5, 5), 1)
    cot = torch.rand(1, 2, 20, 24, generator=g) * 2 - 1
    got_x, _ = _oracle_fp32(x, k, cot, border, True)
    ref_x, _, bx, _, _ = filter2d_bounds(x, k, cot, border, True, wrt_kernel=False)
    n = 25 * fold_count(20, 2, 2, border) * fold_count(24, 2, 2, border)
    check_input_grad("self-test", "unchanged", got_x, ref_x, bx, n, torch.float32)
    bad = got_x.clone()
    bad[0, 1, 19, 0] += 1e-3 * float(bx[0, 1, 19, 0])
    with pytest.raises(AssertionError, match="1 of"):
        check_input_grad("self-test", "perturbed", bad, ref_x, bx, n, torch.float32)


@pytest.mark.parametrize("border", BORDERS)
def test_comparator_catches_two_swapped_taps(border):
    x, k, g = _operands((1, 2, 20, 24), (1, 3, 3), 2)
    cot = torch.rand(1, 2, 20, 24, generator=g) * 2 - 1
    swapped = k.clone()
    swapped[0, 0, 0], swapped[0, 0, 1] = k[0, 0, 1], k[0, 0, 0]
    got_x, got_k = _oracle_fp32(x, swapped, cot, border, True)
    ref_x, ref_k, bx, bk, ap = filter2d_bounds(x, k, cot, border, True)
    n = 9 * fold_count(20, 1, 1, border) * fold_count(24, 1, 1, border)
    with pytest.raises(AssertionError):
        check_input_grad("self-test", "swapped taps", got_x, ref_x, bx, n, torch.float32)


def _stage1_emulated(x, cot, K, border, accumulate):
    """The kernel gradient of one plane as filter2d_bwd_kernel_stage1 computes it (256 threads, thread t sums elements
    t, t + 256, ... in ``accumulate``, a double tree over the threads, one rounding to fp32)."""
    h = K // 2
    cols = F.unfold(F.pad(x, (h, h, h, h), mode=border), K)[0]  # (K*K, H*W): the source element of every term
    terms = cols.double() * cot.reshape(1, -1).double()       # exact in double
    n = terms.shape[1]
    lanes = terms.reshape(K * K, n // 256, 256).to(accumulate)
    s = torch.zeros(K * K, 256, dtype=accumulate)
    for r in range(lanes.shape[1]):
        s = s + lanes[:, r]
    return s.double().sum(1).float().reshape(1, K, K)


@pytest.mark.parametrize("border", ["reflect", "constant"])
def test_comparator_catches_a_kernel_gradient_accumulated_in_fp32(border):
    x, k, g = _operands((1, 1, 256, 256), (1, 3, 3), 3)
    cot = torch.rand(1, 1, 256, 256, generator=g) * 2 - 1
    _, ref_k, _, bk, ap = filter2d_bounds(x, k, cot, border, True)
    n = 256 * 256 + 1
    good = _stage1_emulated(x, cot, 3, border, torch.float64)
    check_kernel_grad("self-test", "double accumulation", good, ref_k, bk, ap, n, torch.float32)
    bad = _stage1_emulated(x, cot, 3, border, torch.float32)
    with pytest.raises(AssertionError):
        check_kernel_grad("self-test", "fp32 accumulation", bad, ref_k, bk, ap, n, torch.float32)


def test_fold_counts():
    assert fold_count(10, 1, 1, "constant") == 1
    assert fold_count(10, 3, 3, "replicate") == 4
    assert fold_count(1, 2, 2, "replicate") == 5
    assert fold_count(10, 2, 2, "reflect") == 2
    assert fold_count(3, 2, 2, "reflect") == 3
    assert fold_count(3, 2, 1, "circular") == 2
    assert fold_count(2, 2, 2, "circular") == 3


# ---------------------------------------------------------------------------------------------------------------------
# 2. direct gradient kernels against float64 on the device
# ---------------------------------------------------------------------------------------------------------------------


def _cuda_operands(shape, kshape, seed, dtype=torch.float32):
    return _operands(shape, kshape, seed, dtype, "cuda")


def _cotangent(g, shape, dtype, layout):
    """A random cotangent of ``shape`` in memory ``layout`` (the stride-0 'sum' / 'mean' layouts are made in _ours)."""
    if layout == "contiguous":
        return torch.rand(shape, generator=g, device="cuda", dtype=dtype) * 2 - 1
    if layout == "channels_last":
        c = torch.rand(shape, generator=g, device="cuda", dtype=dtype) * 2 - 1
        return c.contiguous(memory_format=torch.channels_last) if len(shape) == 4 else c.transpose(1, 2).contiguous().transpose(1, 2)
    if layout == "sliced":
        big = torch.rand(*shape[:-2], shape[-2] + 3, shape[-1] + 5, generator=g, device="cuda", dtype=dtype) * 2 - 1
        return big[..., 1:shape[-2] + 1, 2:shape[-1] + 2]
    raise KeyError(layout)


def _ours(fn, operands, wrt, layout, g):
    """Our gradients of ``fn(*operands)`` w.r.t. ``wrt`` and the cotangent they were taken with (as a dense tensor)."""
    leaves = [t.detach().clone().requires_grad_(i in wrt) for i, t in enumerate(operands)]
    out = fn(*leaves)
    if layout in ("sum", "mean"):
        c = float(torch.rand((), generator=g, device="cuda")) * 2 - 1 if layout == "sum" else 1.0 / out.numel()
        loss = out.sum() * c if layout == "sum" else out.mean()
        grads = torch.autograd.grad(loss, [leaves[i] for i in wrt])
        return grads, torch.full(out.shape, c, device="cuda", dtype=out.dtype)
    cot = _cotangent(g, out.shape, out.dtype, layout)
    return torch.autograd.grad(out, [leaves[i] for i in wrt], cot), cot


def _valid(border, same, H, W, kh, kw):
    if not same:
        return H >= kh and W >= kw
    (ft, rt), (fl, rl) = pads(kh, True), pads(kw, True)
    if border == "reflect":
        return max(ft, rt) < H and max(fl, rl) < W
    if border == "circular":
        return max(ft, rt) <= H and max(fl, rl) <= W
    return True


def run_filter2d(shape, kshape, Bk, border, same, dtype=torch.float32, layout="contiguous", seed=0, group="filter2d"):
    B, C, H, W = shape
    kh, kw = kshape
    x, k, g = _cuda_operands(shape, (Bk, kh, kw), seed, dtype)
    fn = lambda a, b: K.filter2d(a, b, border, padding="same" if same else "valid")  # noqa: E731
    (got_x, got_k), cot = _ours(fn, (x, k), [0, 1], layout, g)
    ref_x, ref_k, bx, bk, ap = filter2d_bounds(x, k, cot, border, same)
    (ft, rt), (fl, rl) = pads(kh, same), pads(kw, same)
    n = kh * kw * fold_count(H, ft, rt, border) * fold_count(W, fl, rl, border)
    what = f"{group} {border} {'same' if same else 'valid'} {shape} k{kh}x{kw} Bk{Bk} {dtype} {layout}"
    check_input_grad(f"{group} d/dinput {dtype}", what + " d/dinput", got_x, ref_x, bx, n, dtype)
    Ho, Wo = cot.shape[-2:]
    n_double = Ho * Wo + B * C + B * C * Ho * Wo  # ours: one plane, then the planes; the reference: everything
    check_kernel_grad(f"{group} d/dkernel {dtype}", what + " d/dkernel", got_k, ref_k, bk, ap, n_double, dtype, plane_folds(B, C))


KERNELS = [(3, 3), (5, 4), (1, 9), (7, 1), (9, 9), (15, 15)]
SMALL = [(3, 2, 61, 68), (1, 1, 33, 260), (2, 3, 37, 70)]


def _small_cases():
    for shape in SMALL + [(4, 2, 37, 70)]:
        bks = [2] if shape[0] == 4 else sorted({1, shape[0]})  # (4, 2, ...): kernel cycling, B = 4, Bk = 2
        for Bk in bks:
            yield pytest.param(shape, Bk, id=f"{'x'.join(map(str, shape))}-Bk{Bk}")


@gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("shape,Bk", list(_small_cases()))
@pytest.mark.parametrize("kshape", KERNELS, ids=lambda k: f"k{k[0]}x{k[1]}")
@pytest.mark.parametrize("same", [True, False], ids=["same", "valid"])
@pytest.mark.parametrize("border", BORDERS)
def test_filter2d_small(border, same, kshape, shape, Bk, dtype):
    run_filter2d(shape, kshape, Bk, border, same, dtype)


@gpu
@pytest.mark.parametrize("shape", [(2, 3, 1080, 1920), (37, 3, 200, 520)], ids=["1080p", "37x3x200x520"])
@pytest.mark.parametrize("kshape", [(3, 3), (5, 4), (15, 15)], ids=lambda k: f"k{k[0]}x{k[1]}")
@pytest.mark.parametrize("per_sample", [False, True], ids=["Bk1", "BkB"])
@pytest.mark.parametrize("border", BORDERS)
def test_filter2d_large(border, per_sample, kshape, shape):
    run_filter2d(shape, kshape, shape[0] if per_sample else 1, border, True)


@gpu
@pytest.mark.parametrize("shape,Bk", [((2, 3, 37, 70), 1), ((2, 3, 37, 70), 2), ((4, 2, 40, 44), 2)])
@pytest.mark.parametrize("same", [True, False], ids=["same", "valid"])
@pytest.mark.parametrize("border", BORDERS)
def test_filter2d_31x31(border, same, shape, Bk):
    run_filter2d(shape, (31, 31), Bk, border, same)


TINY_SHAPES = [(2, 3, 1, 40), (2, 3, 40, 1), (1, 2, 1, 1), (2, 1, 2, 3)]


@gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("shape", TINY_SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("kshape", [(3, 3), (5, 4), (1, 9), (7, 1)], ids=lambda k: f"k{k[0]}x{k[1]}")
@pytest.mark.parametrize("border", BORDERS)
def test_filter2d_tiny_folds(border, kshape, shape, dtype):
    if not _valid(border, True, shape[2], shape[3], *kshape):
        pytest.skip("the border mode does not allow this padding")
    run_filter2d(shape, kshape, shape[0], border, True, dtype)


@gpu
@pytest.mark.parametrize("Bk", [1, 3, 300])
@pytest.mark.parametrize("kshape", [(3, 3), (5, 4)], ids=lambda k: f"k{k[0]}x{k[1]}")
@pytest.mark.parametrize("border", BORDERS)
def test_filter2d_more_planes_than_one_launch(border, kshape, Bk):
    run_filter2d((300, 256, 8, 12), kshape, Bk, border, True)


@gpu
@pytest.mark.parametrize("layout", ["sum", "mean", "channels_last", "sliced"])
@pytest.mark.parametrize("same", [True, False], ids=["same", "valid"])
@pytest.mark.parametrize("border", BORDERS)
def test_filter2d_cotangent_layouts(border, same, layout):
    run_filter2d((2, 3, 37, 70), (5, 4), 2, border, same, layout=layout)


# ---- filter2d_separable, input only: the fast path (fast_filter_bwd=1) and the exact one -------------------------------
def run_sep_input(shape, Ksz, border, fast, dtype=torch.float32, layout="contiguous", seed=0, group="separable d/dinput"):
    B, C, H, W = shape
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.rand(shape, generator=g, device="cuda", dtype=dtype) * 2 - 1
    kx = torch.rand(B, Ksz, generator=g, device="cuda", dtype=dtype)        # asymmetric, per sample
    ky = torch.rand(1, Ksz, generator=g, device="cuda", dtype=dtype) - 0.25  # asymmetric, shared, of both signs
    K.config.set("fast_filter_bwd", int(fast))
    fn_ours = lambda a: K.filter2d_separable(a, kx, ky, border)  # noqa: E731
    (got,), cot = _ours(fn_ours, (x,), [0], layout, g)
    fn = lambda a, b, c: R.filter2d_separable(a, b, c, border)  # noqa: E731
    (ref,) = grads64(fn, (x, kx, ky), cot, [0])
    (bound,) = grads64(fn, (x, kx, ky), cot, [0], absolute=True)
    h = Ksz // 2
    # exact form: Ksz * (fold count) FMAs per pass, two passes; fast form: 2 Ksz + 2; either way within this
    n = Ksz * (fold_count(H, h, h, border) + fold_count(W, h, h, border)) + 2
    what = f"{group} {border} {shape} K{Ksz} fast={fast} {dtype} {layout}"
    check_input_grad(f"{group} {dtype}", what, got, ref, bound, n, dtype)


def _sep_shapes(Ksz):
    h = Ksz // 2
    c = 3 * h + 2  # the fast path needs both sides > 3h + 2 and W % 4 == 0
    return [(2, 3, c, 64), (2, 3, c + 1, 64), (2, 3, 64, c), (2, 3, 64, c + 1), (2, 3, 64, (c + 4) // 4 * 4),
            (2, 3, 40, 70), (2, 3, h + 1, 64)] + SMALL


@gpu
@pytest.mark.parametrize("fast", [1, 0], ids=["fast", "exact"])
@pytest.mark.parametrize("border", ["constant", "reflect", "replicate"])
@pytest.mark.parametrize("Ksz", list(range(3, 18, 2)))
def test_separable_input_gradient(Ksz, border, fast):
    for i, shape in enumerate(_sep_shapes(Ksz)):
        if _valid(border, True, shape[2], shape[3], Ksz, Ksz):
            run_sep_input(shape, Ksz, border, fast, seed=i)


@gpu
@pytest.mark.parametrize("fast", [1, 0], ids=["fast", "exact"])
@pytest.mark.parametrize("border", ["constant", "reflect", "replicate"])
@pytest.mark.parametrize("Ksz", [3, 5, 9, 17])
@pytest.mark.parametrize("shape", [(2, 3, 1080, 1920), (37, 3, 200, 520)], ids=["1080p", "37x3x200x520"])
def test_separable_input_gradient_large(shape, Ksz, border, fast):
    run_sep_input(shape, Ksz, border, fast)


@gpu
@pytest.mark.parametrize("border", ["constant", "reflect", "replicate"])
@pytest.mark.parametrize("Ksz", [3, 7, 15])
def test_separable_input_gradient_fp64(Ksz, border):
    for i, shape in enumerate(SMALL):
        run_sep_input(shape, Ksz, border, 1, dtype=torch.float64, seed=i)


@gpu
@pytest.mark.parametrize("Ksz", [3, 5])
@pytest.mark.parametrize("border", ["constant", "reflect", "replicate"])
def test_separable_input_gradient_more_planes_than_one_launch(border, Ksz):
    run_sep_input((300, 256, 8, 12), Ksz, border, 1)


@gpu
@pytest.mark.parametrize("layout", ["sum", "mean", "channels_last", "sliced"])
@pytest.mark.parametrize("border", ["constant", "reflect", "replicate"])
def test_separable_input_gradient_cotangent_layouts(border, layout):
    run_sep_input((2, 3, 40, 64), 7, border, 1, layout=layout)


# ---- filter2d_separable with x, kx and ky requiring grad: the recomputed-mid path ---------------------------------------
@gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("shape", SMALL + [(2, 3, 1080, 1920)], ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("kw,kh", [(3, 3), (7, 5), (17, 17)])
@pytest.mark.parametrize("same", [True, False], ids=["same", "valid"])
@pytest.mark.parametrize("border", BORDERS)
def test_separable_all_gradients(border, same, kw, kh, shape, dtype):
    if dtype == torch.float64 and shape[2] > 100:
        pytest.skip("fp64 runs at the small shapes")
    if not _valid(border, same, shape[2], shape[3], kh, kw):
        pytest.skip("the border mode does not allow this padding")
    B, C, H, W = shape
    g = torch.Generator(device="cuda").manual_seed(kw * 31 + kh)
    x = torch.rand(shape, generator=g, device="cuda", dtype=dtype) * 2 - 1
    kx = torch.rand(B, kw, generator=g, device="cuda", dtype=dtype) - 0.3
    ky = torch.rand(1, kh, generator=g, device="cuda", dtype=dtype) - 0.3
    padding = "same" if same else "valid"
    (gx, gkx, gky), cot = _ours(lambda a, b, c: K.filter2d_separable(a, b, c, border, padding=padding), (x, kx, ky), [0, 1, 2], "contiguous", g)
    fn = lambda a, b, c: R.filter2d_separable(a, b, c, border, padding=padding)  # noqa: E731
    ref = grads64(fn, (x, kx, ky), cot, [0, 1, 2])
    bound = grads64(fn, (x, kx, ky), cot, [0, 1, 2], absolute=True)
    cy = fold_count(H, *pads(kh, same), border)
    cx = fold_count(W, *pads(kw, same), border)
    Ho, Wo = cot.shape[-2:]
    u = _unit(dtype)
    what = f"separable all {border} {padding} {shape} kx{kw} ky{kh} {dtype}"
    check_input_grad(f"separable all d/dinput {dtype}", what + " d/dx", gx, ref[0], bound[0], kh * cy + kw * cx + 2, dtype)
    # d/dkx pairs x with g_mid (rounded after kh*cy FMAs); d/dky pairs gout with mid = Fx(x) (rounded after kw FMAs); then
    # two roundings of double sums, and the reference's own double sums
    n_double = B * C * H * W * 2 + 2 * B * C
    for name, got, r, b, chain in (("d/dkx", gkx, ref[1], bound[1], kh * cy), ("d/dky", gky, ref[2], bound[2], kw)):
        allowed = (2 * chain * u + 2 * u) * b + n_double * U64 * b + _tiny(dtype)
        _assert_within(f"separable all {name} {dtype}", f"{what} {name}", got, r, allowed, u, b)


# ---- spatial_gradient: every mode, order and normalisation ------------------------------------------------------------
def _sg_taps(mode, order, normalized, dtype):
    taps = R.derivative_taps(mode, order, "cuda", dtype)
    return taps / taps.abs().sum(dim=-1).sum(dim=-1)[..., None, None] if normalized else taps


def _sg_oracle(x, taps):
    """oracle/kornia_restated.py spatial_gradient with the taps as an operand (so that |taps| can enter the bound)."""
    b, c, h, w = x.shape
    half = taps.shape[-1] // 2
    padded = F.pad(x.reshape(b * c, 1, h, w), [half, half, half, half], "replicate")
    return F.conv2d(padded, taps[:, None]).reshape(b, c, taps.shape[0], h, w)


SG_SHAPES = [(2, 3, 1080, 1920), (37, 3, 200, 520), (3, 2, 61, 68), (1, 1, 33, 260), (2, 3, 37, 70),
             (2, 3, 1, 40), (2, 3, 40, 1), (1, 2, 1, 1), (2, 1, 2, 3), (300, 256, 8, 12)]


@gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("shape", SG_SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("normalized", [True, False], ids=["normalized", "raw"])
@pytest.mark.parametrize("mode,order", [("sobel", 1), ("diff", 1), ("sobel", 2), ("diff", 2)])
def test_spatial_gradient(mode, order, normalized, shape, dtype):
    if dtype == torch.float64 and shape[0] * shape[1] * shape[2] * shape[3] > 10 ** 6:
        pytest.skip("fp64 runs at the small shapes")
    x, _, g = _cuda_operands(shape, (1,), sum(shape) + order, dtype)
    layout = "channels_last" if shape[2] == 37 else "sliced" if shape[2] == 61 else "contiguous"
    (got,), cot = _ours(lambda a: K.filters.spatial_gradient(a, mode, order, normalized), (x,), [0], layout, g)
    taps = _sg_taps(mode, order, normalized, dtype)
    with torch.no_grad(), torch.backends.cudnn.flags(enabled=False):
        assert torch.equal(_sg_oracle(x, taps), R.spatial_gradient(x, mode, order, normalized))
    (ref,) = grads64(_sg_oracle, (x, taps), cot, [0])
    (bound,) = grads64(_sg_oracle, (x, taps), cot, [0], absolute=True)
    k = taps.shape[-1]
    n = taps.shape[0] * k * k * fold_count(shape[2], k // 2, k // 2, "replicate") * fold_count(shape[3], k // 2, k // 2, "replicate")
    check_input_grad(f"spatial_gradient {dtype}", f"spatial_gradient {mode} order {order} {normalized} {shape} {dtype}", got, ref, bound, n,
                     dtype)


# ---- motion_blur d/dinput: filter2d's input gradient with the library's motion kernel ---------------------------------
@gpu
@pytest.mark.parametrize("border", ["constant", "reflect"])
@pytest.mark.parametrize("Ksz,shape", [(9, (2, 3, 200, 520)), (9, (1, 3, 1080, 1920)), (31, (2, 3, 200, 520))])
def test_motion_blur_input_gradient(Ksz, shape, border):
    x, _, g = _cuda_operands(shape, (1,), Ksz)
    angle = torch.tensor([17.0, -63.0][: shape[0]], device="cuda")
    direction = torch.tensor([0.4, -0.7][: shape[0]], device="cuda")
    (got,), cot = _ours(lambda a: K.filters.motion_blur(a, Ksz, angle, direction, border), (x,), [0], "contiguous", g)
    kern = K.filters.get_motion_kernel2d(Ksz, angle, direction)
    fn = lambda a, b: R.filter2d(a, b, border)  # noqa: E731
    (ref,) = grads64(fn, (x, kern), cot, [0])
    (bound,) = grads64(fn, (x, kern), cot, [0], absolute=True)
    h = Ksz // 2
    n = Ksz * Ksz * fold_count(shape[2], h, h, border) * fold_count(shape[3], h, h, border)
    check_input_grad("motion_blur d/dinput", f"motion_blur K{Ksz} {shape} {border}", got, ref, bound, n, torch.float32)


# ---------------------------------------------------------------------------------------------------------------------
# 3. composed gradients of the fused ops: ours against the oracle in fp32 and fp64
# ---------------------------------------------------------------------------------------------------------------------
def _rel_l2(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def check_composed(group, what, ours, ref32, ref64, halo):
    """On the border frame (2 halo wide) and on the interior separately:
         max|ours - ref64| <= 4 max|ref32 - ref64| + 2 u max|ref64|
         rel_l2(ours, ref64) <= 2 rel_l2(ref32, ref64) + 1e-7
    i.e. ours is as close to float64 as the oracle's own fp32 composition, up to a small factor."""
    H, W = ref64.shape[-2:]
    f = 2 * halo
    frame = torch.ones(H, W, dtype=torch.bool, device=ref64.device)
    frame[f:H - f, f:W - f] = False
    for name, mask in (("frame", frame), ("interior", ~frame)):
        if not bool(mask.any()):
            continue
        o, r32, r64 = (t.detach().double()[..., mask] for t in (ours, ref32, ref64))
        e_ours, e32 = float((o - r64).abs().max()), float((r32 - r64).abs().max())
        allowed = 4 * e32 + 2 * U32 * float(r64.abs().max())
        rel_ours, rel32 = _rel_l2(o, r64), _rel_l2(r32, r64)
        _record(f"{group} (max err / allowed)", e_ours / max(allowed, 1e-300))
        assert e_ours <= allowed, f"{what} {name}: max|ours - ref64| {e_ours:.3e} > {allowed:.3e} (ref32: {e32:.3e})"
        assert rel_ours <= 2 * rel32 + 1e-7, f"{what} {name}: rel_l2 {rel_ours:.3e} vs ref32 {rel32:.3e}"


def _composed_grads(fn_ours, fn_oracle, inputs, cots):
    """Gradients of sum(out * cot) w.r.t. ``inputs`` for ours (fp32), the oracle in fp32 and in fp64, cuDNN off for the oracle."""
    def run(fn, dtype):
        leaves = [t.detach().to(dtype).requires_grad_(True) for t in inputs]
        outs = fn(*leaves)
        outs = outs if isinstance(outs, (list, tuple)) else [outs]
        loss = sum((o * c.to(dtype)).sum() for o, c in zip(outs, cots))
        return torch.autograd.grad(loss, leaves)

    ours = run(fn_ours, torch.float32)
    with torch.backends.cudnn.flags(enabled=False):
        return ours, run(fn_oracle, torch.float32), run(fn_oracle, torch.float64)


def _images(shape, seed, n=2):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.rand(shape, generator=g, device="cuda")
    return [a] + [(a + 0.2 * torch.rand(shape, generator=g, device="cuda")).clamp(0, 1) for _ in range(n - 1)], g


@gpu
@pytest.mark.parametrize("window", [3, 5, 7, 9, 11])
@pytest.mark.parametrize("shape", [(1, 3, 1080, 1920), (8, 3, 200, 520)], ids=["1080p", "8x3x200x520"])
def test_ssim_gradients(shape, window):
    (a, b), g = _images(shape, window)
    cot = torch.rand(shape, generator=g, device="cuda") * 2 - 1
    ours, r32, r64 = _composed_grads(lambda p, q: K.metrics.ssim(p, q, window), lambda p, q: R.ssim(p, q, window), (a, b), (cot,))
    for name, o, x32, x64 in zip(("d/dimg1", "d/dimg2"), ours, r32, r64):
        check_composed("ssim", f"ssim w{window} {shape} {name}", o, x32, x64, window // 2)
    one = torch.ones((), device="cuda")
    ours, r32, r64 = _composed_grads(lambda p, q: K.losses.ssim_loss(p, q, window), lambda p, q: R.ssim_loss(p, q, window), (a, b), (one,))
    for name, o, x32, x64 in zip(("d/dimg1", "d/dimg2"), ours, r32, r64):
        check_composed("ssim_loss", f"ssim_loss w{window} {shape} {name}", o, x32, x64, window // 2)


@gpu
@pytest.mark.parametrize("with_sigmas", [False, True], ids=["plain", "sigmas"])
@pytest.mark.parametrize("mode", ["sobel", "diff"])
@pytest.mark.parametrize("kind", ["harris", "gftt", "hessian"])
@pytest.mark.parametrize("shape", [(2, 3, 200, 520), (1, 1, 1080, 1920), (3, 2, 61, 68)], ids=lambda s: "x".join(map(str, s)))
def test_response_gradients(shape, kind, mode, with_sigmas):
    (x,), g = _images(shape, len(kind) + len(mode), n=1)
    sig = torch.rand(shape[0], generator=g, device="cuda") + 0.5 if with_sigmas else None
    cot = torch.rand(shape, generator=g, device="cuda") * 2 - 1
    ours_fn = {"harris": lambda t: K.feature.harris_response(t, 0.04, mode, sig),
               "gftt": lambda t: K.feature.gftt_response(t, mode, sig),
               "hessian": lambda t: K.feature.hessian_response(t, mode, sig)}[kind]

    def oracle_fn(t):
        s = None if sig is None else sig.to(t.dtype)
        return {"harris": lambda: RR.harris_response(t, 0.04, mode, s), "gftt": lambda: RR.gftt_response(t, mode, s),
                "hessian": lambda: RR.hessian_response(t, mode, s)}[kind]()

    (o,), (x32,), (x64,) = _composed_grads(ours_fn, oracle_fn, (x,), (cot,))
    halo = 2 if kind == "hessian" else 1 + 3  # stencil, plus the 7x7 structure-tensor blur
    check_composed(f"{kind}_response", f"{kind} {mode} sigmas={with_sigmas} {shape}", o, x32, x64, 2 * halo)


@gpu
def test_sobel_magnitude_gradients():
    for shape in [(2, 3, 200, 520), (1, 1, 1080, 1920), (2, 3, 1, 40)]:
        (x,), g = _images(shape, 7, n=1)
        cot = torch.rand(shape, generator=g, device="cuda") * 2 - 1
        for normalized in (True, False):
            (o,), (x32,), (x64,) = _composed_grads(lambda t: K.filters.sobel(t, normalized), lambda t: R.sobel(t, normalized), (x,), (cot,))
            check_composed("sobel", f"sobel normalized={normalized} {shape}", o, x32, x64, 1)


@gpu
def test_scale_pyramid_gradients():
    sp = K.geometry.transform.ScalePyramid().cuda()
    (x,), g = _images((2, 1, 200, 520), 11, n=1)
    with torch.no_grad():
        levels = SR.scale_pyramid(x)[0]
    cots = [torch.rand(p.shape, generator=g, device="cuda") * 2 - 1 for p in levels]
    (o,), (x32,), (x64,) = _composed_grads(lambda t: sp(t)[0], lambda t: SR.scale_pyramid(t)[0], (x,), cots)
    halo = max(len(t) for t in sp._host_taps.values() if t is not None) // 2
    check_composed("ScalePyramid", "ScalePyramid 2x1x200x520", o, x32, x64, halo)


@gpu
@pytest.mark.parametrize("shape", [(2, 3, 37, 70), (1, 3, 1080, 1920)], ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("ksize", [5, 11])
def test_gaussian_blur_sigma_gradient(shape, ksize):
    """gaussian_blur2d with a sigma that requires grad: the taps are a function of sigma, so every operand of the
    separable filter needs a gradient (the recomputed-mid path)."""
    (x,), g = _images(shape, ksize, n=1)
    sigma = torch.rand(shape[0], 2, generator=g, device="cuda") * 2 + 0.7
    cot = torch.rand(shape, generator=g, device="cuda") * 2 - 1
    ours, r32, r64 = _composed_grads(lambda t, s: K.gaussian_blur2d(t, ksize, s), lambda t, s: R.gaussian_blur2d(t, ksize, s), (x, sigma), (cot,))
    check_composed("gaussian_blur2d sigma", f"gaussian_blur2d K{ksize} {shape} d/dinput", ours[0], r32[0], r64[0], ksize // 2)
    o, a32, a64 = ours[1].double(), r32[1].double(), r64[1]
    e_ours, e32 = float((o - a64).abs().max()), float((a32 - a64).abs().max())
    allowed = 4 * e32 + 2 * U32 * float(a64.abs().max())
    _record("gaussian_blur2d sigma (max err / allowed)", e_ours / max(allowed, 1e-300))
    assert e_ours <= allowed, f"d/dsigma: {e_ours:.3e} > {allowed:.3e} (ref32 {e32:.3e})"
