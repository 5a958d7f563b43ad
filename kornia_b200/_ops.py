"""The library's kernels as registered PyTorch operators (``torch.ops.kornia_b200.*``).

Every entry point of the C ABI (include/kornia_b200.h) that touches an image is wrapped in one operator defined with
``torch.library``: a CUDA implementation (marshals pointers + sizes into the ``extern "C"`` call on the current stream),
a fake / meta implementation (shapes, dtypes and device of the results; what ``torch.compile`` and the ``meta`` device
run) and, for the differentiable ones, an autograd formula whose backward is again one of these operators.  PyTorch
supplies device memory, streams and autograd bookkeeping; every FLOP on an image is executed by kornia_b200/csrc.

This is the "C-ABI equivalent" row of SURVEY.md section 8(b): schemas ``warp_fwd / warp_bwd / remap_fwd / remap_bwd /
sepfilter_fwd / filter2d_fwd / filter2d_bwd_input / filter2d_bwd_kernel`` plus the operators of the callers either side
of the path.  The public functions (geometry/transform/imgwarp.py, filters/filter.py ...) call these operators and
carry no ``torch.compiler.disable``: ``torch.compile(fullgraph=True)`` sees opaque operators with known output shapes.
A CPU tensor reaching an operator raises (CUDA-only engine, no fallback); backward operators have no autograd formula of
their own, so double backward fails loudly ("... does not have an autograd formula") instead of silently dropping terms.
"""
from __future__ import annotations

import ctypes
import os
from typing import List, Optional, Sequence, Tuple

import torch

from . import _lib

NS = "kornia_b200"
_library = torch.library.Library(NS, "DEF")
ops = getattr(torch.ops, NS)

_DTYPES = {torch.float32: _lib.F32, torch.float64: _lib.F64}

# number of kernels of this library launched since import (bench.py reports it as gpu_launches)
launch_count = 0


def _require_cuda(t: torch.Tensor, what: str) -> None:
    if not t.is_cuda:
        raise RuntimeError(
            f"kornia_b200: {what} lives on {t.device}; this engine is CUDA-only (sm_90a) and has no CPU path. "
            "Move the tensors to an H100 (`.cuda()`)."
        )


def _dtype_code(t: torch.Tensor) -> int:
    try:
        return _DTYPES[t.dtype]
    except KeyError:
        raise RuntimeError(f"kornia_b200: unsupported dtype {t.dtype}; float32 and float64 are implemented") from None


def _same(ref: torch.Tensor, other: torch.Tensor, what: str) -> None:
    if other.device != ref.device:
        raise RuntimeError(f"Expected all tensors to be on the same device, but {what} is on {other.device} and the image on {ref.device}")
    if other.dtype != ref.dtype:
        raise RuntimeError(f"expected {what} to have the same dtype as the image, but got {other.dtype} and {ref.dtype}")


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def _stream(t: torch.Tensor):
    return torch.cuda.current_stream(t.device).cuda_stream


def _bump(n: int = 1) -> None:
    global launch_count
    launch_count += n


# Optional per-kernel CUDA-event timing of the forward kernels (bench.py's roofline leg): when a list
# is installed here, every forward C call is bracketed by events recorded on the launching stream.
kernel_events = None


class _Timed:
    def __init__(self, tag: str, ref: torch.Tensor):
        self.tag, self.ref = tag, ref

    def __enter__(self):
        if kernel_events is not None:
            self.start = torch.cuda.Event(enable_timing=True)
            self.stop = torch.cuda.Event(enable_timing=True)
            self.start.record(torch.cuda.current_stream(self.ref.device))
        return self

    def __exit__(self, *exc):
        if kernel_events is not None and exc[0] is None:
            self.stop.record(torch.cuda.current_stream(self.ref.device))
            kernel_events.append((self.tag, self.start, self.stop))
        return False


# ---------------------------------------------------------------------------------------------
# registration helpers
# ---------------------------------------------------------------------------------------------
def _define(name: str, schema: str, cuda_impl, fake_impl, first_tensor: str = "the input") -> None:
    """One operator: schema, CUDA kernel, fake/meta kernel, and a CPU kernel that only says there is none."""
    _library.define(name + schema)
    _library.impl(name, cuda_impl, "CUDA")
    torch.library.register_fake(f"{NS}::{name}", fake_impl, lib=_library)

    def no_cpu_path(*args, **kwargs):
        t = next(a for a in args if isinstance(a, torch.Tensor))
        _require_cuda(t, first_tensor)
        raise RuntimeError(f"kornia_b200::{name}: CUDA-only operator called with host tensors")

    _library.impl(name, no_cpu_path, "CPU")


def _direct(*tensors: Optional[torch.Tensor]) -> bool:
    """True when a call may skip the dispatcher and run the CUDA implementation directly: eager mode, CUDA tensors, and no
    tensor that autograd tracks.  The operator route costs ~20 us per call (dispatcher -> Python kernel -> autograd wrapper),
    which is what a 32 x 3 x 256 x 256 warp spends on the device; large batches do not notice either way."""
    if torch.compiler.is_compiling():
        return False
    grad = torch.is_grad_enabled()
    for t in tensors:
        if t is None:
            continue
        if not t.is_cuda or (grad and t.requires_grad):
            return False
    return True


_HALF = (torch.float16, torch.bfloat16)


def _half_passthrough(fn, image: torch.Tensor, others: Sequence[Optional[torch.Tensor]], *rest):
    """fp16 / bf16 images (the pass-through dtypes of the reference's test matrix, testing/base.py:35-36; not a BASELINE
    configuration): the kernels compute in fp32 -- operands are widened, the result is narrowed back to the image's dtype;
    autograd flows through the casts.  Costs two conversion passes; the arithmetic is at least as accurate as the reference's
    half-precision composition."""
    wide = [None if t is None else (t.float() if t.is_floating_point() else t) for t in others]
    return fn(image.float(), *wide, *rest).to(image.dtype)


def _autograd(name: str, backward, setup_context) -> None:
    torch.library.register_autograd(f"{NS}::{name}", backward, setup_context=setup_context, lib=_library)


def _once_differentiable(name: str) -> None:
    """Backward operators are first-order only: differentiating THROUGH one (create_graph=True: gradient penalties,
    Hessian-vector products) raises instead of silently dropping the second-order terms.  The reference supports double
    backward through its torch-op composition; ``config.set("torch_prelude", 1)`` gives the matrix chain as torch ops, there is no such
    switch for the image kernels."""

    def backward(ctx, *grads):
        raise RuntimeError(f"kornia_b200::{name} is a backward kernel without a derivative of its own: double backward "
                           "(create_graph=True) through the CUDA warp / filter kernels is not implemented")

    _autograd(name, backward, lambda ctx, inputs, output: None)


def _fake_same_device(ref: torch.Tensor, *others: Optional[torch.Tensor]) -> None:
    """What the CUDA kernels require of their operands, checked on fake / meta tensors too: one device for all."""
    for t in others:
        if t is not None and t.device != ref.device:
            raise RuntimeError(f"Expected all tensors to be on the same device, but found at least two devices, {ref.device} and {t.device}!")


# ---------------------------------------------------------------------------------------------
# warp: out = sample(src, map(m, bx, by)); differentiable w.r.t. src and m
# ---------------------------------------------------------------------------------------------
def _warp_fwd_cuda(src, m, bx, by, fill, h, w, projective, interp, pad, align):
    _require_cuda(src, "src")
    _same(src, m, "the transformation matrix")
    dt = _dtype_code(src)
    src_c, m_c = src.contiguous(), m.contiguous()
    bx = bx.to(device=src.device, dtype=src.dtype).contiguous()
    by = by.to(device=src.device, dtype=src.dtype).contiguous()
    fill_c = None if fill is None else fill.to(device=src.device, dtype=src.dtype).contiguous()
    B, C, H, W = src_c.shape
    out = torch.empty((B, C, h, w), device=src.device, dtype=src.dtype)
    if out.numel() > 0 and src_c.numel() > 0:
        with torch.cuda.device(src.device), _Timed("warp_forward", src):
            _lib.call("kb200_warp_forward", _ptr(src_c), _ptr(m_c), _ptr(bx), _ptr(by), _ptr(fill_c), _ptr(out),
                      B, C, H, W, h, w, m_c.shape[0], int(projective), interp, pad, int(align), dt, _stream(src))
        _bump(_lib.last_warp_launches())
    else:
        out.zero_()
    return out


def _warp_fwd_fake(src, m, bx, by, fill, h, w, projective, interp, pad, align):
    _fake_same_device(src, m)
    if m.dtype != src.dtype:
        raise RuntimeError(f"expected the transformation matrix to have the same dtype as the image, but got {m.dtype} and {src.dtype}")
    return src.new_empty((src.shape[0], src.shape[1], h, w))


def _warp_bwd_cuda(gout, src, m, bx, by, fill, h, w, projective, interp, pad, align, need_src, need_m):
    dt = _dtype_code(src)
    src_c, m_c, gout = src.contiguous(), m.contiguous(), gout.contiguous()
    bx = bx.to(device=src.device, dtype=src.dtype).contiguous()
    by = by.to(device=src.device, dtype=src.dtype).contiguous()
    fill_c = None if fill is None else fill.to(device=src.device, dtype=src.dtype).contiguous()
    B, C, H, W = src_c.shape
    none = src.new_empty(0)
    if gout.numel() == 0 or src_c.numel() == 0:
        return (torch.zeros_like(src_c) if need_src else none), (torch.zeros_like(m_c) if need_m else none)
    gsrc = torch.zeros_like(src_c) if need_src else None
    gm = ws = None
    with torch.cuda.device(src.device):
        if need_m:
            gm = torch.empty_like(m_c)
            nbytes = _lib.load().kb200_warp_backward_workspace_bytes(B, h, w, dt)
            ws = torch.empty(nbytes, dtype=torch.uint8, device=src.device)
        with _Timed("warp_backward", src):
            _lib.call("kb200_warp_backward", _ptr(gout), _ptr(src_c), _ptr(m_c), _ptr(bx), _ptr(by), _ptr(fill_c), _ptr(gsrc), _ptr(gm),
                      _ptr(ws), B, C, H, W, h, w, m_c.shape[0], int(projective), interp, pad, int(align), dt, _stream(src))
    _bump(2 if need_m else 1)
    return (gsrc if need_src else none), (gm if need_m else none)


def _warp_bwd_fake(gout, src, m, bx, by, fill, h, w, projective, interp, pad, align, need_src, need_m):
    _fake_same_device(src, gout, m)
    none = src.new_empty(0)
    return (torch.empty_like(src, memory_format=torch.contiguous_format) if need_src else none,
            torch.empty_like(m, memory_format=torch.contiguous_format) if need_m else none)


_define("warp_fwd", "(Tensor src, Tensor m, Tensor bx, Tensor by, Tensor? fill, int h, int w, bool projective, int interp, int pad, "
        "bool align) -> Tensor", _warp_fwd_cuda, _warp_fwd_fake, "src")
_define("warp_bwd", "(Tensor gout, Tensor src, Tensor m, Tensor bx, Tensor by, Tensor? fill, int h, int w, bool projective, int interp, "
        "int pad, bool align, bool need_src, bool need_m) -> (Tensor, Tensor)", _warp_bwd_cuda, _warp_bwd_fake, "src")


_once_differentiable("warp_bwd")


def _warp_setup(ctx, inputs, output):
    src, m, bx, by, fill, h, w, projective, interp, pad, align = inputs
    ctx.save_for_backward(src, m, bx, by, fill)
    ctx.cfg = (h, w, projective, interp, pad, align)


def _warp_backward(ctx, gout):
    src, m, bx, by, fill = ctx.saved_tensors
    need_src, need_m = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
    gsrc = gm = None
    if need_src or need_m:
        gsrc, gm = ops.warp_bwd(gout, src, m, bx, by, fill, *ctx.cfg, need_src, need_m)
    return (gsrc if need_src else None, gm if need_m else None) + (None,) * 9


_autograd("warp_fwd", _warp_backward, _warp_setup)


def warp(src, m, bx, by, fill, h, w, projective, interp, pad, align):
    if src.dtype in _HALF:
        if m.dtype != src.dtype:
            raise RuntimeError(f"expected the transformation matrix to have the same dtype as the image, but got {m.dtype} and {src.dtype}")
        return _half_passthrough(warp, src, (m, bx, by, fill), h, w, projective, interp, pad, align)
    if _direct(src, m, fill):
        return _warp_fwd_cuda(src, m, bx, by, fill, int(h), int(w), bool(projective), int(interp), int(pad), bool(align))
    return ops.warp_fwd(src, m, bx, by, fill, int(h), int(w), bool(projective), int(interp), int(pad), bool(align))


# ---------------------------------------------------------------------------------------------
# the (B,3,3) prelude in one launch: inverse(N_dst @ M3 @ N_src^-1), bit-identical to the torch op sequence
# ---------------------------------------------------------------------------------------------
FUSED_VARIANT = 4  # the contraction orders that reproduce torch's CUDA kernels bit for bit (GPU-tested)


def _prelude_cuda(M, sh, sw, dh, dw, affine):
    _require_cuda(M, "the transformation matrix")
    Mc = M.contiguous()
    out = torch.empty((Mc.shape[0], 3, 3), device=M.device, dtype=M.dtype)
    if out.numel() > 0:
        with torch.cuda.device(M.device):
            _lib.call("kb200_warp_prelude", _ptr(Mc), _ptr(out), Mc.shape[0], 2 if affine else 3, sh, sw, dh, dw, _dtype_code(M),
                      FUSED_VARIANT, _stream(M))
        _bump()
    return out


def _prelude_bwd_cuda(m, gm, sh, sw, dh, dw, affine):
    rows = 2 if affine else 3
    m, gm = m.contiguous(), gm.contiguous()
    gM = torch.empty((m.shape[0], rows, 3), device=m.device, dtype=m.dtype)
    if gM.numel() > 0:
        with torch.cuda.device(m.device):
            _lib.call("kb200_warp_prelude_backward", _ptr(m), _ptr(gm), _ptr(gM), m.shape[0], rows, sh, sw, dh, dw, _dtype_code(m), _stream(m))
        _bump()
    return gM


_define("warp_prelude", "(Tensor M, int sh, int sw, int dh, int dw, bool affine) -> Tensor", _prelude_cuda,
        lambda M, sh, sw, dh, dw, affine: M.new_empty((M.shape[0], 3, 3)), "the transformation matrix")
_define("warp_prelude_bwd", "(Tensor m, Tensor gm, int sh, int sw, int dh, int dw, bool affine) -> Tensor", _prelude_bwd_cuda,
        lambda m, gm, sh, sw, dh, dw, affine: m.new_empty((m.shape[0], 2 if affine else 3, 3)), "the transformation matrix")


_once_differentiable("warp_prelude_bwd")


def _prelude_setup(ctx, inputs, output):
    ctx.save_for_backward(output)
    ctx.cfg = inputs[1:]


def _prelude_backward(ctx, gm):
    (m,) = ctx.saved_tensors
    return ops.warp_prelude_bwd(m, gm, *ctx.cfg), None, None, None, None, None


_autograd("warp_prelude", _prelude_backward, _prelude_setup)


def prelude(M, sh, sw, dh, dw, affine):
    if _direct(M):
        return _prelude_cuda(M, int(sh), int(sw), int(dh), int(dw), bool(affine))
    return ops.warp_prelude(M, int(sh), int(sw), int(dh), int(dw), bool(affine))


# ---------------------------------------------------------------------------------------------
# remap: out = sample(image, (map_x, map_y)); differentiable w.r.t. the image and both maps
# ---------------------------------------------------------------------------------------------
def _remap_fwd_cuda(image, map_x, map_y, normalized, interp, pad, align):
    _require_cuda(image, "image")
    _same(image, map_x, "map_x")
    _same(image, map_y, "map_y")
    dt = _dtype_code(image)
    img, mx, my = image.contiguous(), map_x.contiguous(), map_y.contiguous()
    B, C, H, W = img.shape
    Bmap, h, w = mx.shape
    out = torch.empty((B, C, h, w), device=img.device, dtype=img.dtype)
    if out.numel() > 0 and img.numel() > 0:
        with torch.cuda.device(img.device), _Timed("remap_forward", img):
            _lib.call("kb200_remap_forward", _ptr(img), _ptr(mx), _ptr(my), _ptr(out), B, C, H, W, h, w, Bmap,
                      int(normalized), interp, pad, int(align), dt, _stream(img))
        _bump()
    else:
        out.zero_()
    return out


def _remap_fwd_fake(image, map_x, map_y, normalized, interp, pad, align):
    _fake_same_device(image, map_x, map_y)
    return image.new_empty((image.shape[0], image.shape[1], map_x.shape[1], map_x.shape[2]))


def _remap_bwd_cuda(gout, image, map_x, map_y, normalized, interp, pad, align, need_img, need_map):
    dt = _dtype_code(image)
    img, mx, my, gout = image.contiguous(), map_x.contiguous(), map_y.contiguous(), gout.contiguous()
    B, C, H, W = img.shape
    Bmap, h, w = mx.shape
    none = img.new_empty(0)
    gimg = torch.zeros_like(img) if need_img else None
    gmx = gmy = None
    if need_map:
        gmx = torch.zeros((B, h, w), device=img.device, dtype=img.dtype) if gout.numel() == 0 or img.numel() == 0 else \
            torch.empty((B, h, w), device=img.device, dtype=img.dtype)
        gmy = torch.zeros_like(gmx) if gout.numel() == 0 or img.numel() == 0 else torch.empty_like(gmx)
    if gout.numel() > 0 and img.numel() > 0:
        with torch.cuda.device(img.device), _Timed("remap_backward", img):
            _lib.call("kb200_remap_backward", _ptr(gout), _ptr(img), _ptr(mx), _ptr(my), _ptr(gimg), _ptr(gmx), _ptr(gmy),
                      B, C, H, W, h, w, Bmap, int(normalized), interp, pad, int(align), dt, _stream(img))
        _bump()
    if need_map and Bmap == 1 and B > 1:  # maps were broadcast over the batch (imgwarp.py:695)
        gmx, gmy = gmx.sum(0, keepdim=True), gmy.sum(0, keepdim=True)
    return (gimg if need_img else none), (gmx if need_map else none), (gmy if need_map else none)


def _remap_bwd_fake(gout, image, map_x, map_y, normalized, interp, pad, align, need_img, need_map):
    _fake_same_device(image, gout, map_x, map_y)
    none = image.new_empty(0)
    gmap = image.new_empty(tuple(map_x.shape)) if need_map else none
    return (torch.empty_like(image, memory_format=torch.contiguous_format) if need_img else none), gmap, (torch.empty_like(gmap) if need_map else none)


_define("remap_fwd", "(Tensor image, Tensor map_x, Tensor map_y, bool normalized, int interp, int pad, bool align) -> Tensor",
        _remap_fwd_cuda, _remap_fwd_fake, "image")
_define("remap_bwd", "(Tensor gout, Tensor image, Tensor map_x, Tensor map_y, bool normalized, int interp, int pad, bool align, "
        "bool need_img, bool need_map) -> (Tensor, Tensor, Tensor)", _remap_bwd_cuda, _remap_bwd_fake, "image")


_once_differentiable("remap_bwd")


def _remap_setup(ctx, inputs, output):
    ctx.save_for_backward(*inputs[:3])
    ctx.cfg = inputs[3:]


def _remap_backward(ctx, gout):
    img, mx, my = ctx.saved_tensors
    need = ctx.needs_input_grad
    need_img, need_map = need[0], need[1] or need[2]
    if not (need_img or need_map):
        return (None,) * 7
    gimg, gmx, gmy = ops.remap_bwd(gout, img, mx, my, *ctx.cfg, need_img, need_map)
    return (gimg if need_img else None, gmx if need[1] else None, gmy if need[2] else None, None, None, None, None)


_autograd("remap_fwd", _remap_backward, _remap_setup)


def remap(image, map_x, map_y, normalized, interp, pad, align):
    if image.dtype in _HALF:
        return _half_passthrough(remap, image, (map_x, map_y), normalized, interp, pad, align)
    if _direct(image, map_x, map_y):
        return _remap_fwd_cuda(image, map_x, map_y, bool(normalized), int(interp), int(pad), bool(align))
    return ops.remap_fwd(image, map_x, map_y, bool(normalized), int(interp), int(pad), bool(align))


# ---------------------------------------------------------------------------------------------
# filter2d: depthwise correlation with the border folded into the index; kernel (Bk,kh,kw) already flipped / normalised
# ---------------------------------------------------------------------------------------------
MAX_PLANES = 65535  # gridDim.z / plane-count limit of one filter launch (the warp kernels chunk inside the C library)


def _plane_chunks(B: int, C: int):
    """Batch ranges [b0, b1) whose plane count B'*C fits one launch: feature maps like B=256, C=256 are served by several
    launches over batch slices (samples are independent; a sample's C planes stay together so kernels keep cycling over
    samples as in filter.py:131,141-142)."""
    if B * C <= MAX_PLANES:
        return [(0, B)]
    if C > MAX_PLANES:
        raise RuntimeError(f"kornia_b200: {C} channels per sample exceed the {MAX_PLANES}-plane launch limit")
    step = MAX_PLANES // C
    return [(b0, min(B, b0 + step)) for b0 in range(0, B, step)]


def _kernel_rows(kernel: torch.Tensor, b0: int, b1: int) -> torch.Tensor:
    """Kernels of the samples [b0, b1): sample b uses kernel row b mod Bk."""
    Bk = kernel.shape[0]
    if Bk == 1:
        return kernel
    idx = torch.arange(b0, b1, device=kernel.device) % Bk
    return kernel.index_select(0, idx).contiguous()


def _filter_out_hw(H, W, kh, kw, same):
    return (H, W) if same else (max(H - kh + 1, 0), max(W - kw + 1, 0))


def _check_kernel_batch(B, C, H, W, Bk, numel):
    if Bk == 0 or B % Bk != 0:
        # the reference's view(-1, Bk*C, H, W) (filter.py:142) fails the same way
        raise RuntimeError(f"shape '[-1, {Bk * C}, {H}, {W}]' is invalid for input of size {numel}")


def _filter2d_call(xc, kc, border, same):
    """The C call of filter2d on contiguous operands (shared by the operator and by the large-kernel route of sepfilter)."""
    B, C, H, W = xc.shape
    Bk, kh, kw = kc.shape
    _check_kernel_batch(B, C, H, W, Bk, xc.numel())
    out = torch.empty((B, C) + _filter_out_hw(H, W, kh, kw, same), device=xc.device, dtype=xc.dtype)
    if out.numel() > 0:
        with torch.cuda.device(xc.device), _Timed("filter2d_forward", xc):
            for b0, b1 in _plane_chunks(B, C):
                k = kc if (b0, b1) == (0, B) else _kernel_rows(kc, b0, b1)
                _lib.call("kb200_filter2d_forward", _ptr(xc[b0:b1]), _ptr(k), _ptr(out[b0:b1]), b1 - b0, C, H, W, k.shape[0], kh, kw, border,
                          int(same), _dtype_code(xc), _stream(xc))
                _bump()
    return out


def _filter2d_fwd_cuda(x, kernel, border, same):
    _require_cuda(x, "input")
    _same(x, kernel, "the kernel")
    return _filter2d_call(x.contiguous(), kernel.contiguous(), border, same)


def _filter2d_fwd_fake(x, kernel, border, same):
    _fake_same_device(x, kernel)
    B, C, H, W = x.shape
    Bk, kh, kw = kernel.shape
    _check_kernel_batch(B, C, H, W, Bk, x.numel())
    return x.new_empty((B, C) + _filter_out_hw(H, W, kh, kw, same))


def _filter2d_bwd_input_cuda(gout, kernel, H, W, border, same):
    gout, k = gout.contiguous(), kernel.contiguous()
    B, C = gout.shape[:2]
    Bk, kh, kw = k.shape
    gx = torch.empty((B, C, H, W), device=gout.device, dtype=gout.dtype)
    if gout.numel() == 0:
        return gx.zero_()
    if gx.numel() > 0:
        with torch.cuda.device(gout.device), _Timed("filter2d_backward_input", gout):
            for b0, b1 in _plane_chunks(B, C):
                kk = k if (b0, b1) == (0, B) else _kernel_rows(k, b0, b1)
                _lib.call("kb200_filter2d_backward_input", _ptr(gout[b0:b1]), _ptr(kk), _ptr(gx[b0:b1]), b1 - b0, C, H, W, kk.shape[0], kh, kw,
                          border, int(same), _dtype_code(gout), _stream(gout))
                _bump()
    return gx


def _filter2d_bwd_kernel_cuda(gout, x, Bk, kh, kw, border, same):
    gout, x = gout.contiguous(), x.contiguous()
    B, C, H, W = x.shape
    dt = _dtype_code(x)
    gk = torch.empty((Bk, kh, kw), device=x.device, dtype=x.dtype)
    if gout.numel() == 0 or x.numel() == 0:
        return gk.zero_()
    chunks = _plane_chunks(B, C)
    with torch.cuda.device(x.device), _Timed("filter2d_backward_kernel", x):
        if len(chunks) == 1:
            nbytes = _lib.load().kb200_filter2d_backward_kernel_workspace_bytes(B, C, H, W, Bk, kh, kw, dt)
            ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
            _lib.call("kb200_filter2d_backward_kernel", _ptr(gout), _ptr(x), _ptr(gk), _ptr(ws), B, C, H, W, Bk, kh, kw, border, int(same), dt,
                      _stream(x))
            _bump(2)
        else:  # per-sample kernel gradients of each slice, folded onto the Bk kernel rows (sample b feeds row b mod Bk)
            gk.zero_()
            for b0, b1 in chunks:
                n = b1 - b0
                part = torch.empty((n, kh, kw), device=x.device, dtype=x.dtype)
                nbytes = _lib.load().kb200_filter2d_backward_kernel_workspace_bytes(n, C, H, W, n, kh, kw, dt)
                ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
                _lib.call("kb200_filter2d_backward_kernel", _ptr(gout[b0:b1]), _ptr(x[b0:b1]), _ptr(part), _ptr(ws), n, C, H, W, n, kh, kw, border,
                          int(same), dt, _stream(x))
                _bump(2)
                gk.index_add_(0, torch.arange(b0, b1, device=x.device) % Bk, part)
    return gk


_define("filter2d_fwd", "(Tensor x, Tensor kernel, int border, bool same) -> Tensor", _filter2d_fwd_cuda, _filter2d_fwd_fake, "input")
_define("filter2d_bwd_input", "(Tensor gout, Tensor kernel, int H, int W, int border, bool same) -> Tensor", _filter2d_bwd_input_cuda,
        lambda gout, kernel, H, W, border, same: (_fake_same_device(gout, kernel), gout.new_empty(tuple(gout.shape[:2]) + (H, W)))[1], "input")
_define("filter2d_bwd_kernel", "(Tensor gout, Tensor x, int Bk, int kh, int kw, int border, bool same) -> Tensor", _filter2d_bwd_kernel_cuda,
        lambda gout, x, Bk, kh, kw, border, same: (_fake_same_device(x, gout), x.new_empty((Bk, kh, kw)))[1], "input")


_once_differentiable("filter2d_bwd_input")
_once_differentiable("filter2d_bwd_kernel")


def _filter2d_setup(ctx, inputs, output):
    x, kernel, border, same = inputs
    ctx.save_for_backward(x, kernel)
    ctx.cfg = (border, same)


def _filter2d_backward(ctx, gout):
    x, k = ctx.saved_tensors
    border, same = ctx.cfg
    gx = gk = None
    if ctx.needs_input_grad[0]:
        gx = ops.filter2d_bwd_input(gout, k, x.shape[2], x.shape[3], border, same)
    if ctx.needs_input_grad[1]:
        gk = ops.filter2d_bwd_kernel(gout, x, k.shape[0], k.shape[1], k.shape[2], border, same)
    return gx, gk, None, None


_autograd("filter2d_fwd", _filter2d_backward, _filter2d_setup)


def filter2d(x, kernel, border, same):
    if x.dtype in _HALF:
        return _half_passthrough(filter2d, x, (kernel,), border, same)
    if _direct(x, kernel):
        return _filter2d_fwd_cuda(x, kernel, int(border), bool(same))
    return ops.filter2d_fwd(x, kernel, int(border), bool(same))


# ---------------------------------------------------------------------------------------------
# separable filter: row pass then column pass in ONE kernel (one read + one write of the image)
# ---------------------------------------------------------------------------------------------
def _sepfilter_fwd_cuda(x, kx, ky, border, same):
    _require_cuda(x, "input")
    _same(x, kx, "kernel_x")
    _same(x, ky, "kernel_y")
    dt = _dtype_code(x)
    xc, kxc, kyc = x.contiguous(), kx.contiguous(), ky.contiguous()
    B, C, H, W = xc.shape
    (Bkx, kw), (Bky, kh) = kxc.shape, kyc.shape
    if Bkx == 0 or Bky == 0 or B % Bkx != 0 or B % Bky != 0:
        raise RuntimeError(f"shape '[-1, {max(Bkx, Bky) * C}, {H}, {W}]' is invalid for input of size {xc.numel()}")
    out = torch.empty((B, C) + _filter_out_hw(H, W, kh, kw, same), device=x.device, dtype=x.dtype)
    if out.numel() > 0:
        try:
            with torch.cuda.device(x.device), _Timed("sepfilter_forward", x):
                for b0, b1 in _plane_chunks(B, C):
                    whole = (b0, b1) == (0, B)
                    kxs, kys = (kxc, kyc) if whole else (_kernel_rows(kxc, b0, b1), _kernel_rows(kyc, b0, b1))
                    _lib.call("kb200_sepfilter_forward", _ptr(xc[b0:b1]), _ptr(kxs), _ptr(kys), _ptr(out[b0:b1]), b1 - b0, C, H, W, kxs.shape[0], kw,
                              kys.shape[0], kh, border, int(same), dt, _stream(x))
                    _bump()
        except _lib.Unsupported:
            # kernels too large for the one-pass shared-memory tile: two 1-D passes of the 2-D kernel
            mid = _filter2d_call(xc, kxc[:, None, :].contiguous(), border, same)
            out = _filter2d_call(mid, kyc[:, :, None].contiguous(), border, same)
    return out


def _sepfilter_fwd_fake(x, kx, ky, border, same):
    _fake_same_device(x, kx, ky)
    B, C, H, W = x.shape
    return x.new_empty((B, C) + _filter_out_hw(H, W, ky.shape[1], kx.shape[1], same))


_define("sepfilter_fwd", "(Tensor x, Tensor kx, Tensor ky, int border, bool same) -> Tensor", _sepfilter_fwd_cuda, _sepfilter_fwd_fake, "input")


def _sepfilter_setup(ctx, inputs, output):
    x, kx, ky, border, same = inputs
    ctx.save_for_backward(x, kx, ky)
    ctx.cfg = (border, same)


def _sepfilter_backward(ctx, gout):
    """The 1-D adjoints composed by hand: g_mid = Fy^T(gout), gx = Fx^T(g_mid); d/dky pairs gout with mid = Fx(x) (recomputed,
    one generic pass, only when ky needs a gradient), d/dkx pairs g_mid with x.  Same C calls, same bits as differentiating
    the two-pass composition of the reference (filter.py:205-207), without the forward passes autograd would rebuild."""
    x, kx, ky = ctx.saved_tensors
    border, same = ctx.cfg
    need = ctx.needs_input_grad
    H, W = x.shape[2], x.shape[3]
    kx2, ky2 = kx[:, None, :], ky[:, :, None]
    if need[0] and not (need[1] or need[2]) and same and fast_filter_bwd_enabled():
        return _sep_input_gradient(gout, kx, ky, border), None, None, None, None
    Hm, Wm = H, (W if same else max(W - kx.shape[1] + 1, 0))  # shape of mid = Fx(x): the row pass keeps the height
    gx = gkx = gky = None
    g_mid = None
    if need[0] or need[1]:
        g_mid = ops.filter2d_bwd_input(gout, ky2, Hm, Wm, border, same)
    if need[0]:
        gx = ops.filter2d_bwd_input(g_mid, kx2, H, W, border, same)
    if need[1]:
        gkx = ops.filter2d_bwd_kernel(g_mid, x, kx.shape[0], 1, kx.shape[1], border, same)[:, 0, :]
    if need[2]:
        mid = ops.filter2d_fwd(x, kx2, border, same)
        gky = ops.filter2d_bwd_kernel(gout, mid, ky.shape[0], ky.shape[1], 1, border, same)[:, :, 0]
    return gx, gkx, gky, None, None


_autograd("sepfilter_fwd", _sepfilter_backward, _sepfilter_setup)


def sepfilter(x, kx, ky, border, same):
    if x.dtype in _HALF:
        return _half_passthrough(sepfilter, x, (kx, ky), border, same)
    if _direct(x, kx, ky):
        return _sepfilter_fwd_cuda(x, kx, ky, int(border), bool(same))
    return ops.sepfilter_fwd(x, kx, ky, int(border), bool(same))


def fast_filter_bwd_enabled() -> bool:
    from . import config

    return config.enabled("fast_filter_bwd")


def _sep_input_gradient(gout: torch.Tensor, kx: torch.Tensor, ky: torch.Tensor, border: int) -> torch.Tensor:
    """d/dinput of the 'same' separable filter.  Exact form: the two adjoint passes of the composition.  When the one-pass
    tiled kernel covers the shape, the image-sized work runs through it instead (adjoint = correlation with the flipped
    taps under a 'constant' border) and only the border bands take the exact form (filters/_adjoint.py).  Everything goes
    through registered operators, so the path is the same under eager, AOT-traced and compiled backward passes."""
    from .filters._adjoint import separable_adjoint

    def exact(g, kx_, ky_):
        H, W = g.shape[2], g.shape[3]
        g_mid = ops.filter2d_bwd_input(g, ky_[:, :, None], H, W, border, True)
        return ops.filter2d_bwd_input(g_mid, kx_[:, None, :], H, W, border, True)

    def forward_constant(g, kx_, ky_):
        return ops.sepfilter_fwd(g, kx_, ky_, _lib.CONSTANT, True)

    kw, kh = kx.shape[-1], ky.shape[-1]
    fast = gout.dtype == torch.float32 and kw == kh and kw % 2 == 1 and 3 <= kw <= 17 and border != _lib.CIRCULAR and gout.shape[-1] % 4 == 0
    return separable_adjoint(gout, kx, ky, border, forward_constant, exact) if fast else exact(gout, kx, ky)


# ---------------------------------------------------------------------------------------------
# callers with a kernel of their own: derivative stencils / Sobel, SSIM, unsharp (blur + lerp), pyrdown, undistort
# ---------------------------------------------------------------------------------------------
def _spatial_gradient_fwd_cuda(x, taps, nout, k, magnitude, eps):
    _require_cuda(x, "input")
    dt = _dtype_code(x)
    xc = x.contiguous()
    B, C, H, W = xc.shape
    out = torch.empty((B, C, H, W) if magnitude else (B, C, nout, H, W), device=x.device, dtype=x.dtype)
    if out.numel() > 0:
        host_taps = (ctypes.c_double * len(taps))(*taps)
        with torch.cuda.device(x.device), _Timed("spatial_gradient_forward", x):
            _lib.call("kb200_spatial_gradient_forward", _ptr(xc), host_taps, _ptr(out), B * C, H, W, nout, k, int(magnitude), float(eps), dt,
                      _stream(x))
        _bump()
    return out


def _spatial_gradient_bwd_cuda(gout, taps, nout, k):
    gout = gout.contiguous()
    B, C, _, H, W = gout.shape
    gx = torch.empty((B, C, H, W), device=gout.device, dtype=gout.dtype)
    if gx.numel() > 0:
        host_taps = (ctypes.c_double * len(taps))(*taps)
        with torch.cuda.device(gout.device):
            _lib.call("kb200_spatial_gradient_backward", _ptr(gout), host_taps, _ptr(gx), B * C, H, W, nout, k, _dtype_code(gout), _stream(gout))
        _bump()
    return gx


_define("spatial_gradient_fwd", "(Tensor x, float[] taps, int nout, int k, bool magnitude, float eps) -> Tensor", _spatial_gradient_fwd_cuda,
        lambda x, taps, nout, k, magnitude, eps: x.new_empty(tuple(x.shape) if magnitude else (x.shape[0], x.shape[1], nout, x.shape[2], x.shape[3])),
        "input")
_define("spatial_gradient_bwd", "(Tensor gout, float[] taps, int nout, int k) -> Tensor", _spatial_gradient_bwd_cuda,
        lambda gout, taps, nout, k: gout.new_empty((gout.shape[0], gout.shape[1], gout.shape[3], gout.shape[4])), "input")


_once_differentiable("spatial_gradient_bwd")


def _spatial_gradient_setup(ctx, inputs, output):
    _, taps, nout, k, magnitude, _ = inputs
    ctx.cfg = (list(taps), nout, k, magnitude)


def _spatial_gradient_backward(ctx, gout):
    taps, nout, k, magnitude = ctx.cfg
    if magnitude:
        raise RuntimeError("kornia_b200: the fused Sobel magnitude is forward-only; sobel() composes the "
                           "differentiable path when the input requires grad")
    return ops.spatial_gradient_bwd(gout, taps, nout, k), None, None, None, None, None


_autograd("spatial_gradient_fwd", _spatial_gradient_backward, _spatial_gradient_setup)


def spatial_gradient(x, taps: Sequence[float], nout: int, k: int, magnitude: bool, eps: float):
    """``nout`` k x k derivative stencils over a replicate border in one kernel: x (B,C,H,W) -> (B,C,nout,H,W), or the Sobel
    magnitude (B,C,H,W) when ``magnitude`` (forward only).  ``taps``: nout*k*k floats whose values are exact in x.dtype."""
    return ops.spatial_gradient_fwd(x, [float(t) for t in taps], int(nout), int(k), bool(magnitude), float(eps))


def _ssim_fwd_cuda(img1, img2, kernel, C1, C2, eps):
    _require_cuda(img1, "img1")
    _require_cuda(img2, "img2")
    a, b, kc = img1.contiguous(), img2.contiguous(), kernel.contiguous()
    B, C, H, W = a.shape
    out = torch.empty_like(a)
    with torch.cuda.device(a.device), _Timed("ssim_forward", a):
        _lib.call("kb200_ssim_forward", _ptr(a), _ptr(b), _ptr(kc), _ptr(out), B * C, H, W, kc.shape[-1], float(C1), float(C2), float(eps),
                  _dtype_code(a), _stream(a))
    _bump()
    return out


_define("ssim_fwd", "(Tensor img1, Tensor img2, Tensor kernel, float C1, float C2, float eps) -> Tensor", _ssim_fwd_cuda,
        lambda img1, img2, kernel, C1, C2, eps: (_fake_same_device(img1, img2, kernel), torch.empty_like(img1, memory_format=torch.contiguous_format))[1],
        "img1")


HARRIS, GFTT, HESSIAN = 0, 1, 2  # kind of kb200_feature_response_forward


def _feature_response_cuda(x, stencil, stencil_k, blur, k, k_tensor, s4, kind):
    _require_cuda(x, "input")
    xc = x.contiguous()
    B, C, H, W = xc.shape
    out = torch.empty_like(xc)
    host_taps = (ctypes.c_double * len(stencil))(*stencil)
    with torch.cuda.device(x.device), _Timed("feature_response_forward", x):
        _lib.call("kb200_feature_response_forward", _ptr(xc), host_taps, _ptr(blur), float(k), _ptr(k_tensor), _ptr(s4), _ptr(out), B * C, C, H, W,
                  stencil_k, 0 if blur is None else blur.shape[-1], kind, _dtype_code(x), _stream(x))
    _bump()
    return out


_define("feature_response_fwd",
        "(Tensor x, float[] stencil, int stencil_k, Tensor? blur, float k, Tensor? k_tensor, Tensor? s4, int kind) -> Tensor",
        _feature_response_cuda,
        lambda x, stencil, stencil_k, blur, k, k_tensor, s4, kind: (_fake_same_device(x, blur, k_tensor, s4),
                                                                      torch.empty_like(x, memory_format=torch.contiguous_format))[1])


def _scale_octave_cuda(x, taps, ksizes):
    _require_cuda(x, "input")
    xc = x.contiguous()
    B, C, H, W = xc.shape
    L = len(ksizes)
    out = torch.empty((B, C, L, H, W), device=x.device, dtype=x.dtype)
    host_taps = (ctypes.c_double * max(len(taps), 1))(*taps)
    host_k = (ctypes.c_int * L)(*ksizes)
    with torch.cuda.device(x.device), _Timed("scale_octave_forward", x):
        _lib.call("kb200_scale_octave_forward", _ptr(xc), host_taps, host_k, L, _ptr(out), B * C, H, W, _dtype_code(x), _stream(x))
    _bump()
    return out


_define("scale_octave_fwd", "(Tensor x, float[] taps, int[] ksizes) -> Tensor", _scale_octave_cuda,
        lambda x, taps, ksizes: x.new_empty((x.shape[0], x.shape[1], len(ksizes), x.shape[2], x.shape[3])))


def _dense_planes(x: torch.Tensor) -> torch.Tensor:
    """``x`` itself when each H x W plane is dense (the kernels take the outer strides), else a contiguous copy."""
    H, W = x.shape[-2:]
    if (W == 1 or x.stride(-1) == 1) and (H == 1 or x.stride(-2) == W):
        return x
    return x.contiguous()


def _nms2d_cuda(x, k, mask_only):
    _require_cuda(x, "input")
    B, C, H, W = x.shape
    out = torch.empty((B, C, H, W), device=x.device, dtype=torch.bool if mask_only else x.dtype)
    if out.numel() == 0:
        return out
    xs = _dense_planes(x)
    with torch.cuda.device(x.device), _Timed("nms2d_forward", x):
        _lib.call("kb200_nms2d_forward", _ptr(xs), _ptr(out), B, C, H, W, xs.stride(0), xs.stride(1), k, 0 if mask_only else 1,
                  _dtype_code(x), _stream(x))
    _bump()
    return out


_define("nms2d_fwd", "(Tensor x, int k, bool mask_only) -> Tensor", _nms2d_cuda,
        lambda x, k, mask_only: x.new_empty(x.shape, dtype=torch.bool if mask_only else x.dtype))

NMS3_MAX_MASK, NMS3_MAX_VALUES, NMS3_MINMAX = 0, 1, 2  # mode of kb200_nms3d_forward


def _nms3d_call(x, out0, out1, mode):
    _require_cuda(x, "input")
    if out0.numel() == 0:
        return
    B, C, L, H, W = x.shape
    xs = _dense_planes(x)
    with torch.cuda.device(x.device), _Timed("nms3d_forward", x):
        _lib.call("kb200_nms3d_forward", _ptr(xs), _ptr(out0), _ptr(out1), B, C, L, H, W, xs.stride(0), xs.stride(1), xs.stride(2), mode,
                  _dtype_code(x), _stream(x))
    _bump()


def _nms3d_cuda(x, mask_only):
    out = torch.empty(x.shape, device=x.device, dtype=torch.bool if mask_only else x.dtype)
    _nms3d_call(x, out, None, NMS3_MAX_MASK if mask_only else NMS3_MAX_VALUES)
    return out


def _nms3d_minmax_cuda(x):
    mx = torch.empty(x.shape, device=x.device, dtype=torch.bool)
    mn = torch.empty(x.shape, device=x.device, dtype=torch.bool)
    _nms3d_call(x, mx, mn, NMS3_MINMAX)
    return mx, mn


_define("nms3d_fwd", "(Tensor x, bool mask_only) -> Tensor", _nms3d_cuda,
        lambda x, mask_only: x.new_empty(x.shape, dtype=torch.bool if mask_only else x.dtype))
_define("nms3d_minmax_fwd", "(Tensor x) -> (Tensor, Tensor)", _nms3d_minmax_cuda,
        lambda x: (x.new_empty(x.shape, dtype=torch.bool), x.new_empty(x.shape, dtype=torch.bool)))


def _quad_interp3d_cuda(x, mask, n_iters, max_subpixel_shift, strict_maxima_bonus, dilation_radius, allow_scale_steps):
    """coords (B, C, 3, D, H, W) and y (the strides of x.clone()); ``dilation_radius`` 0 is the iterative form."""
    _require_cuda(x, "input")
    B, C, D, H, W = x.shape
    coords = torch.empty((B, C, 3, D, H, W), device=x.device, dtype=x.dtype)
    y = torch.empty_like(x)
    if x.numel() == 0:
        return coords, y
    xs = _dense_planes(x)
    radius = min(dilation_radius, max(D, H, W))  # a radius past the largest side reaches every voxel either way
    with torch.cuda.device(x.device), _Timed("quad_interp3d_forward", x):
        _lib.call("kb200_quad_interp3d_forward", _ptr(xs), _ptr(mask), _ptr(coords), _ptr(y), B, C, D, H, W, xs.stride(0), xs.stride(1),
                  xs.stride(2), *y.stride(), n_iters, radius, max_subpixel_shift, strict_maxima_bonus, strict_maxima_bonus > 0,
                  allow_scale_steps, _dtype_code(x), _stream(x))
    _bump()
    return coords, y


_define("quad_interp3d_fwd",
        "(Tensor x, Tensor? mask, int n_iters, float max_subpixel_shift, float strict_maxima_bonus, int dilation_radius, "
        "bool allow_scale_steps) -> (Tensor, Tensor)", _quad_interp3d_cuda,
        lambda x, mask, *_: (x.new_empty((x.shape[0], x.shape[1], 3) + tuple(x.shape[2:])), torch.empty_like(x)))


def _patches(x: torch.Tensor) -> torch.Tensor:
    """``x`` (N, 1, P, P) itself when its column stride is 1 (the kernels take the batch and row strides), else a copy."""
    return x if x.shape[-1] == 1 or x.stride(-1) == 1 else x.contiguous()


def _check_patch_args(x: torch.Tensor, weighting: torch.Tensor, what: str) -> None:
    """What the per-patch kernels read: (N, 1, P, P) patches and a P x P weighting of the patches' dtype and device."""
    if x.dim() != 4 or x.shape[1] != 1 or x.shape[2] != x.shape[3]:
        raise RuntimeError(f"kornia_b200: expected (N, 1, P, P) patches, got {tuple(x.shape)}")
    P = x.shape[-1]
    if weighting.numel() != P * P or weighting.shape[-2:] != (P, P):
        raise RuntimeError(f"kornia_b200: {what} must be {P} x {P} for {P} x {P} patches, got {tuple(weighting.shape)}")
    _fake_same_device(x, weighting)
    _same(x, weighting, what)


def _check_sift_args(x, gk, pk, num_ang_bins, num_spatial_bins, stride, pad) -> None:
    _check_patch_args(x, gk, "gk")
    K = pk.shape[-1]
    if pk.dim() < 2 or pk.shape[-2] != K or pk.numel() != K * K or K < 1:
        raise RuntimeError(f"kornia_b200: the pooling weights must be one square K x K kernel, got {tuple(pk.shape)}")
    _fake_same_device(x, pk)
    _same(x, pk, "the pooling weights")
    if num_ang_bins < 1 or num_spatial_bins < 1 or stride < 1 or pad < 0:
        raise RuntimeError(f"kornia_b200: bad SIFT configuration num_ang_bins={num_ang_bins} num_spatial_bins={num_spatial_bins} "
                           f"stride={stride} pad={pad}")


def _check_orientation_args(x, weighting, smooth, num_ang_bins) -> None:
    _check_patch_args(x, weighting, "weighting")
    if smooth.numel() != 5:
        raise RuntimeError(f"kornia_b200: the angular smoothing must have 5 taps, got {tuple(smooth.shape)}")
    _fake_same_device(x, smooth)
    _same(x, smooth, "the angular smoothing")
    if num_ang_bins < 1:
        raise RuntimeError(f"kornia_b200: bad num_ang_bins={num_ang_bins}")


def _sift_describe_cuda(x, gk, pk, num_ang_bins, num_spatial_bins, stride, pad, rootsift, clipval, eps):
    """(N, A * S * S) descriptors of the (N, 1, P, P) patches ``x``; ``gk`` the P x P weighting, ``pk`` the K x K pooling weights."""
    _require_cuda(x, "input")
    _check_sift_args(x, gk, pk, num_ang_bins, num_spatial_bins, stride, pad)
    N, P = x.shape[0], x.shape[-1]
    out = torch.empty((N, num_ang_bins * num_spatial_bins ** 2), device=x.device, dtype=x.dtype)
    if N == 0:
        return out
    xs, gkc, pkc = _patches(x), gk.contiguous(), pk.contiguous()
    with torch.cuda.device(x.device), _Timed("sift_describe_forward", x):
        _lib.call("kb200_sift_describe_forward", _ptr(xs), _ptr(gkc), _ptr(pkc), _ptr(out), N, P, xs.stride(0), xs.stride(-2), num_ang_bins,
                  num_spatial_bins, pkc.shape[-1], stride, pad, int(rootsift), clipval, eps, _dtype_code(x), _stream(x))
    _bump()
    return out


_define("sift_describe_fwd",
        "(Tensor x, Tensor gk, Tensor pk, int num_ang_bins, int num_spatial_bins, int stride, int pad, bool rootsift, float clipval, "
        "float eps) -> Tensor", _sift_describe_cuda,
        lambda x, gk, pk, num_ang_bins, num_spatial_bins, stride, pad, *_: (_check_sift_args(x, gk, pk, num_ang_bins, num_spatial_bins, stride, pad),
                                                                            x.new_empty((x.shape[0], num_ang_bins * num_spatial_bins ** 2)))[1])


def _patch_orientation_cuda(x, weighting, smooth, num_ang_bins, eps):
    """(N,) dominant gradient angles of the (N, 1, P, P) patches ``x``; ``smooth`` the 5 circular smoothing taps."""
    _require_cuda(x, "input")
    _check_orientation_args(x, weighting, smooth, num_ang_bins)
    N, P = x.shape[0], x.shape[-1]
    out = torch.empty((N,), device=x.device, dtype=x.dtype)
    if N == 0:
        return out
    xs, wc, sc = _patches(x), weighting.contiguous(), smooth.contiguous()
    with torch.cuda.device(x.device), _Timed("patch_orientation_forward", x):
        _lib.call("kb200_patch_orientation_forward", _ptr(xs), _ptr(wc), _ptr(sc), _ptr(out), N, P, xs.stride(0), xs.stride(-2), num_ang_bins,
                  eps, _dtype_code(x), _stream(x))
    _bump()
    return out


_define("patch_orientation_fwd", "(Tensor x, Tensor weighting, Tensor smooth, int num_ang_bins, float eps) -> Tensor",
        _patch_orientation_cuda,
        lambda x, weighting, smooth, num_ang_bins, eps: (_check_orientation_args(x, weighting, smooth, num_ang_bins), x.new_empty((x.shape[0],)))[1])


_PATCH_MAX_LEVELS = 32  # the kernel's level table (csrc/laf_patches.cuh)


def _check_patch_levels(levels, laf, PS: int, select_level: bool) -> None:
    """What the patch extraction kernel reads: 1..32 fp32 (B_l, C, h_l, w_l) levels of one batch and channel count, each
    the halving (h // 2, w // 2) of the one before, with a batch of at least the LAFs'; fp32 (B, N, 2, 3) LAFs on the same
    device; PS >= 1.  Without level selection exactly one level (the image)."""
    if len(levels) < 1 or len(levels) > _PATCH_MAX_LEVELS or (not select_level and len(levels) != 1):
        raise RuntimeError(f"kornia_b200: expected 1..{_PATCH_MAX_LEVELS} pyramid levels (1 without level selection), got {len(levels)}")
    if laf.dim() != 4 or tuple(laf.shape[2:]) != (2, 3):
        raise RuntimeError(f"kornia_b200: expected (B, N, 2, 3) LAFs, got {tuple(laf.shape)}")
    if PS < 1:
        raise RuntimeError(f"kornia_b200: bad patch size {PS}")
    x0 = levels[0]
    for l, x in enumerate(levels):
        if x.dim() != 4:
            raise RuntimeError(f"kornia_b200: pyramid level {l} must be (B, C, H, W), got {tuple(x.shape)}")
        if x.shape[0] != x0.shape[0] or x.shape[1] != x0.shape[1]:
            raise RuntimeError(f"kornia_b200: pyramid level {l} {tuple(x.shape)} does not share level 0's batch and channels {tuple(x0.shape[:2])}")
        if l > 0 and (x.shape[2] != levels[l - 1].shape[2] // 2 or x.shape[3] != levels[l - 1].shape[3] // 2):
            raise RuntimeError(f"kornia_b200: pyramid level {l} {tuple(x.shape[2:])} is not the halving of level {l - 1} "
                               f"{tuple(levels[l - 1].shape[2:])}")
        _fake_same_device(laf, x)
        _same(x0, x, f"pyramid level {l}")
    if x0.shape[0] < laf.shape[0]:
        raise RuntimeError(f"kornia_b200: {laf.shape[0]} LAF sets for {x0.shape[0]} images")
    _fake_same_device(x0, laf)
    _same(x0, laf, "the LAFs")


def _affine_base(PS: int, device) -> torch.Tensor:
    """affine_grid's base coordinates (align_corners=False) as ATen builds them on ``device``: linspace(-1, 1, PS) *
    (PS - 1) / PS, or 0 for PS = 1.  Built once per (PS, device) with those torch ops, so they are ATen's values bit for bit."""
    from .geometry._prelude import _cached

    def build():
        if PS <= 1:
            return torch.zeros(1, device=device)
        return torch.linspace(-1, 1, PS, device=device) * (PS - 1) / PS

    return _cached(("laf_patch_base", PS, str(device)), build)


def _extract_patches_cuda(levels, laf, PS, normalize, select_level):
    """(B, N, C, PS, PS) patches at the LAFs ``laf`` (B, N, 2, 3), sampled from ``levels`` (the image, then its pyrdowns)."""
    _require_cuda(laf, "the LAFs")
    _check_patch_levels(levels, laf, PS, select_level)
    B, N, C = laf.shape[0], laf.shape[1], levels[0].shape[1]
    out = torch.empty((B, N, C, PS, PS), device=laf.device, dtype=laf.dtype)
    if B * N == 0:
        return out
    lv = [x if x.shape[-1] == 1 or x.stride(-1) == 1 else x.contiguous() for x in levels]
    lafc = laf.contiguous()
    base = _affine_base(PS, laf.device)
    ptrs = (ctypes.c_void_p * len(lv))(*[x.data_ptr() for x in lv])
    dims = (ctypes.c_longlong * (5 * len(lv)))(*[v for x in lv for v in (x.shape[2], x.shape[3], x.stride(0), x.stride(1),
                                                                         x.stride(2) if x.shape[2] > 1 else x.shape[3])])
    with torch.cuda.device(laf.device), _Timed("extract_patches_forward", laf):
        _lib.call("kb200_extract_patches_forward", ptrs, dims, len(lv), _ptr(lafc), _ptr(base), _ptr(out), B, N, C, PS, int(normalize),
                  int(select_level), _dtype_code(laf), _stream(laf))
    _bump()
    return out


_define("extract_patches_fwd", "(Tensor[] levels, Tensor laf, int PS, bool normalize, bool select_level) -> Tensor", _extract_patches_cuda,
        lambda levels, laf, PS, normalize, select_level: (_check_patch_levels(levels, laf, PS, select_level),
                                                          laf.new_empty((laf.shape[0], laf.shape[1], levels[0].shape[1], PS, PS)))[1],
        first_tensor="the LAFs")


def _patch_affine_shape_cuda(x, weighting, eps):
    """(N, 1, 3) normalised second-moment shapes (a, b, c) of the (N, 1, P, P) patches ``x``."""
    _require_cuda(x, "input")
    _check_patch_args(x, weighting, "weighting")
    N, P = x.shape[0], x.shape[-1]
    out = torch.empty((N, 1, 3), device=x.device, dtype=x.dtype)
    if N == 0:
        return out
    xs, wc = _patches(x), weighting.contiguous()
    with torch.cuda.device(x.device), _Timed("patch_affine_shape_forward", x):
        _lib.call("kb200_patch_affine_shape_forward", _ptr(xs), _ptr(wc), _ptr(out), N, P, xs.stride(0), xs.stride(-2), eps, _dtype_code(x),
                  _stream(x))
    _bump()
    return out


_define("patch_affine_shape_fwd", "(Tensor x, Tensor weighting, float eps) -> Tensor", _patch_affine_shape_cuda,
        lambda x, weighting, eps: (_check_patch_args(x, weighting, "weighting"), x.new_empty((x.shape[0], 1, 3)))[1])


def _check_laf_affine_args(levels, laf, weighting, PS: int) -> None:
    """The patch extraction's levels and LAFs (one channel), and a PS x PS weighting of their dtype and device."""
    _check_patch_levels(levels, laf, PS, True)
    if levels[0].shape[1] != 1:
        raise RuntimeError(f"kornia_b200: the affine shape is estimated on one-channel images, got {levels[0].shape[1]} channels")
    if weighting.numel() != PS * PS or weighting.shape[-2:] != (PS, PS):
        raise RuntimeError(f"kornia_b200: weighting must be {PS} x {PS}, got {tuple(weighting.shape)}")
    _fake_same_device(laf, weighting)
    _same(laf, weighting, "weighting")


def _laf_affine_shape_cuda(levels, laf, weighting, PS, eps, preserve_orientation):
    """(B, N, 2, 3) LAFs of ``laf`` with the affine shape estimated on ``levels`` (the image, then its pyrdowns)."""
    _require_cuda(laf, "the LAFs")
    _check_laf_affine_args(levels, laf, weighting, PS)
    B, N = laf.shape[0], laf.shape[1]
    out = torch.empty((B, N, 2, 3), device=laf.device, dtype=laf.dtype)
    if B * N == 0:
        return out
    lv = [x if x.shape[-1] == 1 or x.stride(-1) == 1 else x.contiguous() for x in levels]
    lafc, wc = laf.contiguous(), weighting.contiguous()
    base = _affine_base(PS, laf.device)
    ptrs = (ctypes.c_void_p * len(lv))(*[x.data_ptr() for x in lv])
    dims = (ctypes.c_longlong * (5 * len(lv)))(*[v for x in lv for v in (x.shape[2], x.shape[3], x.stride(0), x.stride(1),
                                                                         x.stride(2) if x.shape[2] > 1 else x.shape[3])])
    with torch.cuda.device(laf.device), _Timed("laf_affine_shape_forward", laf):
        _lib.call("kb200_laf_affine_shape_forward", ptrs, dims, len(lv), _ptr(lafc), _ptr(base), _ptr(wc), _ptr(out), B, N, PS, eps,
                  int(preserve_orientation), _dtype_code(laf), _stream(laf))
    _bump()
    return out


_define("laf_affine_shape_fwd", "(Tensor[] levels, Tensor laf, Tensor weighting, int PS, float eps, bool preserve_orientation) -> Tensor",
        _laf_affine_shape_cuda,
        lambda levels, laf, weighting, PS, eps, preserve_orientation: (_check_laf_affine_args(levels, laf, weighting, PS),
                                                                        laf.new_empty((laf.shape[0], laf.shape[1], 2, 3)))[1],
        first_tensor="the LAFs")


def _sepfilter_lerp_cuda(x, kx, ky, border, weight):
    _require_cuda(x, "input")
    xc, kxc, kyc = x.contiguous(), kx.contiguous(), ky.contiguous()
    B, C, H, W = xc.shape
    out = torch.empty_like(xc)
    with torch.cuda.device(x.device), _Timed("sepfilter_lerp_forward", x):
        _lib.call("kb200_sepfilter_lerp_forward", _ptr(xc), _ptr(kxc), _ptr(kyc), _ptr(out), B, C, H, W, kxc.shape[0], kxc.shape[1], kyc.shape[0],
                  kyc.shape[1], border, 1, float(weight), _dtype_code(x), _stream(x))
    _bump()
    return out


_define("sepfilter_lerp_fwd", "(Tensor x, Tensor kx, Tensor ky, int border, float weight) -> Tensor", _sepfilter_lerp_cuda,
        lambda x, kx, ky, border, weight: (_fake_same_device(x, kx, ky), torch.empty_like(x, memory_format=torch.contiguous_format))[1], "input")


def _pyrdown_cuda(x, kernel, border):
    _require_cuda(x, "input")
    xc, kc = x.contiguous(), kernel.contiguous()
    B, C, H, W = xc.shape
    out = torch.empty((B, C, H // 2, W // 2), device=x.device, dtype=x.dtype)
    if out.numel() == 0:
        raise _lib.Unsupported("empty output")
    with torch.cuda.device(x.device), _Timed("pyrdown_forward", x):
        _lib.call("kb200_pyrdown_forward", _ptr(xc), _ptr(kc), _ptr(out), B, C, H, W, kc.shape[0], border, _dtype_code(x), _stream(x))
    _bump()
    return out


_define("pyrdown_fwd", "(Tensor x, Tensor kernel, int border) -> Tensor", _pyrdown_cuda,
        lambda x, kernel, border: (_fake_same_device(x, kernel), x.new_empty((x.shape[0], x.shape[1], x.shape[2] // 2, x.shape[3] // 2)))[1], "input")


def pyrdown_fused(x: torch.Tensor, kernel: torch.Tensor, border: int) -> torch.Tensor:
    """5x5 correlation + exact 2x bilinear decimation in one kernel (forward only): (B,C,H,W) -> (B,C,H/2,W/2).
    Raises ``_lib.Unsupported`` outside the kernel's envelope (the caller then composes filter2d + interpolate)."""
    return ops.pyrdown_fwd(x, kernel, int(border))


def _undistort_cuda(image, lens):
    _require_cuda(image, "image")
    img, ln = image.contiguous(), lens.to(device=image.device, dtype=image.dtype).contiguous()
    B, C, H, W = img.shape
    out = torch.empty_like(img)
    if out.numel() == 0:
        raise _lib.Unsupported("empty image")
    with torch.cuda.device(image.device), _Timed("undistort_forward", image):
        _lib.call("kb200_undistort_forward", _ptr(img), _ptr(ln), _ptr(out), B, C, H, W, _dtype_code(image), _stream(image))
    _bump()
    return out


_define("undistort_fwd", "(Tensor image, Tensor lens) -> Tensor", _undistort_cuda,
        lambda image, lens: torch.empty_like(image, memory_format=torch.contiguous_format), "image")


def undistort_fused(image: torch.Tensor, lens: torch.Tensor) -> torch.Tensor:
    """Lens model + bilinear resampling in one kernel (forward only): image (B,C,H,W), lens (B,16).  Raises
    ``_lib.Unsupported`` outside the kernel's envelope (the caller then builds the maps and calls remap)."""
    return ops.undistort_fwd(image, lens)


# ---------------------------------------------------------------------------------------------
# wire format in front of the path: interleaved uint8 (B,H,W,C) in, planar fp32 (B,C,h,w) out
# ---------------------------------------------------------------------------------------------
def _warp_u8_cuda(image, m, bx, by, fill, h, w, projective, interp, pad, align, normalize):
    _require_cuda(image, "image")
    if image.dtype != torch.uint8:
        raise RuntimeError(f"kornia_b200: expected a uint8 image, got {image.dtype}")
    if m.device != image.device:
        raise RuntimeError(f"Expected all tensors to be on the same device, but the transformation matrix is on {m.device} and the image on {image.device}")
    img = image.contiguous()
    f32 = dict(device=image.device, dtype=torch.float32)
    m_c, bx, by = m.to(**f32).contiguous(), bx.to(**f32).contiguous(), by.to(**f32).contiguous()
    fill_c = None if fill is None else fill.to(**f32).contiguous()
    B, H, W, C = img.shape
    out = torch.empty((B, C, h, w), **f32)
    if out.numel() > 0 and img.numel() > 0:
        with torch.cuda.device(image.device), _Timed("warp_u8hwc_forward", image):
            _lib.call("kb200_warp_u8hwc_forward", _ptr(img), _ptr(m_c), _ptr(bx), _ptr(by), _ptr(fill_c), _ptr(out), B, C, H, W, h, w,
                      m_c.shape[0], int(projective), interp, pad, int(align), int(normalize), _stream(image))
        _bump()
    else:
        out.zero_()
    return out


_define("warp_u8hwc_fwd", "(Tensor image, Tensor m, Tensor bx, Tensor by, Tensor? fill, int h, int w, bool projective, int interp, int pad, "
        "bool align, int normalize) -> Tensor", _warp_u8_cuda,
        lambda image, m, bx, by, fill, h, w, projective, interp, pad, align, normalize:
        (_fake_same_device(image, m), image.new_empty((image.shape[0], image.shape[3], h, w), dtype=torch.float32))[1], "image")


def warp_u8hwc(image, m, bx, by, fill, h, w, projective, interp, pad, align, normalize) -> torch.Tensor:
    """Warp of an interleaved uint8 batch (B,H,W,C) into planar fp32 (B,C,h,w) in one kernel (kb200_warp_u8hwc_forward):
    the bytes are converted inside the sampler (``normalize``: 0 raw, 1 times 1/255 as torch's CUDA backend does,
    2 divided by 255).  ``m`` is the (B|1,3,3) fp32 sampling matrix of the warp prelude.  Forward only."""
    return ops.warp_u8hwc_fwd(image, m, bx, by, fill, int(h), int(w), bool(projective), int(interp), int(pad), bool(align), int(normalize))


def _undistort_u8_cuda(image, lens, normalize):
    _require_cuda(image, "image")
    if image.dtype != torch.uint8:
        raise RuntimeError(f"kornia_b200: expected a uint8 image, got {image.dtype}")
    img = image.contiguous()
    ln = lens.to(device=image.device, dtype=torch.float32).contiguous()
    B, H, W, C = img.shape
    out = torch.empty((B, C, H, W), device=image.device, dtype=torch.float32)
    if out.numel() == 0:
        raise _lib.Unsupported("empty image")
    with torch.cuda.device(image.device), _Timed("undistort_u8hwc_forward", image):
        _lib.call("kb200_undistort_u8hwc_forward", _ptr(img), _ptr(ln), _ptr(out), B, C, H, W, int(normalize), _stream(image))
    _bump()
    return out


_define("undistort_u8hwc_fwd", "(Tensor image, Tensor lens, int normalize) -> Tensor", _undistort_u8_cuda,
        lambda image, lens, normalize: image.new_empty((image.shape[0], image.shape[3], image.shape[1], image.shape[2]), dtype=torch.float32), "image")


def undistort_u8hwc(image: torch.Tensor, lens: torch.Tensor, normalize: int) -> torch.Tensor:
    """undistort_image of an interleaved uint8 batch (B,H,W,C) -> planar fp32 (B,C,H,W) in one kernel; lens (B,16) as for
    undistort_fused.  Raises ``_lib.Unsupported`` outside the kernel's envelope.  Forward only."""
    return ops.undistort_u8hwc_fwd(image, lens, int(normalize))


# ---------------------------------------------------------------------------------------------
# one-launch matrix builders of the callers (get_rotation_matrix2d, get_perspective_transform)
# ---------------------------------------------------------------------------------------------
def _rotation_cuda(center, angle, scale):
    _require_cuda(center, "center")
    c, a, s = center.contiguous(), angle.contiguous(), scale.contiguous()
    out = torch.empty((c.shape[0], 2, 3), device=c.device, dtype=c.dtype)
    if out.numel() > 0:
        with torch.cuda.device(c.device):
            _lib.call("kb200_rotation_matrix2d", _ptr(c), _ptr(a), _ptr(s), _ptr(out), c.shape[0], _dtype_code(c), FUSED_VARIANT, _stream(c))
        _bump()
    return out


_define("rotation_matrix2d", "(Tensor center, Tensor angle, Tensor scale) -> Tensor", _rotation_cuda,
        lambda center, angle, scale: (_fake_same_device(center, angle, scale), center.new_empty((center.shape[0], 2, 3)))[1], "center")


def _perspective_cuda(points_src, points_dst):
    _require_cuda(points_src, "points_src")
    ps, pd = points_src.contiguous(), points_dst.contiguous()
    out = torch.empty((ps.shape[0], 3, 3), device=ps.device, dtype=ps.dtype)
    if out.numel() > 0:
        with torch.cuda.device(ps.device):
            _lib.call("kb200_perspective_from_points", _ptr(ps), _ptr(pd), _ptr(out), ps.shape[0], _dtype_code(ps), FUSED_VARIANT, _stream(ps))
        _bump()
    return out


_define("perspective_from_points", "(Tensor points_src, Tensor points_dst) -> Tensor", _perspective_cuda,
        lambda points_src, points_dst: (_fake_same_device(points_src, points_dst), points_src.new_empty((points_src.shape[0], 3, 3)))[1], "points_src")


# ---------------------------------------------------------------------------------------------
# names of round 1 (``X.apply(...)``), kept for tools/ and tests that call the bridges directly
# ---------------------------------------------------------------------------------------------
class _Apply:
    def __init__(self, fn):
        self.apply = fn


WarpFunction = _Apply(warp)
RemapFunction = _Apply(remap)
Filter2dFunction = _Apply(filter2d)
SepFilterFunction = _Apply(sepfilter)
SpatialGradientFunction = _Apply(spatial_gradient)

OPERATORS: Tuple[str, ...] = (
    "warp_fwd", "warp_bwd", "warp_prelude", "warp_prelude_bwd", "remap_fwd", "remap_bwd", "filter2d_fwd", "filter2d_bwd_input",
    "filter2d_bwd_kernel", "sepfilter_fwd", "spatial_gradient_fwd", "spatial_gradient_bwd", "ssim_fwd", "sepfilter_lerp_fwd", "pyrdown_fwd",
    "undistort_fwd", "warp_u8hwc_fwd", "undistort_u8hwc_fwd", "rotation_matrix2d", "perspective_from_points", "feature_response_fwd",
    "scale_octave_fwd", "nms2d_fwd", "nms3d_fwd", "nms3d_minmax_fwd", "quad_interp3d_fwd", "sift_describe_fwd",
    "patch_orientation_fwd", "extract_patches_fwd", "patch_affine_shape_fwd", "laf_affine_shape_fwd",
)
