"""LAFAffineShapeEstimator and PatchAffineShapeEstimator on the H100: the fused paths (csrc/affine_shape.cuh) against the
library composition and the reference's op sequence restated over ATen.

    python tools/bench_affine_shape.py [--reps 7] [--out results/bench_affine_shape.jsonl]

LAF workloads, fp32 under torch.inference_mode(), uniform-noise images, LAFs with random rotation, shear, anisotropy and
log-uniform scales over the built levels: LAFAffineShapeEstimator(32) at 1x1x1080x1920 with N = 8000 and 65536, and at
8x1x480x640 with N = 2000 per image.  Arms: ``call`` the public call (pyrdowns included), ``kernel`` the operator alone on
prebuilt levels, ``composition`` ``_composed_laf_affine_shape`` (its extraction and patch estimator take their own fused
kernels), ``reference`` the reference's sequence over ATen (the oracle's pyrdown, ``grid_sample`` extraction, the
patch estimator's composition over ATen's conv2d gradient, ``torch.inverse``).  To tell sampling from reduction, each row
also times the extraction kernel alone (``extract_kernel_ms``: sampling plus writing the patch stack) and the patch
estimator kernel alone on that stack (``patch_kernel_ms``: staging plus the reduction).

Patch workloads: PatchAffineShapeEstimator(19 / 32) on N = 8000 and 65536 noise patches; arms ``kernel``, ``composition``
and ``reference``.  Per call CUDA events after a warm-up, the arms alternated call by call, medians reported.  Each row
states the largest difference between the fused and the composed result.  The card's name and power limit are printed
first."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from kornia_b200 import _ops  # noqa: E402
from kornia_b200.feature import affine_shape as AS  # noqa: E402
from kornia_b200.feature import laf as LAF  # noqa: E402
from oracle import kornia_restated as R  # noqa: E402


def card() -> dict:
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        info["power_limit_and_max_sm_clock"] = q.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        info["power_limit_and_max_sm_clock"] = f"unavailable ({e})"
    return info


def timed(fn) -> float:
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e)


def lafs(B, N, h, w, PS, gen):
    top = LAF._built_levels(h, w, PS) - 1
    u = torch.rand(B, N, generator=gen) * (top + 2.0) - 1.0
    s = torch.pow(2.0, u) * PS / 2.0
    ang = torch.rand(B, N, generator=gen) * 6.283185307
    r = torch.exp(torch.randn(B, N, generator=gen) * 0.3)
    sh = torch.randn(B, N, generator=gen) * 0.2
    c, si = torch.cos(ang), torch.sin(ang)
    A = torch.stack([torch.stack([c * r.sqrt(), c * sh - si / r.sqrt()], -1),
                     torch.stack([si * r.sqrt(), si * sh + c / r.sqrt()], -1)], -2) * s[..., None, None]
    cx, cy = torch.rand(B, N, generator=gen) * (w - 1), torch.rand(B, N, generator=gen) * (h - 1)
    return torch.cat([A, torch.stack([cx, cy], -1)[..., None]], -1).cuda()


class _AtenSobel(torch.nn.Module):
    def forward(self, x):
        return R.spatial_gradient(x, "sobel", 1, True)


def reference_patch(det, patches):
    """PatchAffineShapeEstimator's op sequence with ATen's conv2d Sobel gradient."""
    saved = det.gradient
    det.gradient = _AtenSobel()
    try:
        return AS._composed_patch_affine_shape(det, patches)
    finally:
        det.gradient = saved


def reference_laf(m, laf, img):
    """LAFAffineShapeEstimator's op sequence over ATen: the oracle's pyrdown, the grid_sample extraction, the patch
    estimator over conv2d."""
    PS, det = m.patch_size, m.affine_shape_detector
    saved = LAF.pyrdown
    LAF.pyrdown = R.pyrdown
    try:
        B, N = laf.shape[:2]
        patches = LAF._composed_extract_pyramid(img, LAF.make_upright(laf), PS, True).view(-1, 1, PS, PS)
    finally:
        LAF.pyrdown = saved
    ellipse_shape = reference_patch(det, patches)
    ellipses = torch.cat([laf.view(-1, 2, 3)[..., 2].unsqueeze(1), ellipse_shape], dim=2).view(B, N, 5)
    scale_orig, ori_orig = LAF.get_laf_scale(laf), LAF.get_laf_orientation(laf)
    out = LAF.ellipse_to_laf(ellipses)
    out = LAF.scale_laf(out, scale_orig / LAF.get_laf_scale(out))
    return LAF.set_laf_orientation(out, ori_orig)


def run(arms, reps):
    for fn in arms.values():
        fn()
    times = {k: [] for k in arms}
    for r in range(reps):
        order = list(arms)[r % len(arms):] + list(arms)[: r % len(arms)]
        for k in order:
            times[k].append(timed(arms[k]))
    return {k: statistics.median(v) for k, v in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    print(json.dumps({"card": card()}))
    rows = []
    PS = 32
    for B, h, w, N in [(1, 1080, 1920, 8000), (1, 1080, 1920, 65536), (8, 480, 640, 2000)]:
        gen = torch.Generator().manual_seed(N + B)
        img = torch.rand(B, 1, h, w, generator=gen).cuda()
        laf = lafs(B, N, h, w, PS, gen)
        m = AS.LAFAffineShapeEstimator(PS).cuda()
        det = m.affine_shape_detector
        with torch.inference_mode():
            fused = m(laf, img)
            levels = [img]
            for _ in range(LAF._built_levels(h, w, PS) - 1):
                levels.append(LAF.pyrdown(levels[-1]))
            comp = AS._composed_laf_affine_shape(m, laf, img)
            diff = float((fused - comp).abs().max())
            del comp
            up = LAF.make_upright(laf)
            stack = _ops.ops.extract_patches_fwd(levels, up, PS, True, True).view(-1, 1, PS, PS)
            arms = {"kernel": lambda: _ops.ops.laf_affine_shape_fwd(levels, laf, det.weighting, PS, float(det.eps), True),
                    "call": lambda: m(laf, img),
                    "composition": lambda: AS._composed_laf_affine_shape(m, laf, img),
                    "reference": lambda: reference_laf(m, laf, img),
                    "extract_kernel": lambda: _ops.ops.extract_patches_fwd(levels, up, PS, True, True),
                    "patch_kernel": lambda: _ops.ops.patch_affine_shape_fwd(stack, det.weighting, float(det.eps))}
            med = run(arms, args.reps)
        row = {"workload": f"LAFAffineShapeEstimator({PS}) {B}x1x{h}x{w} N={N}", "levels": len(levels), "kernel_ms": round(med["kernel"], 4),
               "call_ms": round(med["call"], 4), "composition_ms": round(med["composition"], 4), "reference_ms": round(med["reference"], 4),
               "speedup_vs_reference": round(med["reference"] / med["call"], 1),
               "speedup_vs_composition": round(med["composition"] / med["call"], 1), "extract_kernel_ms": round(med["extract_kernel"], 4),
               "patch_kernel_ms": round(med["patch_kernel"], 4), "max_abs_diff_vs_composition": diff}
        rows.append(row)
        print(json.dumps(row), flush=True)
        del img, laf, levels, fused, stack, up
        torch.cuda.empty_cache()
    for P in (19, 32):
        for N in (8000, 65536):
            gen = torch.Generator().manual_seed(N + P)
            x = torch.rand(N, 1, P, P, generator=gen).cuda()
            det = AS.PatchAffineShapeEstimator(P).cuda()
            with torch.inference_mode():
                fused = det(x)
                diff = float((fused - AS._composed_patch_affine_shape(det, x)).abs().max())
                med = run({"kernel": lambda: det(x), "composition": lambda: AS._composed_patch_affine_shape(det, x),
                           "reference": lambda: reference_patch(det, x)}, args.reps)
            row = {"workload": f"PatchAffineShapeEstimator({P}) N={N}", "kernel_ms": round(med["kernel"], 4),
                   "composition_ms": round(med["composition"], 4), "reference_ms": round(med["reference"], 4),
                   "speedup_vs_reference": round(med["reference"] / med["kernel"], 1), "max_abs_diff_vs_composition": diff}
            rows.append(row)
            print(json.dumps(row), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "a") as f:
            for row in rows:
                f.write(json.dumps(row) + "\n")


if __name__ == "__main__":
    main()
