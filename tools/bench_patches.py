"""extract_patches_from_pyramid on the H100: the fused path (this library's pyrdown for the sampled levels, then the
kernel of csrc/laf_patches.cuh) against the library composition (``_composed_extract_pyramid``) and the reference's op
sequence restated over ATen (the same composition over the oracle's ``pyrdown``: F.pad + F.conv2d + F.interpolate).

    python tools/bench_patches.py [--reps 7] [--out results/bench_patches.jsonl]

Workloads, fp32 under torch.inference_mode(), uniform-noise images, LAFs with random rotation, shear, anisotropy and
log-uniform scales over the built levels: 1x1x1080x1920 with N = 8000 at PS = 19 and 41, 8x3x480x640 with N = 2000 per
image at PS = 32, and 1x1x1080x1920 with N = 65536 at PS = 41.  Per call CUDA events after a warm-up, the three arms
alternated call by call, medians reported.  ``kernel_ms`` times the extraction operator alone on prebuilt levels;
``call_ms`` the public call, pyrdowns included.  ``of_hbm_roofline`` is the time to write the B*N*C*PS*PS output once at
3.35 TB/s over ``kernel_ms``.  Each row states the largest difference between the fused and the composed patches.  The
card's name and power limit are printed first."""
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
from kornia_b200.feature import laf as LAF  # noqa: E402
from oracle import kornia_restated as R  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


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


def reference(img, laf, PS):
    saved = LAF.pyrdown
    LAF.pyrdown = R.pyrdown
    try:
        return LAF._composed_extract_pyramid(img, laf, PS, True)
    finally:
        LAF.pyrdown = saved


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    print(json.dumps({"card": card()}))
    rows = []
    for B, C, h, w, N, PS in [(1, 1, 1080, 1920, 8000, 19), (1, 1, 1080, 1920, 8000, 41), (8, 3, 480, 640, 2000, 32),
                              (1, 1, 1080, 1920, 65536, 41)]:
        gen = torch.Generator().manual_seed(N + PS)
        img = torch.rand(B, C, h, w, generator=gen).cuda()
        laf = lafs(B, N, h, w, PS, gen)
        with torch.inference_mode():
            levels = [img]
            for _ in range(LAF._built_levels(h, w, PS) - 1):
                levels.append(LAF.pyrdown(levels[-1]))
            fused = LAF.extract_patches_from_pyramid(img, laf, PS)
            comp = LAF._composed_extract_pyramid(img, laf, PS, True)
            diff = float((fused - comp).abs().max())
            del comp
            arms = {"kernel": lambda: _ops.ops.extract_patches_fwd(levels, laf, PS, True, True),
                    "fused": lambda: LAF.extract_patches_from_pyramid(img, laf, PS),
                    "composition": lambda: LAF._composed_extract_pyramid(img, laf, PS, True),
                    "reference": lambda: reference(img, laf, PS)}
            for fn in arms.values():
                fn()
            times = {k: [] for k in arms}
            for r in range(args.reps):
                order = list(arms)[r % 4:] + list(arms)[: r % 4]
                for k in order:
                    times[k].append(timed(arms[k]))
        med = {k: statistics.median(v) for k, v in times.items()}
        floor_ms = B * N * C * PS * PS * 4 / HBM_BYTES_PER_S * 1e3
        row = {"workload": f"{B}x{C}x{h}x{w} N={N} PS={PS}", "levels": len(levels), "kernel_ms": round(med["kernel"], 4),
               "call_ms": round(med["fused"], 4), "composition_ms": round(med["composition"], 4), "reference_ms": round(med["reference"], 4),
               "speedup_vs_reference": round(med["reference"] / med["fused"], 1), "speedup_vs_composition": round(med["composition"] / med["fused"], 1),
               "of_hbm_roofline": round(floor_ms / med["kernel"], 3), "max_abs_diff_vs_composition": diff}
        rows.append(row)
        print(json.dumps(row), flush=True)
        del img, laf, levels, fused
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "a") as f:
            for row in rows:
                f.write(json.dumps(row) + "\n")


if __name__ == "__main__":
    main()
