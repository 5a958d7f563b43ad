"""Feature responses on the H100: the fused kernels (csrc/corner_vwalk.cuh for Harris / GFTT, grad_tiled_kernel's Hessian
epilogue) against the library composition (this library's spatial_gradient / gaussian_blur2d + torch ops, ``_composed_*``)
and the reference composition (tests/responses_restated.py: F.pad + F.conv2d + torch ops) on the same GPU.

    python tools/bench_responses.py [--shapes 64x1 32x3] [--reps 7] [--out results/bench_responses.jsonl]

Workload: B x C x 1080 x 1920 fp32 with the default arguments ('sobel', k = 0.04, no sigmas).  Per-call CUDA events after a
warm-up, the three arms alternated call by call (their order rotated from repeat to repeat), the median reported; the fused
output is compared bit for bit with the library composition at every size timed.  HBM floor: ``out.copy_(x)`` on the same
tensors (8 B per element: 4 read, 4 written), measured in the same call.  The card's name and power limit are printed first."""
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

import kornia_b200 as K  # noqa: E402
import responses_restated as RR  # noqa: E402
from kornia_b200.feature import responses as FR  # noqa: E402

# FMAs per output element of the fused kernels (operation counts behind DESIGN.md's bound): Harris / GFTT compute both 3x3
# stencils (18 FMAs, zeros included) at 10 positions per 4 outputs, 3 products, 7-tap row sums and column sums of 3 planes
FMA_PER_ELEMENT = {"harris": 18 * 10 / 4 + 3 * 10 / 4 + 3 * 7 + 3 * 7, "gftt": 18 * 10 / 4 + 3 * 10 / 4 + 3 * 7 + 3 * 7,
                   "hessian_sobel": 3 * 25}
FP32_FMA_PER_S = 67e12 / 2  # H100 SXM data sheet, dense fp32
HBM_BYTES_PER_S = 3.35e12


def card() -> dict:
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
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


ARMS = {
    "harris": (lambda x: K.feature.harris_response(x), lambda x: FR._composed_harris(x, 0.04, "sobel", None), lambda x: RR.harris_response(x)),
    "gftt": (lambda x: K.feature.gftt_response(x), lambda x: FR._composed_gftt(x, "sobel", None), lambda x: RR.gftt_response(x)),
    "hessian": (lambda x: K.feature.hessian_response(x), lambda x: FR._composed_hessian(x, "sobel", None), lambda x: RR.hessian_response(x)),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", nargs="+", default=["64x1", "32x3"])
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_responses needs a GPU"
    print(json.dumps({"card": card()}), flush=True)
    H, W = 1080, 1920
    rows = []
    gen = torch.Generator(device="cuda").manual_seed(0)
    for shape in args.shapes:
        B, C = (int(v) for v in shape.split("x"))
        x = torch.rand(B, C, H, W, device="cuda", generator=gen)
        out = torch.empty_like(x)
        n = x.numel()
        with torch.no_grad():
            for name, (fused, lib, ref) in ARMS.items():
                a, b = fused(x), lib(x)
                same = bool(((a.view(torch.int32) == b.view(torch.int32)) | (a.isnan() & b.isnan())).all())
                del a, b
                ref(x)
                arms = {"fused": fused, "library_composition": lib, "reference_composition": ref, "copy_floor": lambda t: out.copy_(t)}
                times = {k: [] for k in arms}
                order = list(arms)
                for r in range(args.reps):
                    for k in order[r % len(order):] + order[:r % len(order)]:
                        times[k].append(timed(lambda: arms[k](x)))
                med = {k: statistics.median(v) for k, v in times.items()}
                fkey = "hessian_sobel" if name == "hessian" else name
                fma_bound = n * FMA_PER_ELEMENT[fkey] / FP32_FMA_PER_S * 1e3
                hbm_bound = n * 8 / HBM_BYTES_PER_S * 1e3
                row = {"fn": name, "shape": [B, C, H, W], "bit_identical": same, "ms": {k: round(v, 4) for k, v in med.items()},
                       "ms_all": {k: [round(t, 4) for t in v] for k, v in times.items()},
                       "speedup_vs_library": round(med["library_composition"] / med["fused"], 2),
                       "speedup_vs_reference": round(med["reference_composition"] / med["fused"], 2),
                       "datasheet_bounds_ms": {"hbm": round(hbm_bound, 4), "fp32_fma": round(fma_bound, 4)}}
                print(json.dumps(row), flush=True)
                rows.append(row)
                torch.cuda.empty_cache()
        del x, out
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for row in rows:
                f.write(json.dumps(row) + "\n")


if __name__ == "__main__":
    main()
