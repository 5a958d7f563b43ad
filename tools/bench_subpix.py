"""Sub-pixel refinement on the H100: the fused kernel (csrc/quad_interp.cuh) against the library composition
(``_composed_*`` of kornia_b200/geometry/subpix/quad_interp.py, the reference's op sequence).

    python tools/bench_subpix.py [--reps 7] [--out results/bench_subpix.jsonl]

Workloads, fp32, no gradient, on BlobHessian responses of ScalePyramid octaves (hessian_response of each blur level times
sigma^4, the levels of one octave as (B, 1, 5, 1080, 1920)) for B = 1 and 16: conv_quad_interp3d with nms3d_minmax's
max mask (ScaleSpaceDetector's default refiner on CUDA), conv_quad_interp3d computing its own NMS, and
iterative_quad_interp3d.  Per-call CUDA events after a warm-up, the two arms alternated call by call (order rotated from
repeat to repeat), the median reported.  Every fused result is compared bit for bit with the composition in the same
run.  Floor: 21 B per element (4 B read, 1 B of mask, 16 B written) at the data sheet's 3.35 TB/s, computed from shapes,
not measured.  The card's name and power limit are printed first."""
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

import kornia_b200 as K  # noqa: E402
from kornia_b200.geometry.subpix import quad_interp as Q  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
FLOOR_BYTES_PER_ELEMENT = 21


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


def timed(fn) -> float:
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e)


def blob_octave(B: int, g: torch.Generator) -> torch.Tensor:
    """(B, 1, 5, 1080, 1920): the BlobHessian response of the first five levels of a ScalePyramid octave of a smoothed
    noise image, as ScaleSpaceDetector builds it."""
    img = K.filters.gaussian_blur2d(torch.rand(B, 1, 1080, 1920, device="cuda", generator=g), (9, 9), (2.0, 2.0))
    pyr, sigmas, _ = K.geometry.ScalePyramid(3, 1.6, 15)(img)
    octave, sig = pyr[0][:, :, :5], sigmas[0][:, :5]
    L = octave.shape[2]
    resp = K.feature.hessian_response(octave.permute(0, 2, 1, 3, 4).reshape(B * L, 1, 1080, 1920), sigmas=sig.reshape(-1))
    return resp.view(B, L, 1, 1080, 1920).permute(0, 2, 1, 3, 4)


def same(a, b):
    return all(bool(((p.view(torch.int32) == q.view(torch.int32)) | (p.isnan() & q.isnan())).all()) for p, q in zip(a, b))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_subpix needs a GPU")
    info = card()
    print(json.dumps({"card": info}))
    rows = []
    g = torch.Generator(device="cuda").manual_seed(0)
    with torch.no_grad():
        for B in (1, 16):
            x = blob_octave(B, g)
            mask, _ = K.geometry.nms3d_minmax(x)
            workloads = {
                "conv_quad_interp3d with the nms3d_minmax mask": (lambda: Q.conv_quad_interp3d(x, 5, 0.0, 0.6, mask),
                                                                  lambda: Q._composed_conv_quad_interp3d(x, 5, 0.0, 0.6, mask, 1, True)),
                "conv_quad_interp3d": (lambda: Q.conv_quad_interp3d(x), lambda: Q._composed_conv_quad_interp3d(x, 5, 10.0, 0.6, None, 1, True)),
                "iterative_quad_interp3d": (lambda: Q.iterative_quad_interp3d(x),
                                            lambda: Q._composed_iterative_quad_interp3d(x, 5, 10.0, 0.6, True, None, None)),
            }
            for name, (fused, composed) in workloads.items():
                identical = same(fused(), composed())
                arms = {"fused": fused, "composed": composed}
                for fn in arms.values():
                    fn()
                    fn()
                times = {k: [] for k in arms}
                order = list(arms)
                for r in range(args.reps):
                    for k in order[r % 2:] + order[: r % 2]:
                        times[k].append(timed(arms[k]))
                med = {k: statistics.median(v) for k, v in times.items()}
                floor_ms = x.numel() * FLOOR_BYTES_PER_ELEMENT / HBM_BYTES_PER_S * 1e3
                row = {"workload": f"{name} {tuple(x.shape)}", "maxima": int(mask.sum()), "bit_identical_to_composition": identical,
                       **{f"{k}_ms": round(v, 4) for k, v in med.items()}, "floor_21B_ms": round(floor_ms, 4),
                       "fused_share_of_floor": round(floor_ms / med["fused"], 3), "speedup_vs_composed": round(med["composed"] / med["fused"], 1)}
                rows.append(row)
                print(json.dumps(row))
            del x, mask
            torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for row in [{"card": info}] + rows:
                f.write(json.dumps(row) + "\n")
    if not all(r["bit_identical_to_composition"] for r in rows):
        raise SystemExit("a fused result differs from the composition")


if __name__ == "__main__":
    main()
