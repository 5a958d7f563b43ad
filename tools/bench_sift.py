"""SIFTDescriptor and PatchDominantGradientOrientation on the H100: the fused kernels (csrc/siftdesc.cuh,
csrc/patch_orientation.cuh) against the library composition (``_composed_sift`` / ``_composed_orientation``) and the
reference's own GPU op sequence (its forward restated over ATen: ``F.pad`` + ``F.conv2d`` gradients, the per-bin
one-hot products, ``nn.Conv2d`` / ``adaptive_avg_pool2d`` pooling and the circular ``nn.Conv1d``, on cuDNN defaults).

    python tools/bench_sift.py [--reps 7] [--out results/bench_sift.jsonl]

Workloads, fp32 under torch.inference_mode(), on uniform random patches: SIFTDescriptor(41) at N = 8000 and 65536,
SIFTDescriptor(32) at 65536, PatchDominantGradientOrientation(19) and (32) at 8000 and 65536.  Per-call CUDA events after a
warm-up, the three arms alternated call by call, the median reported.  Each row states whether the fused output is within
1e-5 of the composition (SIFT: every element, NaN positions equal; orientation: every angle whose top-two smoothed bins
are more than 1e-5 apart, relative).  The card's name and power limit are printed first."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from kornia_b200 import feature as KF  # noqa: E402
from kornia_b200.feature import orientation as OR, siftdesc as SD  # noqa: E402

PI = torch.tensor(3.14159265358979323846)
DIFF = [[[0.0, 0.0, 0.0], [-0.5, 0.0, 0.5], [0.0, 0.0, 0.0]], [[0.0, -0.5, 0.0], [0.0, 0.0, 0.0], [0.0, 0.5, 0.0]]]
SOBEL = [[[-0.125, 0.0, 0.125], [-0.25, 0.0, 0.25], [-0.125, 0.0, 0.125]], [[-0.125, -0.25, -0.125], [0.0, 0.0, 0.0], [0.125, 0.25, 0.125]]]


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


def _grad(x, stencil):
    w = torch.tensor(stencil, device=x.device, dtype=x.dtype).unsqueeze(1)  # (2, 1, 3, 3)
    return F.conv2d(F.pad(x, [1, 1, 1, 1], "replicate"), w).unsqueeze(1)  # (B, 1, 2, P, P)


def _bins(mag, o_big, n, dtype):
    b0_ = torch.floor(o_big)
    w1_ = o_big - b0_
    b0 = b0_ % n
    b1 = (b0 + 1) % n
    return [(b0 == i).to(dtype) * ((1.0 - w1_) * mag) + (b1 == i).to(dtype) * (w1_ * mag) for i in range(n)]


def reference_sift(m, x):
    g = _grad(x, DIFF)
    gx, gy = g[:, :, 0], g[:, :, 1]
    mag = torch.sqrt(gx * gx + gy * gy + m.eps)
    ori = torch.atan2(gy, gx + m.eps) + 2.0 * PI
    mag = mag * m.gk.expand_as(mag).type_as(mag).to(mag.device)
    o_big = float(m.num_ang_bins) * ori / (2.0 * PI)
    out = torch.cat([m.pk(p) for p in _bins(mag, o_big, m.num_ang_bins, x.dtype)], 1).view(x.shape[0], -1)
    out = F.normalize(torch.clamp(F.normalize(out, p=2), 0.0, float(m.clipval)), p=2)
    return torch.sqrt(F.normalize(out, p=1) + m.eps) if m.rootsift else out


def reference_orientation(m, x):
    n = m.num_ang_bins
    g = _grad(x, SOBEL)
    gx, gy = g[:, :, 0], g[:, :, 1]
    mag = torch.sqrt(gx * gx + gy * gy + m.eps) * m.weighting
    ori = torch.atan2(gy, gx + m.eps) + 2.0 * PI
    o_big = float(n) * (ori + 1.0 * PI) / (2.0 * PI)
    hist = torch.cat([F.adaptive_avg_pool2d(p, (1, 1)) for p in _bins(mag, o_big, n, x.dtype)], 1).view(-1, 1, n)
    hist = m.angular_smooth(hist).view(-1, n)
    values, idx = hist.max(1)
    left = torch.gather(hist, 1, ((n + idx - 1) % n).reshape(-1, 1)).reshape(-1)
    right = torch.gather(hist, 1, ((idx + 1) % n).reshape(-1, 1)).reshape(-1)
    c = 0.5 * (left - right) / (left + right - 2.0 * values)
    return -((2.0 * PI * (idx.to(x.dtype) + c) / float(n)) - PI), hist


def agree(kind, fused, composed, hist):
    if kind == "sift":
        if not torch.equal(fused.isnan(), composed.isnan()):
            return False
        ok = ~composed.isnan()
        return bool((fused[ok] - composed[ok]).abs().max() <= 1e-5)
    top = hist.topk(2, 1).values
    clear = (top[:, 0] - top[:, 1]).abs() > 1e-5 * top[:, 0].abs()
    d = (fused - composed).abs()
    d = torch.minimum(d, 2 * torch.pi - d)
    print(json.dumps({"orientation_angles_within_1e-5_of_the_composition": f"{int((d[clear] <= 1e-5).sum())} of {int(clear.sum())} "
                      f"clear cases ({int((~clear).sum())} below the margin)"}))
    return bool(d[clear].max() <= 1e-5) and torch.equal(fused.isnan(), composed.isnan())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    print(json.dumps({"card": card()}))
    workloads = [("sift", 41, 8000), ("sift", 41, 65536), ("sift", 32, 65536), ("orientation", 19, 8000), ("orientation", 19, 65536),
                 ("orientation", 32, 8000), ("orientation", 32, 65536)]
    rows = []
    for kind, P, N in workloads:
        m = (KF.SIFTDescriptor(P) if kind == "sift" else KF.PatchDominantGradientOrientation(P)).cuda()
        x = torch.rand(N, 1, P, P, device="cuda", generator=torch.Generator(device="cuda").manual_seed(N + P))
        comp = SD._composed_sift if kind == "sift" else OR._composed_orientation
        ref = reference_sift if kind == "sift" else (lambda mm, xx: reference_orientation(mm, xx)[0])
        with torch.inference_mode():
            fused_out = m(x)
            comp_out = comp(m, x)
            hist = None if kind == "sift" else reference_orientation(m, x)[1]
            arms = {"fused": lambda: m(x), "composition": lambda: comp(m, x), "reference": lambda: ref(m, x)}
            for fn in arms.values():
                fn()
            times = {k: [] for k in arms}
            for r in range(args.reps):
                order = list(arms)[r % 3:] + list(arms)[: r % 3]
                for k in order:
                    times[k].append(timed(arms[k]))
        med = {k: statistics.median(v) for k, v in times.items()}
        row = {"workload": f"{'SIFTDescriptor' if kind == 'sift' else 'PatchDominantGradientOrientation'}({P})", "N": N,
               "fused_ms": round(med["fused"], 4), "composition_ms": round(med["composition"], 4), "reference_ms": round(med["reference"], 4),
               "speedup_vs_reference": round(med["reference"] / med["fused"], 1), "speedup_vs_composition": round(med["composition"] / med["fused"], 1),
               "matches_composition": agree(kind, fused_out, comp_out, hist)}
        rows.append(row)
        print(json.dumps(row), flush=True)
        del m, x, fused_out, comp_out
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "a") as f:
            for row in rows:
                f.write(json.dumps(row) + "\n")


if __name__ == "__main__":
    main()
