"""Non-maximum suppression on the H100: the fused kernels (csrc/nms.cuh) against the library composition (``_composed_*``
of kornia_b200/geometry/subpix/nms.py) and the reference's op sequence restated here (one ATen kernel per comparison and
per ``&``; the one-hot ``F.conv2d`` of the replicate-padded image for 15 x 15, cuDNN with torch's default settings).

    python tools/bench_nms.py [--reps 7] [--out results/bench_nms.jsonl]

Workloads, fp32, no gradient: nms3d_minmax on (1, 1, 5, 1080, 1920) and (16, 1, 5, 1080, 1920) (ScaleSpaceDetector's
octave 0), nms2d (5, 5) mask_only on (16, 1, 1080, 1920) (DISK, XFeat), NonMaximaSuppression2d((15, 15)) values on
(4, 1, 1080, 1920) (KeyNet's MultiResolutionDetector).  Per-call CUDA events after a warm-up, the arms alternated call by
call (order rotated from repeat to repeat), the median reported.  The fused result is compared bit for bit with the
library composition in the same run.  HBM floor: ``out.copy_(x)`` of the input (8 B per element); the fused kernel must
move 4 B read plus 1 B (mask) or 4 B (values) written per element and output.  The card's name and power limit are
printed first."""
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

from kornia_b200.geometry.subpix import nms as N  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


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


# ---- the reference's op sequence (kornia/geometry/subpix/nms.py), restated: one kernel per slice comparison and per `&`
def _ref_explicit(x, r, greater=True):
    def sl(d):
        return slice(d, d - 2 * r if d < 2 * r else None)

    if x.dim() == 4:
        ct = x[..., sl(r), sl(r)]
        offs = [(a, b) for a in range(2 * r + 1) for b in range(2 * r + 1) if (a, b) != (r, r)]
    else:
        ct = x[..., sl(1), sl(1), sl(1)]
        offs = [(a, b, c) for a in range(3) for b in range(3) for c in range(3) if (a, b, c) != (1, 1, 1)]
    m = None
    for o in offs:
        nb = x[(...,) + tuple(sl(d) for d in o)]
        c = ct > nb if greater else ct < nb
        m = c if m is None else m & c
    return m


def ref_nms3d_minmax(x):
    B, C, D, H, W = x.shape
    mx = torch.zeros(B, C, D, H, W, device=x.device, dtype=torch.bool)
    mn = torch.zeros(B, C, D, H, W, device=x.device, dtype=torch.bool)
    is_max, is_min = _ref_explicit(x, 1, True), _ref_explicit(x, 1, False)
    mx[..., 1:-1, 1:-1, 1:-1] = is_max
    mn[..., 1:-1, 1:-1, 1:-1] = is_min
    return mx, mn


def ref_nms2d_explicit(x, k, mask_only):
    B, C, H, W = x.shape
    r = k // 2
    mask = torch.zeros(B, C, H, W, device=x.device, dtype=torch.bool)
    mask[..., r:-r, r:-r] = _ref_explicit(x, r)
    return mask if mask_only else x * mask.to(x.dtype)


def ref_nms2d_general(x, k, kernel, mask_only):
    B, C, H, W = x.shape
    p = (k - 1) // 2
    xp = F.pad(x, [p, p, p, p], mode="replicate")
    nb = F.conv2d(xp.view(B * C, 1, H + 2 * p, W + 2 * p), kernel, stride=1).view(B, C, -1, H, W)
    mask = x > nb.max(dim=2)[0]
    return mask if mask_only else x * mask.to(x.dtype)


def workloads():
    m15 = N.NonMaximaSuppression2d((15, 15)).cuda()
    m5 = N.NonMaximaSuppression2d((5, 5)).cuda()
    for shape in ((1, 1, 5, 1080, 1920), (16, 1, 5, 1080, 1920)):
        yield (f"nms3d_minmax {shape}", shape, 2 * 1,
               lambda x: N.nms3d_minmax(x), lambda x: N._composed_nms3d_minmax(x), ref_nms3d_minmax)
    yield ("nms2d (5, 5) mask_only (16, 1, 1080, 1920)", (16, 1, 1080, 1920), 1,
           lambda x: N.nms2d(x, (5, 5), True), lambda x: N._composed_nms2d(x, (5, 5), m5.padding, m5.kernel, True),
           lambda x: ref_nms2d_explicit(x, 5, True))
    yield ("NonMaximaSuppression2d((15, 15)) values (4, 1, 1080, 1920)", (4, 1, 1080, 1920), 4,
           lambda x: m15(x), lambda x: N._composed_nms2d(x, (15, 15), m15.padding, m15.kernel, False),
           lambda x: ref_nms2d_general(x, 15, m15.kernel, False))


def same(a, b):
    if isinstance(a, tuple):
        return all(same(p, q) for p, q in zip(a, b))
    if a.dtype == torch.bool:
        return torch.equal(a, b)
    return bool(((a.view(torch.int32) == b.view(torch.int32)) | (a.isnan() & b.isnan())).all())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_nms needs a GPU")
    info = card()
    print(json.dumps({"card": info}))
    rows = []
    g = torch.Generator(device="cuda").manual_seed(0)
    with torch.no_grad():
        for name, shape, out_bytes, fused, composed, ref in workloads():
            x = torch.rand(shape, device="cuda", generator=g)
            floor_out = torch.empty_like(x)
            identical = same(fused(x), composed(x))
            arms = {"fused": lambda: fused(x), "composed": lambda: composed(x), "reference": lambda: ref(x), "copy_floor": lambda: floor_out.copy_(x)}
            for fn in arms.values():  # warm-up (and cuDNN's algorithm choice)
                fn()
                fn()
            times = {k: [] for k in arms}
            order = list(arms)
            for r in range(args.reps):
                for k in order[r % len(order):] + order[: r % len(order)]:
                    times[k].append(timed(arms[k]))
            med = {k: statistics.median(v) for k, v in times.items()}
            need = x.numel() * (4 + out_bytes)
            row = {"workload": name, "bit_identical_to_composition": identical, **{f"{k}_ms": round(v, 4) for k, v in med.items()},
                   "fused_GBps": round(need / med["fused"] / 1e6, 1), "fused_share_of_hbm_bound": round(need / HBM_BYTES_PER_S * 1e3 / med["fused"], 3),
                   "speedup_vs_composed": round(med["composed"] / med["fused"], 1), "speedup_vs_reference": round(med["reference"] / med["fused"], 1)}
            rows.append(row)
            print(json.dumps(row))
            del x, floor_out
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
