"""Motion-blur filter2d on the H100: the zero-skipping kernel (csrc/filter2d_taps.cuh, odd K 9..31) against the generic
kernel (``tiled_filter=0``) and the reference composition (F.pad + grouped F.conv2d, tests/motion_restated.py) on the same GPU.

    python tools/bench_motion.py [--batches 64 256] [--reps 5] [--out results/bench_motion.jsonl]

Workload: B x 3 x 1080 x 1920 fp32, K in {7, 9, 15, 31}, nearest and bilinear motion kernels with per-sample angles and
directions, and a dense box kernel at K = 9 and 15 (dense filter2d users).  K = 7 runs on the existing K <= 7 tiled kernel
and is there for comparison.  Per-launch CUDA events after a warm-up, the arms alternated launch by launch, the median
reported; the outputs of the two CUDA arms are compared bit for bit at every size timed.  HBM floor: the time of
``out.copy_(x)`` on the same tensors (24 B per RGB pixel: 12 read, 12 written), measured in the same call.  The card's name
and power limit are printed first."""
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
from kornia_b200 import config  # noqa: E402


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


def kernels(kind: str, B: int, ksize: int, gen) -> torch.Tensor:
    if kind == "box":
        return torch.full((1, ksize, ksize), 1.0 / (ksize * ksize), device="cuda")
    angle = (torch.rand(B, generator=gen) * 360.0 - 180.0).cuda()
    direction = (torch.rand(B, generator=gen) * 2.0 - 1.0).cuda()
    return K.filters.get_motion_kernel2d(ksize, angle, direction, kind)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[64, 256])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ref-batch", type=int, default=32)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_motion needs a GPU"
    info = card()
    print(json.dumps({"card": info}), flush=True)
    rows = []
    H, W = 1080, 1920
    cases = [(k, kind) for k in (7, 9, 15, 31) for kind in ("nearest", "bilinear")] + [(9, "box"), (15, "box")]
    gen = torch.Generator().manual_seed(0)
    for B in args.batches:
        x = torch.rand(B, 3, H, W, device="cuda")
        out = torch.empty_like(x)
        floor = [timed(lambda: out.copy_(x)) for _ in range(3)]
        floor_ms = statistics.median(floor)
        del out
        for ksize, kind in cases:
            k = kernels(kind, B, ksize, gen)
            taps = int((k != 0).sum()) / k.shape[0]
            new = K.filters.filter2d(x, k, "reflect")  # warm-up and the output compared below
            with config.override(tiled_filter=0):
                gen_out = K.filters.filter2d(x, k, "reflect")
            identical = bool(torch.equal(new.view(torch.int32), gen_out.view(torch.int32)))
            del new, gen_out
            t_new, t_gen = [], []
            for _ in range(args.reps):  # alternated
                t_new.append(timed(lambda: K.filters.filter2d(x, k, "reflect")))
                with config.override(tiled_filter=0):
                    t_gen.append(timed(lambda: K.filters.filter2d(x, k, "reflect")))
            mn, mg = statistics.median(t_new), statistics.median(t_gen)
            row = {"B": B, "K": ksize, "kernel": kind, "nonzero_taps": round(taps, 1), "default_ms": round(mn, 3), "generic_ms": round(mg, 3),
                   "speedup": round(mg / mn, 2), "default_gpix_s": round(B * H * W / mn / 1e6, 2), "generic_gpix_s": round(B * H * W / mg / 1e6, 2),
                   "hbm_floor_ms": round(floor_ms, 3), "default_frac_of_floor": round(floor_ms / mn, 3), "bit_identical": identical,
                   "default_spread_ms": [round(min(t_new), 3), round(max(t_new), 3)], "generic_spread_ms": [round(min(t_gen), 3), round(max(t_gen), 3)]}
            rows.append(row)
            print(json.dumps(row), flush=True)
        del x
        torch.cuda.empty_cache()

    # the reference composition (kernel build + F.pad + grouped conv2d) against ours end to end, on a smaller batch
    import motion_restated as MR

    B = args.ref_batch
    x = torch.rand(B, 3, H, W, device="cuda")
    angle = (torch.rand(B, generator=gen) * 360.0 - 180.0).cuda()
    direction = (torch.rand(B, generator=gen) * 2.0 - 1.0).cuda()
    for ksize in (9, 15, 31):
        for mode in ("nearest", "bilinear"):
            ours = lambda: K.filters.motion_blur(x, ksize, angle, direction, "reflect", mode)  # noqa: E731
            ref = lambda: MR.motion_blur(x, ksize, angle, direction, "reflect", mode)  # noqa: E731
            a, b = ours(), ref()
            err = float((a - b).abs().max())
            del a, b
            t_o, t_r = [], []
            for _ in range(args.reps):
                t_o.append(timed(ours))
                t_r.append(timed(ref))
            mo, mr = statistics.median(t_o), statistics.median(t_r)
            row = {"B": B, "K": ksize, "mode": mode, "motion_blur_ms": round(mo, 3), "reference_ms": round(mr, 3), "speedup": round(mr / mo, 2),
                   "max_abs_diff": err}
            rows.append(row)
            print(json.dumps(row), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(json.dumps({"card": info}) + "\n")
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
