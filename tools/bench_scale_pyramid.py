"""ScalePyramid on the H100: the octave kernel (csrc/octave_vwalk.cuh) against the library composition
(``ScalePyramid._composed_pyramid``: this library's filter2d_separable per level + torch.stack) and the reference
composition (tests/scale_pyramid_restated.py: F.pad + grouped F.conv2d per pass, cuDNN on) on the same GPU.

    python tools/bench_scale_pyramid.py [--reps 7] [--out results/bench_scale_pyramid.jsonl]

Workloads: ScalePyramid() on 16x1x1080x1920, ScalePyramid(3, 1.6, 16, extra_levels=2) (ScaleSpaceDetector's) on
8x3x720x1280, ScalePyramid(3, 1.6, 32, double_image=True) (SIFTFeature's) on 4x1x1080x1920, fp32, no gradient.  Per-call
CUDA events after a warm-up, the arms alternated call by call (order rotated from repeat to repeat), the median reported;
the fused pyramid is compared bit for bit with the library composition at every size timed.  HBM floor: ``out.copy_(x)``
of the input (8 B per element).  Octave 0's kernel alone is timed too, with the bytes it must move (4 B read, 4 B written
per level) and the FMAs it issues over the data-sheet rates.  The card's name and power limit are printed first."""
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

import scale_pyramid_restated as SR  # noqa: E402
from kornia_b200._ops import ops  # noqa: E402
from kornia_b200.geometry.transform import ScalePyramid  # noqa: E402

FP32_FMA_PER_S = 67e12 / 2  # H100 SXM data sheet, dense fp32
HBM_BYTES_PER_S = 3.35e12
BAND = 128  # stored columns per CTA of the octave kernel (OCT_BW)

WORKLOADS = [
    ("default", {}, (16, 1, 1080, 1920)),
    ("detector", {"n_levels": 3, "init_sigma": 1.6, "min_size": 16, "extra_levels": 2}, (8, 3, 720, 1280)),
    ("double_image", {"n_levels": 3, "init_sigma": 1.6, "min_size": 32, "double_image": True}, (4, 1, 1080, 1920)),
]


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


def octave0_counts(ks):
    """(bytes, FMAs) per input element of octave 0: the kernel reads the seed once and writes L levels; every stage row-
    and column-filters its level on the band plus the support of the stages after it (E columns on each side)."""
    r = [(k - 1) // 2 for k in ks]
    L = len(ks)
    fma = 0.0
    for l in range(L):
        if ks[l] == 0:
            continue
        E = sum(r[l + 1:])
        fma += 2 * ks[l] * (BAND + 2 * E) / BAND
    return 4 + 4 * L, fma


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_scale_pyramid needs a GPU"
    print(json.dumps({"card": card()}), flush=True)
    torch.backends.cudnn.enabled = True
    rows = []
    gen = torch.Generator(device="cuda").manual_seed(0)
    for name, kw, shape in WORKLOADS:
        sp = ScalePyramid(**kw).cuda()
        x = torch.rand(*shape, device="cuda", generator=gen)
        floor = torch.empty_like(x)
        L = sp.n_levels + sp.extra_levels
        blur = sp._gk_init is not None
        names = (["_gk_init"] if blur else []) + [f"_gk_{i}" for i in range(L - 1)]
        taps = [v for n in names for v in sp._host_taps[n]]
        ks = ([len(sp._host_taps["_gk_init"])] if blur else [0]) + [len(sp._host_taps[f"_gk_{i}"]) for i in range(L - 1)]
        seed0 = sp._seed(x)[0]
        with torch.no_grad():
            a, b = sp(x), sp._composed_pyramid(x)
            same = all(bool(((p.view(torch.int32) == q.view(torch.int32)) | (p.isnan() & q.isnan())).all()) for p, q in zip(a[0], b[0]))
            octaves = len(a[0])
            del a, b
            ref = lambda t: SR.scale_pyramid(t, **kw)  # noqa: E731
            ref(x)
            arms = {"fused": lambda t: sp(t), "library_composition": lambda t: sp._composed_pyramid(t), "reference_composition": ref,
                    "octave0_kernel": lambda t: ops.scale_octave_fwd(seed0, taps, ks), "copy_floor": lambda t: floor.copy_(t)}
            times = {k: [] for k in arms}
            order = list(arms)
            for r in range(args.reps):
                for k in order[r % len(order):] + order[:r % len(order)]:
                    times[k].append(timed(lambda: arms[k](x)))
        med = {k: statistics.median(v) for k, v in times.items()}
        n0 = seed0.numel()
        bpe, fpe = octave0_counts(ks)
        hbm = n0 * bpe / HBM_BYTES_PER_S * 1e3
        fma = n0 * fpe / FP32_FMA_PER_S * 1e3
        row = {"workload": name, "module": repr(sp), "shape": list(shape), "octaves": octaves, "bit_identical": same,
               "ms": {k: round(v, 4) for k, v in med.items()}, "ms_all": {k: [round(t, 4) for t in v] for k, v in times.items()},
               "speedup_vs_library": round(med["library_composition"] / med["fused"], 2),
               "speedup_vs_reference": round(med["reference_composition"] / med["fused"], 2),
               "octave0": {"bytes_per_element": bpe, "fma_per_element": round(fpe, 1), "datasheet_bounds_ms": {"hbm": round(hbm, 4), "fp32_fma": round(fma, 4)},
                           "bound_by": "fp32_fma" if fma > hbm else "hbm", "kernel_over_bound": round(med["octave0_kernel"] / max(hbm, fma), 2)}}
        print(json.dumps(row), flush=True)
        rows.append(row)
        del x, floor, seed0
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for row in rows:
                f.write(json.dumps(row) + "\n")


if __name__ == "__main__":
    main()
