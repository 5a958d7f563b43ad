"""Headline warp (B x 3 x 1080 x 1920, bilinear, zeros): kernel variants against each other and against the card's read+write
ceiling, interleaved in one process; bit comparison first.

    python tools/ab_headline.py [--batch B] [--reps R] [ARM ...]

An ARM is ``name=value[,name=value...]`` (device switches of kornia_b200.config, applied around the call), ``default`` (the
switches as loaded) or ``copy`` (``out.copy_(src)`` on tensors of the workload's size: the same 24 B per pixel a warp moves).
Every warp arm is checked with torch.equal against the first one.  Kernel time comes from CUDA events around each forward
launch (the same events bench.py's roofline.kernel_ms uses); each repeat of each arm is the mean of --steps launches, and the
arms take turns in an order that rotates from repeat to repeat."""
import argparse
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench
import kornia_b200 as K
from kornia_b200 import _ops

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=256)
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--steps", type=int, default=20)
ap.add_argument("arms", nargs="*", default=["default", "sweep=0", "dyn_sched=0", "copy"])
args = ap.parse_args()

try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                           str(torch.cuda.current_device())], capture_output=True, text=True, timeout=60).stdout.strip()
except (OSError, subprocess.SubprocessError) as e:
    card = f"{torch.cuda.get_device_name()} (nvidia-smi unavailable: {e})"
print("card (name, power limit, max SM clock):", card, flush=True)

B = args.batch
torch.manual_seed(1000)
x = torch.rand(B, 3, 1080, 1920, device="cuda")
M = bench.make_homographies(B, 1000).cuda()


def parse(arm):
    if arm in ("default", "copy"):
        return {}
    return {k: int(v) for k, v in (kv.split("=") for kv in arm.split(","))}


def call(arm):
    if arm == "copy":
        return lambda: copy_out.copy_(x)
    return lambda: K.warp_perspective(x, M, (1080, 1920))


copy_out = torch.empty_like(x)
warp_arms = [a for a in args.arms if a != "copy"]
want = None
for arm in warp_arms:
    with K.config.override(**parse(arm)):
        got = call(arm)()
    if want is None:
        want = got
        print(f"reference for the bit comparison: {arm}", flush=True)
    else:
        print(f"{arm}: bit-identical to {warp_arms[0]}: {torch.equal(got, want)}", flush=True)
    del got
del want
torch.cuda.empty_cache()


def timed(arm):
    f = call(arm)
    for _ in range(3):
        f()
    torch.cuda.synchronize()
    if arm == "copy":
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(args.steps):
            f()
        e.record()
        torch.cuda.synchronize()
        return s.elapsed_time(e) / args.steps
    _ops.kernel_events = []
    for _ in range(args.steps):
        f()
    torch.cuda.synchronize()
    ev, _ops.kernel_events = _ops.kernel_events, None
    return statistics.mean(s.elapsed_time(e) for (_, s, e) in ev)


res = {a: [] for a in args.arms}
for rep in range(args.reps):
    # Each repeat starts one arm further on, so that no arm always runs right after the same neighbour: on an H100 held to
    # 400 W the arm that followed the copy ran up to 30 % slower than in its other repeats.
    order = args.arms[rep % len(args.arms):] + args.arms[:rep % len(args.arms)]
    for arm in order:
        with K.config.override(**parse(arm)):
            res[arm].append(timed(arm))
    print(f"repeat {rep}: " + ", ".join(f"{arm} {res[arm][-1]:.3f}" for arm in order), flush=True)
gb = 24.0 * B * 1080 * 1920 / 1e6  # bytes the launch must move (read 12 + write 12 per pixel), in MB -> MB / ms = GB / s
print(f"B={B}, {args.reps} interleaved repeats of {args.steps} launches; min / median / max kernel ms, GB/s at the min:", flush=True)
for arm in args.arms:
    r = sorted(res[arm])
    print(f"  {arm:32s} {r[0]:.4f} / {statistics.median(r):.4f} / {r[-1]:.4f} ms  spread {r[-1] - r[0]:.4f}  "
          f"{gb / r[0]:.0f} GB/s ({gb / r[0] / 3350 * 100:.1f} % of 3.35 TB/s)", flush=True)
