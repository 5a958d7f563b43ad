"""Headline warp (B x 3 x 1080 x 1920, bilinear, zeros): strips dealt out in advance against handed out at run time (switch dyn_sched),
interleaved in one process; bit comparison first.  python tools/ab_headline.py [B]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench
import kornia_b200 as K

B = int(sys.argv[1]) if len(sys.argv) > 1 else 256
x = torch.rand(B, 3, 1080, 1920, device="cuda")
M = bench.make_homographies(B, 1000).cuda()
f = lambda: K.warp_perspective(x, M, (1080, 1920))  # noqa: E731
with K.config.override(dyn_sched=0):
    want = f()
with K.config.override(dyn_sched=1):
    got = f()
print("bit-identical:", torch.equal(got, want), flush=True)
del got, want


def t(n=20):
    for _ in range(3):
        f()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(n):
        f()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / n


res = {0: [], 1: []}
for rep in range(4):
    for v in (0, 1):
        with K.config.override(dyn_sched=v):
            res[v].append(t())
gb = 24.0 * B * 1080 * 1920 / 1e6
for v in (0, 1):
    a = min(res[v])
    print(f"dyn_sched={v}: {a:.4f} ms / call ({gb / a / 3350 * 100:.1f} % of 3.35 TB/s)  all: {['%.4f' % r for r in res[v]]}", flush=True)
