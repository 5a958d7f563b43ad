"""remap: one CTA per tile (remap_tiled_kernel) against the pipelined persistent kernel (remap_piped_kernel, switch remap_piped),
interleaved, B=64x3x1080x1920, radial undistortion map (shared and per sample) and a per-sample flow field; bit comparison first."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import kornia_b200 as K

dev = "cuda"
B = int(sys.argv[1]) if len(sys.argv) > 1 else 64
x = torch.rand(B, 3, 1080, 1920, device=dev)
ys, xs = torch.meshgrid(torch.arange(1080, dtype=torch.float32, device=dev), torch.arange(1920, dtype=torch.float32, device=dev), indexing="ij")
r2 = ((xs - 960) / 960) ** 2 + ((ys - 540) / 540) ** 2
mx = (960 + (xs - 960) * (1 + 0.02 * r2))[None].contiguous()
my = (540 + (ys - 540) * (1 + 0.02 * r2))[None].contiguous()
mxb, myb = mx.expand(B, -1, -1).contiguous(), my.expand(B, -1, -1).contiguous()
amp = torch.linspace(0.5, 4.0, B, device=dev)[:, None, None]
fx = (xs[None] + amp * torch.sin(ys / 40.0)[None]).contiguous()
fy = (ys[None] + amp * torch.cos(xs / 55.0)[None]).contiguous()


def t(fn, n=10):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(n):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / n


cases = (("shared radial map", mx, my, 24.0), ("per-sample radial maps", mxb, myb, 32.0), ("per-sample flow field", fx, fy, 32.0))
for pad in ("zeros", "border", "reflection"):
    for name, ax, ay, bpp in cases:
        f = lambda: K.remap(x, ax, ay, padding_mode=pad, align_corners=True)
        with K.config.override(remap_piped=0):
            want = f()
        with K.config.override(remap_piped=2):
            got = f()
        same = torch.equal(got, want)
        del got, want
        rows = []
        for rep in range(2):
            for piped in (0, 1):
                with K.config.override(remap_piped=2 * piped):
                    rows.append((piped, t(f)))
        a = min(ms for p, ms in rows if p == 0)
        b = min(ms for p, ms in rows if p == 1)
        gb = bpp * B * 1080 * 1920 / 1e6
        print(f"{pad:10s} {name:24s} bit-identical={same}  per-tile {a:.3f} ms ({gb/a/3350*100:4.1f} %)  piped {b:.3f} ms ({gb/b/3350*100:4.1f} %)  x{a/b:.2f}   all: "
              + " ".join(f"{p}:{ms:.3f}" for p, ms in rows), flush=True)
