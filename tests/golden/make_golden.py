"""Generate the golden vectors under tests/golden/ by running the UNMODIFIED reference.

Run in the build container only (needs /root/reference):

    python tests/golden/make_golden.py

The reference (kornia 0.9.0rc1 @ b4f5a78a) is imported from /root/reference with an empty stub
module standing in for the un-vendored Rust wheel ``kornia_rs`` (image IO; the warp / filter path
never calls it: SURVEY.md section 8c).  Every case stores the exact inputs, the keyword arguments
(JSON) and the reference's CPU fp32 outputs (plus autograd gradients where marked), so the
fixtures travel to the GPU box where /root/reference does not exist.

Output: tests/golden/warp.*.npz, tests/golden/filter.*.npz (shards under 1 MB; inputs are stored once per shard,
content-addressed).
"""
from __future__ import annotations

import glob
import hashlib
import json
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))


def import_reference():
    stub = tempfile.mkdtemp(prefix="kornia_rs_stub_")
    with open(os.path.join(stub, "kornia_rs.py"), "w") as f:
        f.write("# empty stand-in for the kornia_rs wheel (image codecs; unused on the hot path)\n")
    sys.path.insert(0, "/root/reference")
    sys.path.insert(0, stub)
    import kornia  # noqa: F401

    return kornia


def t2n(t):
    return t.detach().cpu().numpy()


class Bag:
    def __init__(self):
        self.arrays = {}
        self.meta = {}

    def _put(self, t):
        # content-addressed so the shared inputs are stored once
        a = np.ascontiguousarray(t2n(t))
        key = "a" + hashlib.sha1(a.tobytes() + str(a.shape).encode() + str(a.dtype).encode()).hexdigest()[:12]
        self.arrays[key] = a
        return key

    def add(self, name, op, inputs: dict, kwargs: dict, outputs: dict):
        assert name not in self.meta, name
        self.meta[name] = {
            "op": op,
            "kwargs": kwargs,
            "inputs": {k: self._put(v) for k, v in inputs.items()},
            "outputs": {k: self._put(v) for k, v in outputs.items()},
        }

    SHARD_BYTES = 800_000  # uncompressed array bytes per shard: every stored file stays under 1 MB

    def save(self, path):
        """``x.npz`` is written as shards ``x.0.npz``, ``x.1.npz``, ... of whole cases, each with the ``__meta__`` of its
        cases (an input shared by cases of two shards is stored in both); tests/conftest.py:Golden reads them back as one."""
        stem = path[: -len(".npz")]
        for old in glob.glob(glob.escape(stem) + ".*.npz"):  # a save with fewer shards must not leave stale cases behind
            os.remove(old)
        shards, keys, size = [], None, 0
        for name, m in self.meta.items():
            need = set(m["inputs"].values()) | set(m["outputs"].values())
            extra = sum(self.arrays[k].nbytes for k in need - (keys or set()))
            if keys is None or (size + extra > self.SHARD_BYTES and shards[-1]):
                shards.append({})
                keys, size = set(), 0
                extra = sum(self.arrays[k].nbytes for k in need)
            shards[-1][name] = m
            keys |= need
            size += extra
        for i, meta in enumerate(shards):
            arrays = {k: self.arrays[k] for m in meta.values() for k in list(m["inputs"].values()) + list(m["outputs"].values())}
            arrays["__meta__"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
            np.savez_compressed(f"{stem}.{i}.npz", **arrays)
        print(f"{stem}.*.npz: {len(self.meta)} cases in {len(shards)} shards of at most "
              f"{max(os.path.getsize(f'{stem}.{i}.npz') for i in range(len(shards))) / 1024:.0f} kB")


def smooth_image(B, C, H, W, gen):
    """Band-limited test image (SURVEY.md 8d): sum of 6 sinusoids <= 8 cycles/image in [0,1]."""
    yy = torch.linspace(0, 1, H)[:, None]
    xx = torch.linspace(0, 1, W)[None, :]
    img = torch.zeros(B, C, H, W)
    for _ in range(6):
        fx = torch.randint(0, 9, (B, C, 1, 1), generator=gen).float()
        fy = torch.randint(0, 9, (B, C, 1, 1), generator=gen).float()
        ph = torch.rand(B, C, 1, 1, generator=gen) * 6.2831853
        img = img + torch.sin(6.2831853 * (fx * xx + fy * yy) + ph)
    return img / 12 + 0.5


def jitter_homography(kornia, B, H, W, gen, sigma_px):
    """benchmarks/geometry/flagship.py:101-107 recipe: corners -> corners + sigma*randn."""
    quad = torch.tensor([[0.0, 0.0], [W - 1.0, 0.0], [W - 1.0, H - 1.0], [0.0, H - 1.0]]).expand(B, 4, 2)
    dst = quad + sigma_px * torch.randn(B, 4, 2, generator=gen)
    return kornia.geometry.transform.get_perspective_transform(quad, dst)


def main():
    kornia = import_reference()
    import kornia.filters as KF
    import kornia.geometry.transform as KT

    torch.manual_seed(0)
    torch.set_num_threads(1)
    gen = torch.Generator().manual_seed(1234)

    # ------------------------------------------------------------------ warps
    bag = Bag()
    B, C, H, W = 2, 3, 23, 31
    src = torch.rand(B, C, H, W, generator=gen)
    Hm = jitter_homography(kornia, B, H, W, gen, 3.0)
    # one strongly projective / partially out-of-view matrix
    Hm_wild = Hm.clone()
    Hm_wild[0] = torch.tensor([[0.9, 0.25, -6.0], [-0.2, 1.1, 4.0], [1.5e-3, -2.0e-3, 1.0]])
    fill3 = torch.tensor([0.25, 0.5, 0.75])
    for mode in ("bilinear", "nearest", "bicubic"):
        for pad in ("zeros", "border", "reflection", "fill"):
            for ac in (True, False):
                for tag, MM, dsize in (("jit", Hm, (19, 27)), ("wild", Hm_wild, (24, 36))):
                    kw = dict(dsize=list(dsize), mode=mode, padding_mode=pad, align_corners=ac)
                    ins = dict(src=src, M=MM)
                    if pad == "fill":
                        ins["fill_value"] = fill3
                    out = KT.warp_perspective(src, MM, dsize, mode=mode, padding_mode=pad, align_corners=ac,
                                              fill_value=fill3 if pad == "fill" else None)
                    bag.add(f"wp_{mode}_{pad}_{int(ac)}_{tag}", "warp_perspective", ins, kw, dict(out=out))

    # cfg1 of BASELINE.json: warp_affine B=4 3x64x64, 30 deg rotation about the centre
    torch.manual_seed(0)
    src64 = torch.rand(4, 3, 64, 64)
    A30 = KT.get_rotation_matrix2d(torch.tensor([[32.0, 32.0]]), torch.tensor([30.0]), torch.ones(1, 2)).repeat(4, 1, 1)
    bag.add("cfg1_warp_affine", "warp_affine", dict(src=src64, M=A30),
            dict(dsize=[64, 64], mode="bilinear", padding_mode="zeros", align_corners=True),
            dict(out=KT.warp_affine(src64, A30, (64, 64))))

    srcA = torch.rand(3, 5, 14, 17, generator=gen)
    A = torch.tensor([[[0.9, -0.3, 2.0], [0.25, 1.1, -1.5]]]).repeat(3, 1, 1) + 0.05 * torch.randn(3, 2, 3, generator=gen)
    fill5 = torch.rand(5, generator=gen)
    for mode in ("bilinear", "nearest", "bicubic"):
        for pad in ("zeros", "border", "reflection", "fill"):
            for ac in (True, False):
                for tag, MM in (("per", A), ("shared", A[:1])):
                    kw = dict(dsize=[12, 15], mode=mode, padding_mode=pad, align_corners=ac)
                    ins = dict(src=srcA, M=MM)
                    if pad == "fill":
                        ins["fill_value"] = fill5
                    out = KT.warp_affine(srcA, MM, (12, 15), mode=mode, padding_mode=pad, align_corners=ac,
                                         fill_value=fill5 if pad == "fill" else None)
                    bag.add(f"wa_{mode}_{pad}_{int(ac)}_{tag}", "warp_affine", ins, kw, dict(out=out))
    # fill with scalar-like fill values (imgwarp.py:311-314)
    for tag, fv in (("fill1", torch.tensor([0.3])), ("fill0d", torch.tensor(0.7))):
        out = KT.warp_affine(srcA, A, (12, 15), padding_mode="fill", fill_value=fv)
        bag.add(f"wa_{tag}", "warp_affine", dict(src=srcA, M=A, fill_value=fv),
                dict(dsize=[12, 15], mode="bilinear", padding_mode="fill", align_corners=True), dict(out=out))

    # remap
    img = torch.rand(2, 3, 13, 17, generator=gen)
    ys, xs = torch.meshgrid(torch.arange(11.0), torch.arange(14.0), indexing="ij")
    mx = (xs * 1.1 - 1.5)[None].repeat(2, 1, 1) + 0.7 * torch.randn(2, 11, 14, generator=gen)
    my = (ys * 1.3 - 2.0)[None].repeat(2, 1, 1) + 0.7 * torch.randn(2, 11, 14, generator=gen)
    for mode in ("bilinear", "nearest", "bicubic"):
        for pad in ("zeros", "border", "reflection"):
            for ac in (None, True, False):
                kw = dict(mode=mode, padding_mode=pad, align_corners=ac, normalized_coordinates=False)
                bag.add(f"rm_{mode}_{pad}_{ac}", "remap", dict(image=img, map_x=mx, map_y=my), kw,
                        dict(out=KT.remap(img, mx, my, **kw)))
    kw = dict(mode="bilinear", padding_mode="zeros", align_corners=True, normalized_coordinates=False)
    bag.add("rm_broadcast", "remap", dict(image=img, map_x=mx[:1], map_y=my[:1]), kw,
            dict(out=KT.remap(img, mx[:1], my[:1], **kw)))
    nx = torch.rand(2, 11, 14, generator=gen) * 2.4 - 1.2
    ny = torch.rand(2, 11, 14, generator=gen) * 2.4 - 1.2
    kw = dict(mode="bilinear", padding_mode="border", align_corners=None, normalized_coordinates=True)
    bag.add("rm_normalized", "remap", dict(image=img, map_x=nx, map_y=ny), kw, dict(out=KT.remap(img, nx, ny, **kw)))

    # gradients (reference autograd): d/dsrc and d/dM of sum(out * cot)
    def grads(fn, tensors, wrt):
        leaves = {k: (v.clone().requires_grad_(True) if k in wrt else v) for k, v in tensors.items()}
        out = fn(**leaves)
        cot = torch.rand(out.shape, generator=gen) - 0.5
        g = torch.autograd.grad((out * cot).sum(), [leaves[k] for k in wrt], allow_unused=True)
        outs = {"out": out, "cot": cot}
        for k, gi in zip(wrt, g):
            outs[f"grad_{k}"] = gi if gi is not None else torch.zeros_like(leaves[k])
        return outs

    smooth = smooth_image(2, 3, H, W, gen)
    for mode in ("bilinear", "nearest", "bicubic"):
        for pad in ("zeros", "border", "reflection", "fill"):
            for ac in (True, False):
                kw = dict(dsize=[19, 27], mode=mode, padding_mode=pad, align_corners=ac)
                fv = fill3 if pad == "fill" else None
                o = grads(lambda src, M: KT.warp_perspective(src, M, (19, 27), mode=mode, padding_mode=pad,
                                                             align_corners=ac, fill_value=fv),
                          dict(src=smooth, M=Hm), ("src", "M"))
                ins = dict(src=smooth, M=Hm, cot=o.pop("cot"))
                if fv is not None:
                    ins["fill_value"] = fv
                bag.add(f"g_wp_{mode}_{pad}_{int(ac)}", "warp_perspective_grad", ins, kw, o)
    for pad in ("zeros", "border", "reflection"):
        for tag, MM in (("per", A), ("shared", A[:1])):
            kw = dict(dsize=[12, 15], mode="bilinear", padding_mode=pad, align_corners=False)
            o = grads(lambda src, M: KT.warp_affine(src, M, (12, 15), padding_mode=pad, align_corners=False),
                      dict(src=srcA, M=MM), ("src", "M"))
            bag.add(f"g_wa_{pad}_{tag}", "warp_affine_grad", dict(src=srcA, M=MM, cot=o.pop("cot")), kw, o)
    for mode in ("bilinear", "bicubic"):
        for pad in ("zeros", "border", "reflection"):
            kw = dict(mode=mode, padding_mode=pad, align_corners=None, normalized_coordinates=False)
            o = grads(lambda image, map_x, map_y: KT.remap(image, map_x, map_y, **kw),
                      dict(image=img, map_x=mx, map_y=my), ("image", "map_x", "map_y"))
            bag.add(f"g_rm_{mode}_{pad}", "remap_grad", dict(image=img, map_x=mx, map_y=my, cot=o.pop("cot")), kw, o)
    bag.save(os.path.join(HERE, "warp.npz"))

    # ------------------------------------------------------------------ filters
    bag = Bag()
    x = torch.rand(4, 3, 13, 16, generator=gen)
    kernels = {
        "k3x3": torch.randn(1, 3, 3, generator=gen),
        "k5x4": torch.randn(1, 5, 4, generator=gen),      # even width: asymmetric padding
        "k2x2": torch.randn(1, 2, 2, generator=gen),
        "k7x1": torch.randn(1, 7, 1, generator=gen),
        "k1x9": torch.randn(1, 1, 9, generator=gen),
        "k3x5_B": torch.randn(4, 3, 5, generator=gen),    # per-sample kernels
        "k3x3_cyc": torch.randn(2, 3, 3, generator=gen),  # Bk=2 cycles over B=4 (filter.py:141-142)
    }
    for kn, k in kernels.items():
        for border in ("constant", "reflect", "replicate", "circular"):
            for normalized in (False, True):
                for padding in ("same", "valid"):
                    for behaviour in ("corr", "conv"):
                        if behaviour == "conv" and (normalized or padding == "valid" or border != "reflect"):
                            continue
                        kw = dict(border_type=border, normalized=normalized, padding=padding, behaviour=behaviour)
                        bag.add(f"f2d_{kn}_{border}_{int(normalized)}_{padding}_{behaviour}", "filter2d",
                                dict(input=x, kernel=k), kw, dict(out=KF.filter2d(x, k, **kw)))
    kx = torch.randn(1, 5, generator=gen)
    ky = torch.randn(1, 7, generator=gen)
    kxB = torch.randn(4, 3, generator=gen)
    kyB = torch.randn(4, 9, generator=gen)
    for tag, (a, b) in (("shared", (kx, ky)), ("batched", (kxB, kyB))):
        for border in ("constant", "reflect", "replicate", "circular"):
            for padding in ("same", "valid"):
                kw = dict(border_type=border, normalized=(tag == "batched"), padding=padding)
                bag.add(f"sep_{tag}_{border}_{padding}", "filter2d_separable", dict(input=x, kernel_x=a, kernel_y=b), kw,
                        dict(out=KF.filter2d_separable(x, a, b, **kw)))
    # gaussian taps (kernels.py:552) and blur
    for ks, sg in ((3, 2.5), (5, 1.5), (11, 2.0), (4, 0.8)):
        taps = KF.get_gaussian_kernel1d(ks, sg, force_even=True)
        bag.add(f"taps_{ks}_{sg}", "gaussian_taps", {}, dict(kernel_size=ks, sigma=sg), dict(out=taps))
    xb = torch.rand(2, 3, 21, 24, generator=gen)
    sig_t = torch.tensor([[1.5, 0.9], [2.0, 2.5]])
    for ks in (3, (5, 5), (5, 7), (11, 11)):
        for border in ("constant", "reflect", "replicate", "circular"):
            for separable in (True, False):
                for tag, sg in (("tuple", (2.0, 1.25)), ("tensor", sig_t)):
                    kw = dict(kernel_size=list(ks) if isinstance(ks, tuple) else ks, border_type=border, separable=separable)
                    ins = dict(input=xb)
                    if tag == "tensor":
                        ins["sigma"] = sg
                    else:
                        kw["sigma"] = list(sg)
                    name = f"gb_{ks if isinstance(ks, int) else 'x'.join(map(str, ks))}_{border}_{int(separable)}_{tag}"
                    bag.add(name, "gaussian_blur2d", ins, kw, dict(out=KF.gaussian_blur2d(xb, ks, sg, border, separable)))
    # sigma batch (2) != input batch (4): kernel planes cycle (tests/filters/test_gaussian.py:431-439)
    bag.add("gb_cycle", "gaussian_blur2d", dict(input=x, sigma=sig_t), dict(kernel_size=[3, 5], border_type="reflect", separable=True),
            dict(out=KF.gaussian_blur2d(x, (3, 5), sig_t)))

    # gradients
    def fgrads(fn, tensors, wrt):
        leaves = {k: (v.clone().requires_grad_(True) if k in wrt else v) for k, v in tensors.items()}
        out = fn(**leaves)
        cot = torch.rand(out.shape, generator=gen) - 0.5
        g = torch.autograd.grad((out * cot).sum(), [leaves[k] for k in wrt])
        outs = {"out": out, "cot": cot}
        for k, gi in zip(wrt, g):
            outs[f"grad_{k}"] = gi
        return outs

    for kn in ("k3x3", "k5x4", "k3x5_B", "k3x3_cyc"):
        for border in ("constant", "reflect", "replicate", "circular"):
            for normalized in (False, True):
                kw = dict(border_type=border, normalized=normalized, padding="same", behaviour="corr")
                o = fgrads(lambda input, kernel: KF.filter2d(input, kernel, **kw), dict(input=x, kernel=kernels[kn]), ("input", "kernel"))
                bag.add(f"g_f2d_{kn}_{border}_{int(normalized)}", "filter2d_grad", dict(input=x, kernel=kernels[kn], cot=o.pop("cot")), kw, o)
    kw = dict(border_type="reflect", normalized=False, padding="valid", behaviour="conv")
    o = fgrads(lambda input, kernel: KF.filter2d(input, kernel, **kw), dict(input=x, kernel=kernels["k5x4"]), ("input", "kernel"))
    bag.add("g_f2d_valid_conv", "filter2d_grad", dict(input=x, kernel=kernels["k5x4"], cot=o.pop("cot")), kw, o)
    for border in ("constant", "reflect", "replicate", "circular"):
        kw = dict(border_type=border, normalized=False, padding="same")
        o = fgrads(lambda input, kernel_x, kernel_y: KF.filter2d_separable(input, kernel_x, kernel_y, **kw),
                   dict(input=x, kernel_x=kxB, kernel_y=kyB), ("input", "kernel_x", "kernel_y"))
        bag.add(f"g_sep_{border}", "filter2d_separable_grad", dict(input=x, kernel_x=kxB, kernel_y=kyB, cot=o.pop("cot")), kw, o)
    for separable in (True, False):
        kw = dict(kernel_size=[5, 7], border_type="reflect", separable=separable)
        o = fgrads(lambda input, sigma: KF.gaussian_blur2d(input, (5, 7), sigma, "reflect", separable),
                   dict(input=xb, sigma=sig_t), ("input", "sigma"))
        bag.add(f"g_gb_{int(separable)}", "gaussian_blur2d_grad", dict(input=xb, sigma=sig_t, cot=o.pop("cot")), kw, o)
    bag.save(os.path.join(HERE, "filter.npz"))


if __name__ == "__main__":
    main()
