"""Golden vectors for motion blur: get_motion_kernel2d, motion_blur and RandomMotionBlur of the UNMODIFIED reference run
on CPU fp32.  Needs a checkout of the reference (make_golden.import_reference):

    python tests/golden/make_golden_motion.py        ->  tests/golden/motion.npz (shards motion.<k>.npz)

Cases:
  kernel_*   get_motion_kernel2d for K in {3, 5, 9, 15, 31} x number / (B,) tensor arguments x 'nearest' / 'bilinear';
             the kernels are recorded so that a rounding tie of the nearest rotation shows as a kernel mismatch
  blur_*     motion_blur for the four borders (the kernel too), with the gradients of sum(out * cot) w.r.t. the input,
             angle and direction
  aug_*      RandomMotionBlur from a pinned seed: every tensor of the parameter dictionary and the output, for int and
             (min, max) kernel_size, same_on_batch and p < 1
"""
from __future__ import annotations

import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import Bag, import_reference, smooth_image  # noqa: E402


def main():
    import_reference()
    import kornia
    from kornia.filters import get_motion_kernel2d, motion_blur

    torch.set_num_threads(1)
    gen = torch.Generator().manual_seed(777)
    bag = Bag()

    # ---- kernels
    for K in (3, 5, 9, 15, 31):
        for mode in ("nearest", "bilinear"):
            ang, dirn = 35.0 + K, 0.5 - 0.1 * K / 31
            k = get_motion_kernel2d(K, ang, dirn, mode)
            bag.add(f"kernel_K{K}_{mode}_number", "get_motion_kernel2d", {}, {"kernel_size": K, "angle": ang, "direction": dirn, "mode": mode},
                    {"kernel": k})
            angle = torch.rand(4, generator=gen) * 360.0 - 180.0
            direction = torch.rand(4, generator=gen) * 2.4 - 1.2  # a little outside [-1, 1]: the clamp
            k = get_motion_kernel2d(K, angle, direction, mode)
            bag.add(f"kernel_K{K}_{mode}_batched", "get_motion_kernel2d", {"angle": angle, "direction": direction},
                    {"kernel_size": K, "mode": mode}, {"kernel": k})

    # ---- motion_blur with gradients
    x = smooth_image(3, 2, 40, 52, gen)
    for K, border, mode in ((5, "constant", "nearest"), (9, "reflect", "bilinear"), (15, "replicate", "nearest"), (9, "circular", "bilinear"),
                            (31, "constant", "bilinear")):
        angle = torch.rand(3, generator=gen) * 360.0 - 180.0
        direction = torch.rand(3, generator=gen) * 2.0 - 1.0
        cot = torch.rand(3, 2, 40, 52, generator=gen)
        xi, ai, di = x.clone().requires_grad_(True), angle.clone().requires_grad_(True), direction.clone().requires_grad_(True)
        out = motion_blur(xi, K, ai, di, border, mode)
        gx, ga, gd = torch.autograd.grad((out * cot).sum(), [xi, ai, di], allow_unused=True)
        outs = {"out": out.detach(), "kernel": get_motion_kernel2d(K, angle, direction, mode), "cot": cot, "grad_input": gx,
                "grad_angle": ga if ga is not None else torch.zeros_like(angle), "grad_direction": gd if gd is not None else torch.zeros_like(direction)}
        bag.add(f"blur_K{K}_{border}_{mode}", "motion_blur", {"input": x, "angle": angle, "direction": direction},
                {"kernel_size": K, "border_type": border, "mode": mode}, outs)
    out = motion_blur(x, 9, 30.0, -0.3, "reflect")
    bag.add("blur_K9_reflect_number", "motion_blur", {"input": x}, {"kernel_size": 9, "angle": 30.0, "direction": -0.3, "border_type": "reflect",
                                                                     "mode": "nearest"}, {"out": out, "kernel": get_motion_kernel2d(9, 30.0, -0.3)})

    # ---- RandomMotionBlur parameter streams
    noise = torch.rand(5, 3, 24, 32, generator=gen)

    def record(name, ctor, seed):
        aug = kornia.augmentation.RandomMotionBlur(**{k: (tuple(v) if isinstance(v, list) else v) for k, v in ctor.items()})
        torch.manual_seed(seed)
        out = aug(noise)
        outs = {"out": out}
        for k, v in aug._params.items():
            if isinstance(v, torch.Tensor):
                outs[f"param_{k}"] = v
        bag.add(name, "RandomMotionBlur", {"input": noise}, {"ctor": ctor, "seed": seed}, outs)

    record("aug_int", dict(kernel_size=9, angle=35.0, direction=0.5, p=1.0), 1)
    record("aug_tuple", dict(kernel_size=[3, 15], angle=[-20.0, 60.0], direction=[-0.5, 1.0], border_type="reflect", p=1.0), 2)
    record("aug_same_on_batch", dict(kernel_size=[5, 11], angle=45.0, direction=0.3, same_on_batch=True, resample="BILINEAR", p=1.0), 3)
    record("aug_gated", dict(kernel_size=7, angle=90.0, direction=1.0, border_type="replicate", p=0.5), 4)
    record("aug_gated_tuple", dict(kernel_size=[3, 9], angle=10.0, direction=0.0, p=0.3), 5)
    bag.save(os.path.join(HERE, "motion.npz"))


if __name__ == "__main__":
    main()
