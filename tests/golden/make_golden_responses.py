"""Golden vectors for the feature responses: harris_response, gftt_response and hessian_response of the UNMODIFIED
reference run on CPU fp32.  Needs a checkout of the reference (make_golden.import_reference):

    python tests/golden/make_golden_responses.py        ->  tests/golden/responses.npz (shards responses.<k>.npz)

Cases: the three functions x 'sobel' / 'diff', Harris k as a float and as a 0-d tensor, sigmas None and (B,), C in {1, 3},
W % 4 != 0 and H = W = 4; every case records the gradient of sum(out * cot) with respect to the input.
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
    from kornia.feature.responses import gftt_response, harris_response, hessian_response

    torch.set_num_threads(1)
    gen = torch.Generator().manual_seed(4242)
    bag = Bag()
    shapes = [(2, 1, 24, 32), (2, 3, 20, 30), (1, 1, 4, 4)]
    for si, shape in enumerate(shapes):
        x = smooth_image(*shape, gen)
        x = x + 0.05 * torch.rand(shape, generator=gen)  # corners and blobs at more than one scale
        sigmas = torch.rand(shape[0], generator=gen) * 2 + 0.5
        cot = torch.rand(shape, generator=gen)
        for mode in ("sobel", "diff"):
            for with_sigmas in (False, True):
                sig = sigmas if with_sigmas else None
                forms = [("harris", 0.04, False), ("harris", 0.05, True), ("gftt", None, False), ("hessian", None, False)]
                for fn, k, k_tensor in forms:
                    xi = x.clone().requires_grad_(True)
                    ins = {"input": x, "cot": cot}
                    if sig is not None:
                        ins["sigmas"] = sig
                    kw = {"grads_mode": mode}
                    if fn == "harris":
                        kk = torch.tensor(k) if k_tensor else k
                        if k_tensor:
                            ins["k"] = kk
                        else:
                            kw["k"] = k
                        out = harris_response(xi, kk, mode, sig)
                    elif fn == "gftt":
                        out = gftt_response(xi, mode, sig)
                    else:
                        out = hessian_response(xi, mode, sig)
                    (g,) = torch.autograd.grad((out * cot).sum(), [xi])
                    name = f"{fn}_{'x'.join(map(str, shape))}_{mode}_{'sig' if sig is not None else 'nosig'}" + ("_ktensor" if k_tensor else "")
                    bag.add(name, fn + "_response", ins, kw, {"out": out.detach(), "grad_input": g})
    bag.save(os.path.join(HERE, "responses.npz"))


if __name__ == "__main__":
    main()
