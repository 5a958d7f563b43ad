"""The sweep of the headline forward kernel (warp_fwd_tma<DYN>): every run of tiles drawn from one counter in raster order.  Only
who takes which tile changes, so the output must equal, bit for bit, the static deal (dyn_sched=0) and the generic kernel, and
every pixel must be written exactly once -- also at sizes that leave partial strips and partial tiles, with samples of the other
footprint class that the wide kernel skips, and inside a CUDA graph."""
import pytest
import torch

import kornia_b200 as K
from kornia_b200 import _lib
from kornia_b200.geometry import _prelude as P
from test_nonfinite_gpu import bits_equal
from test_parity_gpu import _bench_homographies, _wild_matrices

pytestmark = pytest.mark.gpu
DEV = "cuda"
B, H, W = 40, 1080, 1920  # 40 x 34 strips: above the 8 strips per CTA at which the forward takes the run-time distribution


def _forward_into_nan(src, M, dsize, projective, pad, align, fill=None):
    """kb200_warp_forward (bilinear) into an output prefilled with NaN: a pixel no kernel writes stays NaN."""
    n, C, Hs, Ws = src.shape
    h, w = dsize
    m = P.sampling_matrix(M, (Hs, Ws), (h, w), affine=not projective).contiguous()
    bx, by = P.meshgrid_axes(h, w, src.device, src.dtype) if projective else P.affine_axes(h, w, align, src.device, src.dtype)
    out = torch.full((n, C, h, w), float("nan"), device=src.device)
    _lib.call("kb200_warp_forward", src.data_ptr(), m.data_ptr(), bx.contiguous().data_ptr(), by.contiguous().data_ptr(),
              None if fill is None else fill.data_ptr(), out.data_ptr(), n, C, Hs, Ws, h, w, m.shape[0], int(projective), _lib.BILINEAR,
              _lib.PADDING[pad], int(align), _lib.F32, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return out


@pytest.fixture(scope="module")
def batch():
    torch.manual_seed(7)
    src = torch.rand(B, 3, H, W, device=DEV)
    # bench homographies, then rotations, zooms, a horizon, out-of-view samples: exact-path pixels and samples of the 32 x 32 tiles
    M = torch.cat([_bench_homographies(B - 10, H, W, 11), _wild_matrices(H, W)]).to(DEV)
    return src, M


@pytest.mark.parametrize("pad", ["zeros", "border", "reflection", "fill"])
@pytest.mark.parametrize("projective", [True, False])
def test_sweep_bit_identical_to_static_deal_and_generic(batch, pad, projective):
    src, M = batch
    if not projective:
        M = M[:, :2].contiguous()
    fill = torch.tensor([0.2, 0.5, 0.8], device=DEV) if pad == "fill" else None
    assert K.config.get("dyn_sched") == 1
    for dsize in ((H, W), (1000, 1900)):  # 1000 x 1900: a partial last strip and a partial last tile in every strip
        for align in (True, False):
            run = lambda: _forward_into_nan(src, M, dsize, projective, pad, align, fill)  # noqa: E731
            sweep = run()
            assert _lib.last_warp_variant() == "tma_tile"
            assert not torch.isnan(sweep).any(), (dsize, align, "a pixel was not written")
            with K.config.override(dyn_sched=0):
                deal = run()
            with K.config.override(tma=0):
                gen = run()
                assert _lib.last_warp_variant() == "generic"
            assert bits_equal(sweep, deal), (dsize, align, float((sweep - deal).abs().max()))
            assert bits_equal(sweep, gen), (dsize, align, float((sweep - gen).abs().max()))


def test_sweep_inside_a_cuda_graph():
    """The launch zeroes its work counter on its stream, which a capture records: replays start from zero."""
    many = torch.rand(400, 3, 96, 192, device=DEV)  # 1 200 strips of three tiles
    Mm = _bench_homographies(400, 96, 192, 5).to(DEV)
    with K.config.override(tma=0):
        want = K.warp_perspective(many, Mm, (96, 192))
    with K.config.override(dyn_sched=0):
        deal = K.warp_perspective(many, Mm, (96, 192))
    assert torch.equal(deal, want)
    graphed = K.graphs.GraphedCall(lambda a, b: K.warp_perspective(a, b, (96, 192)), many, Mm)
    for _ in range(3):
        got = graphed(many, Mm)
        assert torch.equal(got, want)
