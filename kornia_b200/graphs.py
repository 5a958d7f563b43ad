"""CUDA-graph replay of a launch-bound call (small images: a 32 x 3 x 256 x 256 warp is a few microseconds of device work behind
several times as much Python, dispatcher and launch cost).  ``GraphedCall(fn, *example_tensors)`` captures ``fn`` once on static buffers -- every kernel
of this library launches on the capturing stream and allocates nothing inside the C ABI, so prelude + warp + blur chains capture
as they are -- and replays it per call: copy the inputs into the static buffers, one ``cudaGraphLaunch``, read the static output.
Forward only, fixed shapes and dtypes (a new shape needs a new capture); the tensors returned are overwritten by the next call.

The reference's answer to the same overhead is ``torch.compile`` (benchmarks/README.md:154: 96 k -> 232 k img/s); this is the
H100-native one: streams and graphs instead of a tracing compiler."""
from __future__ import annotations

from typing import Callable, Sequence

import torch

__all__ = ["GraphedCall"]


class GraphedCall:
    def __init__(self, fn: Callable[..., torch.Tensor], *example: torch.Tensor, warmup: int = 3):
        if not example or not all(isinstance(t, torch.Tensor) and t.is_cuda for t in example):
            raise RuntimeError("kornia_b200.graphs: GraphedCall needs CUDA example tensors (shapes and dtypes are baked into the graph)")
        self._static_in = [t.detach().clone() for t in example]
        self._graph = torch.cuda.CUDAGraph()
        side = torch.cuda.Stream(example[0].device)
        side.wait_stream(torch.cuda.current_stream(example[0].device))
        with torch.no_grad(), torch.cuda.stream(side):
            for _ in range(warmup):  # lazy initialisation (tensor maps, shared-memory attributes, caches) happens outside the capture
                fn(*self._static_in)
        torch.cuda.current_stream(example[0].device).wait_stream(side)
        with torch.no_grad(), torch.cuda.graph(self._graph):
            self._static_out = fn(*self._static_in)

    def __call__(self, *tensors: torch.Tensor):
        if len(tensors) != len(self._static_in):
            raise RuntimeError(f"kornia_b200.graphs: captured with {len(self._static_in)} tensors, called with {len(tensors)}")
        for dst, src in zip(self._static_in, tensors):
            if src.shape != dst.shape or src.dtype != dst.dtype:
                raise RuntimeError(f"kornia_b200.graphs: captured for {tuple(dst.shape)} {dst.dtype}, got {tuple(src.shape)} {src.dtype}")
            if src.data_ptr() != dst.data_ptr():
                dst.copy_(src, non_blocking=True)
        self._graph.replay()
        return self._static_out

    @property
    def inputs(self) -> Sequence[torch.Tensor]:
        """The static input buffers: write into them directly to skip the per-call copies."""
        return self._static_in
