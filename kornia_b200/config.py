"""Kernel-selection switches of the engine.

Every switch is read from the environment ONCE -- ``KB200_<NAME>=0|1`` when the package (for the host-side ones) or the
shared library (for the device-side ones, include/kornia_b200.h: kb200_set_option) is loaded -- and can be changed
afterwards only through this module; nothing on the call path touches ``os.environ``.  Each default names, beside the
kernel in csrc/, the measurement behind it and the GPU it was taken on; the parity tests flip a switch
to run a kernel against the one it stands in for.

Device-side (forwarded to the C library): ``tma`` (TMA-tiled warp / remap / backward kernels; off = generic per-pixel
kernels), ``tiled_filter`` (shared-memory filter kernels; off = generic), ``square_tiles`` (second forward tile shape for
rotated samples), ``tiled_gradient``, ``u8_tiled`` (staged-window uint8 ingest warp; off = per-tap kernel), ``bwd_stride1``
(tiled backward on stride-1 lanes; off = column-pair lanes), ``dyn_sched`` (warp forward and backward: the last rounds of strips /
every warp's work drawn at run time from a per-device ring of counters; off = dealt out in advance), ``sweep`` (forward kernel
under ``dyn_sched``: every run of tiles drawn in raster order, so the grid sweeps each image as one band; off = the strip deal
of the next two switches), ``dyn_chunk`` (tiles per chunk of the strip deal, 10), ``dyn_static`` (percent of the full rounds
the strip deal hands out in advance, 85).
Host-side: ``fused_pyrdown`` (5x5 blur + 2x decimation in one kernel), ``fused_undistort`` (lens model evaluated inside
the sampling kernel), ``fast_filter_bwd`` (input gradient of the separable filter through the one-pass forward kernel),
``torch_prelude`` (the (B,3,3) matrix chain as the reference's torch op sequence instead of one launch; needed for double
backward through M).
"""
from __future__ import annotations

import contextlib
import os

from . import _lib

DEVICE_OPTIONS = ("tma", "tiled_filter", "square_tiles", "tiled_gradient", "u8_tiled", "bwd_stride1", "dyn_sched", "dyn_chunk", "dyn_static",
                  "sweep")
_HOST_DEFAULTS = {"fused_pyrdown": 1, "fused_undistort": 1, "fast_filter_bwd": 1, "torch_prelude": 0}


def _env(name: str, default: int) -> int:
    v = os.environ.get("KB200_" + name.upper(), "")
    if name == "torch_prelude" and not v:
        v = os.environ.get("KORNIA_B200_TORCH_PRELUDE", "")  # round-1 spelling
    try:
        return int(v) if v else default
    except ValueError:
        return default


_host = {k: _env(k, d) for k, d in _HOST_DEFAULTS.items()}
_device_initial: dict = {}


def _remember_initial() -> None:
    if not _device_initial:
        lib = _lib.load()
        for k in DEVICE_OPTIONS:
            _device_initial[k] = int(lib.kb200_get_option(k.encode()))


def get(name: str) -> int:
    if name in _host:
        return _host[name]
    if name in DEVICE_OPTIONS:
        return int(_lib.load().kb200_get_option(name.encode()))
    raise KeyError(f"kornia_b200.config: unknown option {name!r}")


def enabled(name: str) -> bool:
    return _host[name] != 0  # host-side switches only: on the call path of the public functions, no library call


def set(name: str, value) -> None:  # noqa: A001 -- mirrors kb200_set_option
    value = int(value)
    if name in _host:
        _host[name] = value
    elif name in DEVICE_OPTIONS:
        _remember_initial()
        _lib.call("kb200_set_option", name.encode(), value)
    else:
        raise KeyError(f"kornia_b200.config: unknown option {name!r}")


def reset() -> None:
    """Back to what the environment / the built-in defaults said at load time."""
    for k, d in _HOST_DEFAULTS.items():
        _host[k] = _env(k, d)
    if _device_initial:
        for k, v in _device_initial.items():
            _lib.call("kb200_set_option", k.encode(), v)


@contextlib.contextmanager
def override(**values):
    """``with config.override(tma=0): ...`` -- temporary switch values (tests, benchmarks of one kernel against another)."""
    before = {k: get(k) for k in values}
    try:
        for k, v in values.items():
            set(k, v)
        yield
    finally:
        for k, v in before.items():
            set(k, v)
