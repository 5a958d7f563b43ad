"""ctypes binding of ``libkornia_b200.so`` (the C ABI declared in include/kornia_b200.h).

The library is built in-tree by :func:`kornia_b200.build.build` (``__graft_entry__.build()``).
There is no fallback of any kind: if the library is missing or a call fails, a ``RuntimeError``
is raised.
"""
from __future__ import annotations

import ctypes
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_C", "libkornia_b200.so")
ABI_VERSION = 1

F32, F64 = 0, 1
BILINEAR, NEAREST, BICUBIC = 0, 1, 2
ZEROS, BORDER, REFLECTION, FILL = 0, 1, 2, 3
CONSTANT, REFLECT, REPLICATE, CIRCULAR = 0, 1, 2, 3

INTERP = {"bilinear": BILINEAR, "nearest": NEAREST, "bicubic": BICUBIC}
PADDING = {"zeros": ZEROS, "border": BORDER, "reflection": REFLECTION, "fill": FILL}
BORDERS = {"constant": CONSTANT, "reflect": REFLECT, "replicate": REPLICATE, "circular": CIRCULAR}

_vp, _i, _sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t

# name -> (restype, argtypes); must list every symbol of include/kornia_b200.h
SIGNATURES = {
    "kb200_abi_version": (_i, []),
    "kb200_last_error": (ctypes.c_char_p, []),
    "kb200_last_warp_variant": (ctypes.c_char_p, []),
    "kb200_last_warp_launches": (_i, []),
    "kb200_set_option": (_i, [ctypes.c_char_p, _i]),
    "kb200_get_option": (_i, [ctypes.c_char_p]),
    "kb200_warp_forward": (_i, [_vp] * 6 + [_i] * 12 + [_vp]),
    "kb200_warp_prelude": (_i, [_vp, _vp] + [_i] * 8 + [_vp]),
    "kb200_warp_prelude_backward": (_i, [_vp, _vp, _vp] + [_i] * 7 + [_vp]),
    "kb200_warp_backward_workspace_bytes": (_sz, [_i] * 4),
    "kb200_warp_backward": (_i, [_vp] * 9 + [_i] * 12 + [_vp]),
    "kb200_remap_forward": (_i, [_vp] * 4 + [_i] * 12 + [_vp]),
    "kb200_remap_backward": (_i, [_vp] * 7 + [_i] * 12 + [_vp]),
    "kb200_undistort_forward": (_i, [_vp] * 3 + [_i] * 5 + [_vp]),
    "kb200_warp_u8hwc_forward": (_i, [_vp] * 6 + [_i] * 12 + [_vp]),
    "kb200_undistort_u8hwc_forward": (_i, [_vp] * 3 + [_i] * 5 + [_vp]),
    "kb200_filter2d_forward": (_i, [_vp] * 3 + [_i] * 10 + [_vp]),
    "kb200_filter2d_backward_input": (_i, [_vp] * 3 + [_i] * 10 + [_vp]),
    "kb200_filter2d_backward_kernel_workspace_bytes": (_sz, [_i] * 8),
    "kb200_filter2d_backward_kernel": (_i, [_vp] * 4 + [_i] * 10 + [_vp]),
    "kb200_pyrdown_forward": (_i, [_vp] * 3 + [_i] * 7 + [_vp]),
    "kb200_sepfilter_forward": (_i, [_vp] * 4 + [_i] * 11 + [_vp]),
    "kb200_rotation_matrix2d": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "kb200_perspective_from_points": (_i, [_vp, _vp, _vp, _i, _i, _i, _vp]),
    "kb200_ssim_forward": (_i, [_vp] * 4 + [_i] * 4 + [ctypes.c_double] * 3 + [_i, _vp]),
    "kb200_spatial_gradient_forward": (_i, [_vp, _vp, _vp] + [_i] * 6 + [ctypes.c_double, _i, _vp]),
    "kb200_spatial_gradient_backward": (_i, [_vp, _vp, _vp] + [_i] * 6 + [_vp]),
    "kb200_feature_response_forward": (_i, [_vp, _vp, _vp, ctypes.c_double, _vp, _vp, _vp] + [_i] * 8 + [_vp]),
    "kb200_scale_octave_forward": (_i, [_vp, _vp, _vp, _i, _vp] + [_i] * 4 + [_vp]),
    "kb200_nms2d_forward": (_i, [_vp, _vp] + [_i] * 4 + [ctypes.c_longlong] * 2 + [_i] * 3 + [_vp]),
    "kb200_nms3d_forward": (_i, [_vp] * 3 + [_i] * 5 + [ctypes.c_longlong] * 3 + [_i] * 2 + [_vp]),
    "kb200_quad_interp3d_forward": (_i, [_vp] * 4 + [_i] * 5 + [ctypes.c_longlong] * 8 + [_i] * 2 + [ctypes.c_float] * 2 + [_i] * 3 + [_vp]),
    "kb200_sift_describe_forward": (_i, [_vp] * 4 + [ctypes.c_longlong, _i, ctypes.c_longlong, ctypes.c_longlong] + [_i] * 6 + [ctypes.c_float] * 2 + [_i, _vp]),
    "kb200_patch_orientation_forward": (_i, [_vp] * 4 + [ctypes.c_longlong, _i, ctypes.c_longlong, ctypes.c_longlong, _i, ctypes.c_float, _i, _vp]),
    "kb200_extract_patches_forward": (_i, [_vp, _vp, _i, _vp, _vp, _vp, ctypes.c_longlong, ctypes.c_longlong] + [_i] * 5 + [_vp]),
    "kb200_patch_affine_shape_forward": (_i, [_vp] * 3 + [ctypes.c_longlong, _i, ctypes.c_longlong, ctypes.c_longlong, ctypes.c_float, _i, _vp]),
    "kb200_laf_affine_shape_forward": (_i, [_vp, _vp, _i, _vp, _vp, _vp, _vp, ctypes.c_longlong, ctypes.c_longlong, _i, ctypes.c_float, _i, _i,
                                            _vp]),
    "kb200_sepfilter_lerp_forward": (_i, [_vp] * 4 + [_i] * 10 + [ctypes.c_double, _i, _vp]),
    "kb200_debug_fastdiv_mismatches": (_i, [_vp, _vp, _i, _vp, _vp]),
}

_lock = threading.Lock()
_lib = None


def load() -> ctypes.CDLL:
    """Load (once) and type the shared library; raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"kornia_b200: CUDA library not found at {LIB_PATH}. Build it with "
                "`python -c 'import __graft_entry__ as g; g.build()'` (needs nvcc). There is no CPU fallback."
            )
        lib = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError if the symbol is missing
            fn.restype = res
            fn.argtypes = args
        got = lib.kb200_abi_version()
        if got != ABI_VERSION:
            raise RuntimeError(f"kornia_b200: ABI mismatch, library reports {got}, binding expects {ABI_VERSION}")
        _lib = lib
    return _lib


class Unsupported(RuntimeError):
    """The C entry point declined a valid request (status KB200_EUNSUPPORTED): the caller may route it
    through other entry points of the library."""


def call(name: str, *args) -> None:
    """Invoke an int-returning entry point and turn a non-zero status into ``RuntimeError``."""
    lib = load()
    rc = getattr(lib, name)(*args)
    if rc != 0:
        msg = lib.kb200_last_error().decode(errors="replace")
        raise (Unsupported if rc == -3 else RuntimeError)(f"{name} failed (status {rc}): {msg}")


def last_warp_variant() -> str:
    return load().kb200_last_warp_variant().decode()


def last_warp_launches() -> int:
    return int(load().kb200_last_warp_launches())
