"""Host-side contract of the drop-in (no GPU needed): signatures, validation order, exception
types and message fragments -- all raised before any device work (SURVEY.md section 8b) -- and the
C ABI: the library loads and exports every symbol include/kornia_b200.h declares."""
import ctypes
import inspect
import os
import re

import pytest
import torch

import kornia_b200 as K
from kornia_b200 import _lib
from kornia_b200.core import BaseError, ShapeError, TypeCheckError

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_signatures_match_reference():
    # kornia/geometry/transform/imgwarp.py:69-77,177-185,625-633; filters/filter.py:54-61,155-162; gaussian.py:32-38
    want = {
        K.warp_perspective: "(src, M, dsize, mode='bilinear', padding_mode='zeros', align_corners=True, fill_value=None)",
        K.warp_affine: "(src, M, dsize, mode='bilinear', padding_mode='zeros', align_corners=True, fill_value=None)",
        K.remap: "(image, map_x, map_y, mode='bilinear', padding_mode='zeros', align_corners=None, normalized_coordinates=False)",
        K.filter2d: "(input, kernel, border_type='reflect', normalized=False, padding='same', behaviour='corr')",
        K.filter2d_separable: "(input, kernel_x, kernel_y, border_type='reflect', normalized=False, padding='same')",
        K.gaussian_blur2d: "(input, kernel_size, sigma, border_type='reflect', separable=True)",
    }
    for fn, sig in want.items():
        params = inspect.signature(fn).parameters.values()
        got = "(" + ", ".join(p.name if p.default is inspect._empty else f"{p.name}={p.default!r}" for p in params) + ")"
        assert got == sig, fn.__name__


def test_module_layout_mirrors_reference():
    assert K.geometry.transform.warp_perspective is K.warp_perspective
    assert K.geometry.warp_affine is K.warp_affine
    assert K.filters.gaussian_blur2d is K.gaussian_blur2d
    assert K.filters.GaussianBlur2d((3, 3), (1.0, 1.0)).kernel_size == (3, 3)


def test_warp_exceptions():
    # tests/geometry/transform/test_imgwarp.py:232-249,367-384
    img = torch.rand(1, 2, 3, 4)
    for fn, M in ((K.warp_affine, torch.eye(2, 3)[None]), (K.warp_perspective, torch.eye(3)[None])):
        with pytest.raises(TypeError):
            fn(0.0, M, (4, 5))
        with pytest.raises(TypeError):
            fn(img, 0.0, (4, 5))
        with pytest.raises(ValueError):
            fn(torch.rand(2, 3, 4), M, (4, 5))
        with pytest.raises(ValueError):
            fn(img, torch.eye(2, 2)[None], (4, 5))
    with pytest.raises(ValueError, match="only supported for 3 channels"):
        K.warp_perspective(torch.rand(1, 3, 4, 4), torch.eye(3)[None], (4, 4), padding_mode="fill", fill_value=torch.zeros(2))
    with pytest.raises(RuntimeError, match="same batch size"):
        K.warp_perspective(torch.rand(2, 3, 4, 4), torch.eye(3)[None], (4, 4))
    with pytest.raises(ValueError):
        K.warp_perspective(img, torch.eye(3)[None], (4, 4), mode="cubic")


def test_cpu_tensors_fail_loudly():
    with pytest.raises(RuntimeError, match="CUDA-only"):
        K.warp_perspective(torch.rand(1, 3, 4, 4), torch.eye(3)[None], (4, 4))
    with pytest.raises(RuntimeError, match="CUDA-only"):
        K.filter2d(torch.rand(1, 1, 5, 5), torch.ones(1, 3, 3))
    with pytest.raises(RuntimeError, match="CUDA-only"):
        K.remap(torch.rand(1, 1, 5, 5), torch.zeros(1, 2, 2), torch.zeros(1, 2, 2))


def test_filter_exceptions_and_messages():
    # tests/filters/test_filters.py:104-133
    k = torch.ones(1, 1, 1)
    with pytest.raises(TypeCheckError, match="Type mismatch: expected Tensor"):
        K.filter2d(1, k)
    with pytest.raises(TypeCheckError, match="Type mismatch: expected Tensor"):
        K.filter2d(torch.ones(1, 1, 1, 1), 1)
    with pytest.raises(ShapeError, match="Shape dimension mismatch"):
        K.filter2d(torch.ones(1), k)
    with pytest.raises(ShapeError, match=r"\['B', 'C', 'H', 'W'\]"):
        K.filter2d(torch.ones(1), k)
    with pytest.raises(ShapeError, match="Shape dimension mismatch"):
        K.filter2d(torch.ones(1, 1, 1, 1), torch.ones(1))
    with pytest.raises(BaseError, match="Invalid border, a. Ex"):
        K.filter2d(torch.ones(1, 1, 1, 1), k, border_type="a")
    with pytest.raises(BaseError, match="Invalid padding mode, a. Ex"):
        K.filter2d(torch.ones(1, 1, 1, 1), k, padding="a")
    with pytest.raises(BaseError, match="Invalid padding mode, a. Ex"):
        K.filter2d(torch.ones(1, 1, 1, 1), k, behaviour="a")


def test_gaussian_exceptions_and_messages():
    # tests/filters/test_gaussian.py:244-255,356-390
    x = torch.rand(1, 1, 5, 5)
    with pytest.raises(TypeCheckError):
        K.gaussian_blur2d(1, 3, (1.0, 1.0))
    with pytest.raises(TypeCheckError):
        K.gaussian_blur2d(x, 3, 1.0)
    with pytest.raises(BaseError, match="sigma must be positive"):
        K.gaussian_blur2d(x, 3, (0.0, 1.0))
    with pytest.raises(BaseError, match="sigma must be positive"):
        K.gaussian_blur2d(x, 3, torch.tensor([[1.0, -1.0]]))
    for bad in (4, (3, 4), 0, -3):
        with pytest.raises(BaseError, match="Kernel size must be"):
            K.gaussian_blur2d(x, bad, (1.0, 1.0))
    with pytest.raises(ShapeError):
        K.gaussian_blur2d(torch.rand(5, 5), 3, (1.0, 1.0))
    with pytest.raises(ShapeError):
        K.remap(torch.rand(1, 5, 5), torch.zeros(1, 2, 2), torch.zeros(1, 2, 2))


def test_checks_switch():
    # kornia/core/check.py:63-125: disabling checks turns the KORNIA_CHECK* family into no-ops
    import importlib

    C = importlib.import_module("kornia_b200.core.check")

    C.disable_checks()
    try:
        assert not C.checks_enabled()
        C.check_is_tensor(1)
        C.check(False, "x")
        C.check_shape(torch.ones(1), ["B", "C", "H", "W"])
    finally:
        C.enable_checks()
    with pytest.raises(BaseError):
        C.check(False, "x")


def test_gaussian_taps_literals():
    # docstring pins, kornia/filters/kernels.py:572-579,685-703
    from kornia_b200.filters import get_gaussian_kernel1d, get_gaussian_kernel2d

    torch.testing.assert_close(get_gaussian_kernel1d(3, 2.5), torch.tensor([[0.3243, 0.3513, 0.3243]]), atol=1e-4, rtol=0)
    k2 = get_gaussian_kernel2d((3, 5), (1.5, 1.5))
    assert k2.shape == (1, 3, 5)
    torch.testing.assert_close(k2[0, 1], torch.tensor([0.0462, 0.0899, 0.1123, 0.0899, 0.0462]), atol=1e-4, rtol=0)
    torch.testing.assert_close(k2.sum(), torch.tensor(1.0))


def test_prelude_matches_oracle_bitwise():
    from kornia_b200.geometry import _prelude as P
    from oracle import kornia_restated as R

    g = torch.Generator().manual_seed(0)
    M = torch.eye(3)[None].repeat(5, 1, 1) + 0.1 * torch.randn(5, 3, 3, generator=g)
    a = P.inverse3x3(P.normalize_homography(M, (1080, 1920), (720, 1280)))
    b = R.inv3x3(R.normalized_homography(M, (1080, 1920), (720, 1280)))
    assert torch.equal(a, b)
    for x, y in zip(P.meshgrid_axes(7, 9, "cpu", torch.float32), R.meshgrid_axes(7, 9, "cpu")):
        assert torch.equal(x, y)


# ------------------------------------------------------------------ C ABI
def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "kornia_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(kb200_\w+)\s*\(", text)))


def test_c_abi_exports_every_declared_symbol():
    names = _declared_symbols()
    assert len(names) >= 13
    assert os.path.exists(_lib.LIB_PATH), "run __graft_entry__.build() first"
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/kornia_b200.h but not exported"
    assert sorted(_lib.SIGNATURES) == names, "python binding and header disagree"


def test_kernel_selection_switches_agree_everywhere():
    """The option table of the C library, kornia_b200.config and the header's list name the same switches; unknown names are
    refused; a set is read back.  (No GPU needed: the table lives on the host.)"""
    import re
    from kornia_b200 import config

    lib = _lib.load()
    header = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "kornia_b200.h")).read()
    block = header[header.index("Kernel-selection switches"):header.index("int kb200_set_option")]
    named = set(re.findall(r'"([a-z0-9_]+)"', block))
    assert named == set(config.DEVICE_OPTIONS), (sorted(named), sorted(config.DEVICE_OPTIONS))
    int_min = -(2 ** 31)
    for name in config.DEVICE_OPTIONS:
        before = lib.kb200_get_option(name.encode())
        assert before != int_min, name
        assert lib.kb200_set_option(name.encode(), before) == 0
        assert lib.kb200_get_option(name.encode()) == before
    assert lib.kb200_get_option(b"no_such_switch") == int_min
    assert lib.kb200_set_option(b"no_such_switch", 1) != 0
    config.set("dyn_sched", 0)
    assert config.get("dyn_sched") == 0 and lib.kb200_get_option(b"dyn_sched") == 0
    config.reset()
    assert config.get("dyn_sched") == 1
    for name in ("sweep", "dyn_chunk", "dyn_static"):  # removed switches are unknown names
        assert lib.kb200_set_option(name.encode(), 1) != 0, name
        assert lib.kb200_get_option(name.encode()) == int_min, name
        with pytest.raises(KeyError):
            config.set(name, 1)


def test_c_abi_version_and_error_channel():
    lib = _lib.load()
    assert lib.kb200_abi_version() == _lib.ABI_VERSION
    # argument validation happens on the host, before any CUDA call: usable without a GPU
    rc = lib.kb200_warp_forward(None, None, None, None, None, None, 1, 3, 4, 4, 4, 4, 1, 1, 0, 0, 1, 0, None)
    assert rc == -1 and b"null src" in lib.kb200_last_error()
    rc = lib.kb200_filter2d_forward(ctypes.c_void_p(8), ctypes.c_void_p(8), ctypes.c_void_p(8), 3, 1, 4, 4, 2, 3, 3, 1, 1, 0, None)
    assert rc == -1 and b"must divide" in lib.kb200_last_error()


def test_c_abi_validation_of_the_caller_entry_points():
    """Entry points behind the callers of the path (spatial_gradient / sobel, ssim, unsharp, the two matrix builders):
    bad requests are refused on the host, before any CUDA call, with the documented status."""
    lib = _lib.load()
    p8 = ctypes.c_void_p(8)  # non-null dummy; never dereferenced on these paths
    taps = (ctypes.c_double * 18)(*([0.0] * 18))
    assert lib.kb200_spatial_gradient_forward(p8, taps, p8, 6, 8, 8, 2, 4, 0, 0.0, 0, None) == -1          # 4x4 stencils do not exist
    assert b"unsupported stencil" in lib.kb200_last_error()
    assert lib.kb200_spatial_gradient_forward(p8, taps, p8, 6, 8, 8, 3, 3, 1, 1e-6, 0, None) == -1         # magnitude needs two outputs
    assert lib.kb200_spatial_gradient_forward(p8, None, p8, 6, 8, 8, 2, 3, 0, 0.0, 0, None) == -1 and b"null taps" in lib.kb200_last_error()
    assert lib.kb200_spatial_gradient_backward(p8, taps, p8, 0, 8, 8, 2, 3, 0, None) == -1                 # no planes
    assert lib.kb200_spatial_gradient_forward(p8, taps, p8, 6, 8, 8, 2, 3, 0, 0.0, 7, None) == -1 and b"bad dtype" in lib.kb200_last_error()
    assert lib.kb200_ssim_forward(p8, p8, p8, p8, 6, 8, 8, 5, 1e-4, 9e-4, 1e-12, 1, None) == -3            # fp64 -> the host composes
    assert lib.kb200_ssim_forward(p8, p8, p8, p8, 6, 8, 8, 13, 1e-4, 9e-4, 1e-12, 0, None) == -3 and b"up to 11 taps" in lib.kb200_last_error()
    assert lib.kb200_ssim_forward(p8, p8, p8, p8, 6, 8, 8, 4, 1e-4, 9e-4, 1e-12, 0, None) == -3            # even window
    assert lib.kb200_ssim_forward(p8, None, p8, p8, 6, 8, 8, 5, 1e-4, 9e-4, 1e-12, 0, None) == -1
    assert lib.kb200_ssim_forward(p8, p8, p8, p8, 6, 2, 8, 5, 1e-4, 9e-4, 1e-12, 0, None) == -1 and b"reflect border" in lib.kb200_last_error()
    assert lib.kb200_sepfilter_lerp_forward(p8, p8, p8, p8, 2, 3, 8, 8, 1, 5, 1, 5, 1, 1, 2.0, 1, None) == -3  # fp64
    assert lib.kb200_sepfilter_lerp_forward(p8, p8, p8, p8, 2, 3, 8, 8, 1, 13, 1, 13, 1, 1, 2.0, 0, None) == -3  # > 11 taps
    assert lib.kb200_sepfilter_lerp_forward(p8, p8, p8, p8, 2, 3, 8, 8, 1, 5, 1, 5, 3, 1, 2.0, 0, None) == -3   # circular border
    assert lib.kb200_sepfilter_lerp_forward(p8, p8, None, p8, 2, 3, 8, 8, 1, 5, 1, 5, 1, 1, 2.0, 0, None) == -1
    assert lib.kb200_rotation_matrix2d(p8, p8, p8, p8, 0, 0, 4, None) == -1
    assert lib.kb200_rotation_matrix2d(p8, None, p8, p8, 4, 0, 4, None) == -1
    assert lib.kb200_perspective_from_points(p8, p8, None, 4, 0, 4, None) == -1
    assert lib.kb200_perspective_from_points(p8, p8, p8, 4, 3, 4, None) == -1 and b"bad dtype" in lib.kb200_last_error()
    assert isinstance(lib.kb200_last_warp_launches(), int)


def test_c_abi_validation_of_the_wire_format_entry_points():
    """kb200_warp_u8hwc_forward / kb200_undistort_u8hwc_forward refuse bad requests on the host, before any CUDA call."""
    lib = _lib.load()
    p8 = ctypes.c_void_p(8)  # non-null dummy; never dereferenced on these paths
    warp = lib.kb200_warp_u8hwc_forward
    #            src m   bx  by  fill out B  C  H  W  h  w  Bm proj interp pad align normalize stream
    assert warp(None, p8, p8, p8, None, p8, 2, 3, 8, 8, 8, 8, 2, 1, 0, 0, 1, 1, None) == -1 and b"null pointer" in lib.kb200_last_error()
    assert warp(p8, p8, p8, p8, None, p8, 0, 3, 8, 8, 8, 8, 0, 1, 0, 0, 1, 1, None) == -1 and b"non-positive shape" in lib.kb200_last_error()
    assert warp(p8, p8, p8, p8, None, p8, 2, 3, 8, 8, 8, 8, 3, 1, 0, 0, 1, 1, None) == -1 and b"matrix batch" in lib.kb200_last_error()
    assert warp(p8, p8, p8, p8, None, p8, 2, 3, 8, 8, 8, 8, 2, 1, 0, 3, 1, 1, None) == -1 and b"fill vector" in lib.kb200_last_error()
    assert warp(p8, p8, p8, p8, None, p8, 2, 3, 8, 8, 8, 8, 2, 1, 0, 0, 1, 3, None) == -1 and b"normalize" in lib.kb200_last_error()
    assert warp(p8, p8, p8, p8, None, p8, 2, 3, 8, 8, 8, 8, 2, 1, 5, 0, 1, 1, None) == -1 and b"bad interp" in lib.kb200_last_error()
    assert warp(p8, p8, p8, p8, None, p8, 2, 3, 8, 8, 8, 8, 2, 1, 0, 7, 1, 1, None) == -1 and b"bad pad" in lib.kb200_last_error()
    und = lib.kb200_undistort_u8hwc_forward
    assert und(p8, None, p8, 2, 3, 8, 8, 1, None) == -1
    assert und(p8, p8, p8, 2, 3, 8, 8, 9, None) == -1 and b"normalize" in lib.kb200_last_error()
    assert und(p8, p8, p8, 2, 2, 8, 8, 1, None) == -3       # two channels: the host converts and takes the fp32 path
    assert und(p8, p8, p8, 2, 3, 8, 7, 1, None) == -3       # odd width
    assert und(ctypes.c_void_p(9), p8, p8, 2, 3, 8, 8, 1, None) == -3 and b"4-byte aligned" in lib.kb200_last_error()
