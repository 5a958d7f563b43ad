from .blur import BoxBlur, box_blur
from .filter import filter2d, filter2d_separable
from .gaussian import GaussianBlur2d, gaussian_blur2d
from .kernels import (
    gaussian,
    get_box_kernel1d,
    get_box_kernel2d,
    get_diff_kernel2d,
    get_gaussian_discrete_kernel1d,
    get_gaussian_kernel1d,
    get_gaussian_kernel2d,
    get_laplacian_kernel1d,
    get_laplacian_kernel2d,
    get_sobel_kernel2d,
    get_spatial_gradient_kernel2d,
    laplacian_1d,
    normalize_kernel2d,
)
from .laplacian import Laplacian, laplacian
from .sobel import Sobel, SpatialGradient, sobel, spatial_gradient
from .unsharp import UnsharpMask, unsharp_mask
from .motion import MotionBlur, get_motion_kernel2d, motion_blur  # last: it imports geometry.transform, which imports filters

__all__ = ["filter2d", "filter2d_separable", "gaussian_blur2d", "GaussianBlur2d", "box_blur", "BoxBlur", "laplacian",
           "Laplacian", "spatial_gradient", "sobel", "SpatialGradient", "Sobel", "unsharp_mask", "UnsharpMask",
           "motion_blur", "MotionBlur", "get_motion_kernel2d", "gaussian",
           "get_gaussian_kernel1d", "get_gaussian_kernel2d", "get_gaussian_discrete_kernel1d", "get_box_kernel1d", "get_box_kernel2d", "laplacian_1d",
           "get_laplacian_kernel1d", "get_laplacian_kernel2d", "get_sobel_kernel2d", "get_diff_kernel2d",
           "get_spatial_gradient_kernel2d", "normalize_kernel2d"]
