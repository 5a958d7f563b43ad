from . import calibration, subpix, transform
from .calibration import distort_points, undistort_image
from .subpix import (
    AdaptiveQuadInterp3d,
    ConvQuadInterp3d,
    IterativeQuadInterp3d,
    NonMaximaSuppression2d,
    NonMaximaSuppression3d,
    conv_quad_interp3d,
    iterative_quad_interp3d,
    nms2d,
    nms3d,
    nms3d_minmax,
)
from .transform import (
    affine,
    build_laplacian_pyramid,
    build_pyramid,
    center_crop,
    crop_and_resize,
    crop_by_boxes,
    crop_by_transform_mat,
    get_perspective_transform,
    get_rotation_matrix2d,
    pyrdown,
    pyrup,
    ScalePyramid,
    remap,
    rescale,
    resize,
    rotate,
    scale,
    shear,
    translate,
    warp_affine,
    warp_perspective,
)

__all__ = ["transform", "calibration", "subpix", "nms2d", "nms3d", "nms3d_minmax", "NonMaximaSuppression2d", "NonMaximaSuppression3d",
           "conv_quad_interp3d", "iterative_quad_interp3d", "ConvQuadInterp3d", "IterativeQuadInterp3d", "AdaptiveQuadInterp3d", "undistort_image", "distort_points", "pyrdown", "pyrup", "build_pyramid",
           "build_laplacian_pyramid", "ScalePyramid", "resize", "rescale", "remap", "warp_affine", "warp_perspective", "affine", "rotate", "translate", "scale", "shear",
           "crop_and_resize", "center_crop", "crop_by_boxes", "crop_by_transform_mat", "get_perspective_transform",
           "get_rotation_matrix2d"]
