from .affwarp import Rescale, Resize, affine, rescale, resize, resize_to_be_divisible, rotate, scale, shear, translate
from .crop2d import center_crop, crop_and_resize, crop_by_boxes, crop_by_transform_mat
from .imgwarp import remap, warp_affine, warp_perspective
from .ingest import warp_affine_from_uint8, warp_perspective_from_uint8
from .pyramid import PyrDown, PyrUp, ScalePyramid, build_laplacian_pyramid, build_pyramid, pyrdown, pyrup
from .matrices import angle_to_rotation_matrix, deg2rad, get_perspective_transform, get_rotation_matrix2d

__all__ = ["remap", "warp_affine", "warp_perspective", "affine", "rotate", "translate", "scale", "shear", "crop_and_resize",
           "center_crop", "crop_by_boxes", "crop_by_transform_mat", "get_perspective_transform", "get_rotation_matrix2d",
           "angle_to_rotation_matrix", "deg2rad", "resize", "rescale", "resize_to_be_divisible", "Resize", "Rescale", "pyrdown", "pyrup",
           "build_pyramid", "build_laplacian_pyramid", "PyrDown", "PyrUp", "ScalePyramid", "warp_perspective_from_uint8", "warp_affine_from_uint8"]
