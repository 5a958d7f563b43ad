from .affine_shape import LAFAffineShapeEstimator, PatchAffineShapeEstimator
from .laf import (denormalize_laf, ellipse_to_laf, extract_patches_from_pyramid, extract_patches_simple, generate_patch_grid_from_normalized_LAF,
                  get_laf_orientation, get_laf_scale, make_upright, normalize_laf, rotate_laf, scale_laf, set_laf_orientation)
from .orientation import PatchDominantGradientOrientation
from .responses import BlobHessian, CornerGFTT, CornerHarris, gftt_response, harris_response, hessian_response
from .siftdesc import SIFTDescriptor, get_sift_bin_ksize_stride_pad, get_sift_pooling_kernel, sift_describe

__all__ = ["harris_response", "gftt_response", "hessian_response", "CornerHarris", "CornerGFTT", "BlobHessian", "SIFTDescriptor",
           "sift_describe", "get_sift_pooling_kernel", "get_sift_bin_ksize_stride_pad", "PatchDominantGradientOrientation",
           "extract_patches_from_pyramid", "extract_patches_simple", "get_laf_scale", "normalize_laf", "denormalize_laf",
           "generate_patch_grid_from_normalized_LAF", "make_upright", "scale_laf", "ellipse_to_laf", "get_laf_orientation",
           "set_laf_orientation", "rotate_laf", "PatchAffineShapeEstimator", "LAFAffineShapeEstimator"]
