from .laf import (denormalize_laf, extract_patches_from_pyramid, extract_patches_simple, generate_patch_grid_from_normalized_LAF,
                  get_laf_scale, normalize_laf)
from .orientation import PatchDominantGradientOrientation
from .responses import BlobHessian, CornerGFTT, CornerHarris, gftt_response, harris_response, hessian_response
from .siftdesc import SIFTDescriptor, get_sift_bin_ksize_stride_pad, get_sift_pooling_kernel, sift_describe

__all__ = ["harris_response", "gftt_response", "hessian_response", "CornerHarris", "CornerGFTT", "BlobHessian", "SIFTDescriptor",
           "sift_describe", "get_sift_pooling_kernel", "get_sift_bin_ksize_stride_pad", "PatchDominantGradientOrientation",
           "extract_patches_from_pyramid", "extract_patches_simple", "get_laf_scale", "normalize_laf", "denormalize_laf",
           "generate_patch_grid_from_normalized_LAF"]
