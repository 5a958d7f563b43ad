from .orientation import PatchDominantGradientOrientation
from .responses import BlobHessian, CornerGFTT, CornerHarris, gftt_response, harris_response, hessian_response
from .siftdesc import SIFTDescriptor, get_sift_bin_ksize_stride_pad, get_sift_pooling_kernel, sift_describe

__all__ = ["harris_response", "gftt_response", "hessian_response", "CornerHarris", "CornerGFTT", "BlobHessian", "SIFTDescriptor",
           "sift_describe", "get_sift_pooling_kernel", "get_sift_bin_ksize_stride_pad", "PatchDominantGradientOrientation"]
