from .responses import BlobHessian, CornerGFTT, CornerHarris, gftt_response, harris_response, hessian_response

__all__ = ["harris_response", "gftt_response", "hessian_response", "CornerHarris", "CornerGFTT", "BlobHessian"]
