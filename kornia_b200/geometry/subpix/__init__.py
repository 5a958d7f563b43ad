from .nms import NonMaximaSuppression2d, NonMaximaSuppression3d, nms2d, nms3d, nms3d_minmax
from .quad_interp import AdaptiveQuadInterp3d, ConvQuadInterp3d, IterativeQuadInterp3d, conv_quad_interp3d, iterative_quad_interp3d

__all__ = ["nms2d", "nms3d", "nms3d_minmax", "NonMaximaSuppression2d", "NonMaximaSuppression3d", "conv_quad_interp3d",
           "iterative_quad_interp3d", "ConvQuadInterp3d", "IterativeQuadInterp3d", "AdaptiveQuadInterp3d"]
