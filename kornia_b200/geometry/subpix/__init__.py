from .nms import NonMaximaSuppression2d, NonMaximaSuppression3d, nms2d, nms3d, nms3d_minmax

__all__ = ["nms2d", "nms3d", "nms3d_minmax", "NonMaximaSuppression2d", "NonMaximaSuppression3d"]
