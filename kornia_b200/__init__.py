"""kornia_b200 -- H100-native (sm_90a) drop-in for Kornia's warp / filter hot path.

    kornia.geometry.transform.{warp_perspective, warp_affine, remap}
    kornia.filters.{filter2d, filter2d_separable, gaussian_blur2d}

Same function names, signatures, defaults, validation and autograd behaviour; the image work runs
in hand-written CUDA kernels behind the C ABI of ``include/kornia_b200.h``.  CUDA-only: there is
no CPU path and no fallback -- a missing library or a CPU tensor raises.
"""
from __future__ import annotations

from . import augmentation, config, core, feature, filters, geometry, graphs, losses, metrics, streaming
from .filters import filter2d, filter2d_separable, gaussian_blur2d
from .geometry.transform import remap, warp_affine, warp_perspective

__version__ = "0.1.0"

_PATCHED = {}


def install(kornia_module=None) -> None:
    """Rebind the hot-path functions (and the four callers that have a fused kernel of their own here:
    ``get_perspective_transform``, ``spatial_gradient``, ``sobel``, ``ssim``, plus ``motion_blur`` and
    ``get_motion_kernel2d``, whose kernel must be built on the GPU, and the ``harris_response`` / ``gftt_response`` /
    ``hessian_response`` of the classical detectors, the ``ScalePyramid`` class their scale-space detectors build, and the
    non-maximum suppression ``nms2d`` / ``nms3d`` / ``nms3d_minmax`` / ``NonMaximaSuppression2d`` /
    ``NonMaximaSuppression3d`` of the detectors and the sub-pixel refiners, and those refiners ``conv_quad_interp3d`` /
    ``iterative_quad_interp3d`` / ``ConvQuadInterp3d`` / ``IterativeQuadInterp3d`` / ``AdaptiveQuadInterp3d``) on an
    imported ``kornia`` package.  A defining module the package lacks, or a name its module does not define, is skipped.
    The per-keypoint stages of the SIFT-style pipelines are rebound too: ``SIFTDescriptor`` / ``sift_describe`` and
    ``PatchDominantGradientOrientation``, which ``SIFTFeature``, ``SIFTFeatureScaleSpace`` and the ``LAFOrienter``
    constructor build by name, and the patch extraction ``extract_patches_from_pyramid`` / ``extract_patches_simple``
    that ``get_laf_descriptors`` / ``LAFDescriptor``, ``LAFOrienter`` and the affine shape estimators call by name (so
    those reach the fused extraction at call time, whenever they were built), and the affine shape estimators
    ``PatchAffineShapeEstimator`` / ``LAFAffineShapeEstimator`` (classes).  A ``LAFAffineShapeEstimator`` built after
    ``install()`` runs as one kernel per inference call; the reference's own ``LAFAffineShapeEstimator``, built before,
    still builds its default ``PatchAffineShapeEstimator`` by name, so one constructed after ``install()`` gets the fused
    patch estimator.  Rebinding a class affects modules constructed afterwards: a ``ScaleSpaceDetector``,
    ``MultiResolutionDetector``, ``SIFTFeature``, ``SIFTFeatureScaleSpace``, ``LAFOrienter`` or ``LAFAffineShapeEstimator``
    built before ``install()`` keeps the reference pyramid, ``NonMaximaSuppression2d``, sub-pixel refiner, descriptor,
    orienter and affine shape estimator it holds.

    Every module of the package that holds a reference to one of the originals is patched: the
    defining modules and re-export sites (geometry/transform/__init__.py:30, geometry/__init__.py:40,
    filters/__init__.py:37-38) and every ``from ... import warp_perspective``-style importer, so the
    callers either side of the path -- ``RandomPerspective`` / ``RandomAffine`` / ``RandomGaussianBlur``
    (augmentation/_2d/geometric/perspective.py:108, affine.py:154, _2d/intensity/gaussian_blur.py:108),
    ``affine`` / ``rotate`` / ``crop_by_transform_mat``, ``GaussianBlur2d``, ``unsharp_mask``, SSIM ... --
    run on the CUDA kernels without being rewritten.  ``uninstall()`` restores the originals."""
    import importlib
    import sys

    k = kornia_module or importlib.import_module("kornia")
    prefix = k.__name__ + "."
    defining = {
        "warp_perspective": ("geometry.transform.imgwarp", warp_perspective),
        "warp_affine": ("geometry.transform.imgwarp", warp_affine),
        "remap": ("geometry.transform.imgwarp", remap),
        "filter2d": ("filters.filter", filter2d),
        "filter2d_separable": ("filters.filter", filter2d_separable),
        "gaussian_blur2d": ("filters.gaussian", gaussian_blur2d),
        # callers with a kernel of their own here (the rest of the family reaches the kernels through the six above)
        "get_perspective_transform": ("geometry.transform.imgwarp", geometry.transform.get_perspective_transform),
        "spatial_gradient": ("filters.sobel", filters.spatial_gradient),
        "sobel": ("filters.sobel", filters.sobel),
        "ssim": ("metrics.ssim", metrics.ssim),
        # motion blur builds its kernel before filter2d sees the image, with rotate on the CPU for number arguments:
        # both halves are rebound so the reference's MotionBlur / RandomMotionBlur build it on the GPU
        "motion_blur": ("filters.motion", filters.motion_blur),
        "get_motion_kernel2d": ("filters.kernels_geometry", filters.get_motion_kernel2d),
        # the modules CornerHarris / CornerGFTT / BlobHessian (and so ScaleSpaceDetector) call these by their global names
        "harris_response": ("feature.responses", feature.harris_response),
        "gftt_response": ("feature.responses", feature.gftt_response),
        "hessian_response": ("feature.responses", feature.hessian_response),
        # a class: ScaleSpaceDetector (feature/scale_space_detector.py) and integrated.py build theirs from this name
        "ScalePyramid": ("geometry.transform.pyramid", geometry.transform.ScalePyramid),
        # ScaleSpaceDetector, MultiResolutionDetector, DISK, XFeat, ALIKED and the subpix refiners import these by name
        "nms2d": ("geometry.subpix.nms", geometry.subpix.nms2d),
        "nms3d": ("geometry.subpix.nms", geometry.subpix.nms3d),
        "nms3d_minmax": ("geometry.subpix.nms", geometry.subpix.nms3d_minmax),
        "NonMaximaSuppression2d": ("geometry.subpix.nms", geometry.subpix.NonMaximaSuppression2d),
        "NonMaximaSuppression3d": ("geometry.subpix.nms", geometry.subpix.NonMaximaSuppression3d),
        # ScaleSpaceDetector builds its default AdaptiveQuadInterp3d (and checks isinstance against all three classes, so
        # its precomputed NMS masks are still passed) and SIFTFeatureScaleSpace its ConvQuadInterp3d from these names
        "conv_quad_interp3d": ("geometry.subpix.spatial_soft_argmax", geometry.subpix.conv_quad_interp3d),
        "iterative_quad_interp3d": ("geometry.subpix.spatial_soft_argmax", geometry.subpix.iterative_quad_interp3d),
        "ConvQuadInterp3d": ("geometry.subpix.spatial_soft_argmax", geometry.subpix.ConvQuadInterp3d),
        "IterativeQuadInterp3d": ("geometry.subpix.spatial_soft_argmax", geometry.subpix.IterativeQuadInterp3d),
        "AdaptiveQuadInterp3d": ("geometry.subpix.spatial_soft_argmax", geometry.subpix.AdaptiveQuadInterp3d),
        # SIFTFeature / SIFTFeatureScaleSpace (integrated.py) build LAFDescriptor(SIFTDescriptor(41)) and the LAFOrienter
        # constructor its PatchDominantGradientOrientation from these names
        "SIFTDescriptor": ("feature.siftdesc", feature.SIFTDescriptor),
        "sift_describe": ("feature.siftdesc", feature.sift_describe),
        "PatchDominantGradientOrientation": ("feature.orientation", feature.PatchDominantGradientOrientation),
        # get_laf_descriptors / LAFDescriptor (integrated.py), LAFOrienter (orientation.py) and the affine shape estimators
        # (affine_shape.py) import these by name and call them at call time
        "extract_patches_from_pyramid": ("feature.laf", feature.extract_patches_from_pyramid),
        "extract_patches_simple": ("feature.laf", feature.extract_patches_simple),
        # classes: ScaleSpaceDetector(..., aff_module=LAFAffineShapeEstimator(...)) builds its estimator from this name, and
        # LAFAffineShapeEstimator builds its default PatchAffineShapeEstimator from that name at construction
        "PatchAffineShapeEstimator": ("feature.affine_shape", feature.PatchAffineShapeEstimator),
        "LAFAffineShapeEstimator": ("feature.affine_shape", feature.LAFAffineShapeEstimator),
    }
    originals = {}
    for name, (mod, fn) in defining.items():
        try:
            m = importlib.import_module(prefix + mod)
        except ModuleNotFoundError as e:  # a package without that module (an older kornia): nothing to rebind
            if e.name is not None and (prefix + mod).startswith(e.name):
                continue
            raise
        if (m, name) not in _PATCHED and not hasattr(m, name):  # a package whose module does not define it: nothing to rebind
            continue
        originals[name] = (_PATCHED.get((m, name), getattr(m, name)), fn)
    for modname, m in list(sys.modules.items()):
        if m is None or not (modname == k.__name__ or modname.startswith(prefix)):
            continue
        for name, (orig, fn) in originals.items():
            if m.__dict__.get(name) is orig:
                _PATCHED.setdefault((m, name), orig)
                setattr(m, name, fn)


def uninstall() -> None:
    for (m, name), orig in _PATCHED.items():
        setattr(m, name, orig)
    _PATCHED.clear()


__all__ = ["warp_perspective", "warp_affine", "remap", "filter2d", "filter2d_separable", "gaussian_blur2d", "install",
           "uninstall", "augmentation", "config", "core", "feature", "filters", "geometry", "graphs", "losses", "metrics", "streaming"]
