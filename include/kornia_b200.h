/*
 * kornia_b200 -- C ABI of the H100-native (sm_90a) warp / filter engine.
 *
 * The reference (kornia 0.9.0rc1) has no FFI: its boundary for this path is a set of Python
 * functions that bottom out in ATen calls.  Each entry point below replaces one such ATen
 * call site *together with* the elementwise Kornia code that feeds it, and is what a binding
 * (ctypes / cffi / pybind / a TORCH_LIBRARY shim) would bind.  Paths are relative to the
 * reference checkout.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name ends in _host;
 *   - tensors are dense row-major NCHW (images), (B,3,3) (matrices), (B,h,w) (maps);
 *   - `dtype` selects the element type of every floating buffer of the call (KB200_F32/F64);
 *   - `stream` is a cudaStream_t passed as void*; work is enqueued, never synchronised;
 *   - return value: 0 on success, a negative KB200_E* code otherwise; kb200_last_error()
 *     returns a thread-local message for the last failing call;
 *   - scratch is caller-provided (see *_workspace_bytes).  One exception: with the run-time work distribution on (option
 *     "dyn_sched", the default, for kb200_warp_forward / kb200_warp_backward) the first such launch on a device allocates a 128 KB
 *     ring of work counters (cudaMalloc, kept for the life of the process) and every launch zeroes one of them on `stream`
 *     (cudaMemsetAsync: legal inside a stream capture).  With the option 0 no call allocates.
 */
#ifndef KORNIA_B200_H
#define KORNIA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KB200_ABI_VERSION 1

enum { KB200_F32 = 0, KB200_F64 = 1 };
/* torch.nn.functional.grid_sample `mode` as forwarded by imgwarp.py:174,290,702 */
enum { KB200_BILINEAR = 0, KB200_NEAREST = 1, KB200_BICUBIC = 2 };
/* `padding_mode`; FILL is Kornia's own mode (imgwarp.py:172-173,293-320) */
enum { KB200_ZEROS = 0, KB200_BORDER = 1, KB200_REFLECTION = 2, KB200_FILL = 3 };
/* `border_type` of filter2d (filters/filter.py:26) */
enum { KB200_CONSTANT = 0, KB200_REFLECT = 1, KB200_REPLICATE = 2, KB200_CIRCULAR = 3 };

enum {
  KB200_OK = 0,
  KB200_EINVAL = -1,      /* bad argument (shape, enum, null pointer) */
  KB200_ECUDA = -2,       /* a CUDA runtime / driver call failed */
  KB200_EUNSUPPORTED = -3 /* valid request this build does not cover */
};

int kb200_abi_version(void);
const char* kb200_last_error(void);
/* Name of the device-code variant the last kb200_warp_forward call on this thread dispatched to
 * ("tma_tile" or "generic"); for tests and the bench. */
const char* kb200_last_warp_variant(void);
/* Kernels that call launched: 1, or 2 when the tiled path ran both tile shapes (64x32 tiles for near-identity
 * samples, 32x32 tiles for rotated / sheared ones; each kernel skips the other's samples). */
int kb200_last_warp_launches(void);
/* Kernel-selection switches: which of the library's own kernels serves a request.  Names: "tma", "tiled_filter",
 * "square_tiles", "tiled_gradient", "u8_tiled", "bwd_stride1", "dyn_sched"; values 0 = off, 1 = on.  The former switches
 * sweep, dyn_chunk and dyn_static are unknown names (kb200_set_option returns KB200_EINVAL; KB200_<NAME> is ignored).
 * Each is initialised ONCE when the library is loaded (environment KB200_<NAME>, else the built-in default); there is no
 * getenv on the call path.  The parity tests use the setter to run a tiled kernel against the kernel it stands in for.
 * kb200_set_option returns KB200_EINVAL for an unknown name; kb200_get_option returns the value (INT_MIN for an unknown name). */
int kb200_set_option(const char* name, int value);
int kb200_get_option(const char* name);

/* ------------------------------------------------------------------------------------------
 * Fused projective / affine warp, forward.
 * Replaces imgwarp.py:157-174 (warp_perspective: create_meshgrid + 15 elementwise kernels +
 * stack + F.grid_sample) and imgwarp.py:277-290 (warp_affine), including _fill_and_warp
 * (imgwarp.py:293-320) when pad == KB200_FILL.
 *   src   (B,C,H,W)
 *   m     (Bm,3,3)  src_norm <- dst_norm matrices (imgwarp.py:153,254); Bm == B, or 1 (shared)
 *   bx,by (w),(h)   base-grid axes in [-1,1] (grid.py:65-78 / imgwarp.py:271-276)
 *   fill  (C) or NULL; required iff pad == KB200_FILL
 *   out   (B,C,h,w)
 *   projective: 1 = divide by row 2 (imgwarp.py:167-169); 0 = affine rows only (:279-280)
 * ------------------------------------------------------------------------------------------ */
int kb200_warp_forward(const void* src, const void* m, const void* bx, const void* by, const void* fill,
                       void* out, int B, int C, int H, int W, int h, int w, int Bm, int projective,
                       int interp, int pad, int align_corners, int dtype, void* stream);

/* (B,3,3) prelude in one launch: m_out = inverse(N_dst @ (M3 @ inverse(N_src))) with N the pixel->[-1,1]
 * matrices of (H,W) and (h,w) (conversions.py:1717-1725,1753-1765; core/utils.py:159-166) and M3 = M for
 * rows == 3 or M padded with [0,0,1] for rows == 2 (conversions.py:342-345).  Bit-identical to the torch op
 * sequence on the same device for variant 0 (pinned by the GPU tests); not differentiable -- callers that
 * need d/dM keep the torch ops. */
int kb200_warp_prelude(const void* M, void* m_out, int B, int rows, int H, int W, int h, int w, int dtype,
                       int variant, void* stream);

/* Backward of kb200_warp_prelude: gM (B,rows,3) = dL/dM given m (B,3,3) = the prelude's output and gm = dL/dm. */
int kb200_warp_prelude_backward(const void* m, const void* gm, void* gM, int B, int rows, int H, int W, int h, int w,
                                int dtype, void* stream);

/* Backward of the above w.r.t. src and m (replaces grid_sampler_2d_backward + the autograd of
 * imgwarp.py:165-170; SURVEY.md appendix A.5).
 *   gout (B,C,h,w) upstream gradient
 *   gsrc (B,C,H,W) or NULL; MUST be zero-filled by the caller (scatter-add target)
 *   gm   (Bm,3,3)  or NULL; fully overwritten (deterministic two-stage reduction)
 *   workspace: kb200_warp_backward_workspace_bytes(...) bytes when gm != NULL, else may be NULL */
size_t kb200_warp_backward_workspace_bytes(int B, int h, int w, int dtype);
int kb200_warp_backward(const void* gout, const void* src, const void* m, const void* bx, const void* by,
                        const void* fill, void* gsrc, void* gm, void* workspace, int B, int C, int H, int W,
                        int h, int w, int Bm, int projective, int interp, int pad, int align_corners,
                        int dtype, void* stream);

/* ------------------------------------------------------------------------------------------
 * remap (imgwarp.py:681-702: stack + normalize_pixel_coordinates + expand + F.grid_sample).
 *   map_x,map_y (Bmap,h,w), Bmap == B or 1; pixel coordinates unless normalized != 0
 *   backward: gmap_x/gmap_y (B,h,w) per-sample (the caller sums over B when Bmap == 1), or NULL
 * ------------------------------------------------------------------------------------------ */
int kb200_remap_forward(const void* src, const void* map_x, const void* map_y, void* out, int B, int C, int H,
                        int W, int h, int w, int Bmap, int normalized, int interp, int pad, int align_corners,
                        int dtype, void* stream);
int kb200_remap_backward(const void* gout, const void* src, const void* map_x, const void* map_y, void* gsrc,
                         void* gmap_x, void* gmap_y, int B, int C, int H, int W, int h, int w, int Bmap,
                         int normalized, int interp, int pad, int align_corners, int dtype, void* stream);

/* undistort_image (geometry/calibration/undistort.py:183-198: create_meshgrid + distort_points -- ~45 elementwise
 * passes over (B,H*W) coordinates, calibration/distort.py:137-189 -- + remap(align_corners=True)) in ONE kernel: every
 * output pixel evaluates the lens model in registers (one IEEE rounding per reference op) and samples; the (B,H,W)
 * maps never exist.  lens (B,16) = fx, fy, cx, cy, k1, k2, p1, p2, k3, k4, k5, k6, s1, s2, s3, s4 (the tilt terms of
 * the 14-coefficient model must be zero); src and out (B,C,H,W).  fp32, C in {1,3}, W % 4 == 0: anything else returns
 * KB200_EUNSUPPORTED and the host builds the maps and calls kb200_remap_forward.  Forward only.
 * The Python layer calls it when KB200_FUSED_UNDISTORT=1 (the default). */
int kb200_undistort_forward(const void* src, const void* lens, void* out, int B, int C, int H, int W, int dtype, void* stream);

/* Warp straight from a decoder's interleaved uint8 output (SURVEY.md 8f row 4): image_to_tensor
 * (kornia/image/utils.py:27, HWC -> CHW) + _to_float32 (kornia/io/io.py:108-111, image.float() / 255.0) + warp_perspective /
 * warp_affine (imgwarp.py:69,177) in ONE kernel.  src (B,H,W,C) uint8; m / bx / by / fill fp32 as for kb200_warp_forward;
 * out (B,C,h,w) fp32.  normalize: 0 keeps float(byte); 1 multiplies by the fp32 reciprocal of 255, which is how torch's
 * CUDA backend evaluates `image.float() / 255.0` (so the result is bit-identical to the reference's three steps on this
 * device); 2 divides, as torch's CPU backend does (one ulp apart for 126 of the 256 byte values).  Forward only (a uint8 image has no gradient).
 * Bilinear (any of the four paddings), C in {1,3,4}, W % 4 == 0 and a 4-byte aligned src run the
 * shared-memory tiled kernel (warp_u8_tiled.cuh); everything else, or KB200_U8_SIMPLE=1, the per-tap kernel (warp_u8.cuh);
 * the two agree bit for bit. */
int kb200_warp_u8hwc_forward(const void* src_u8, const void* m, const void* bx, const void* by, const void* fill, void* out,
                             int B, int C, int H, int W, int h, int w, int Bm, int projective, int interp, int pad,
                             int align_corners, int normalize, void* stream);

/* undistort_image (calibration/undistort.py:183-198) straight from decoder bytes: image_to_tensor + _to_float32 +
 * create_meshgrid + distort_points + remap(align_corners=True) in ONE kernel -- the lens model of kb200_undistort_forward
 * (same (B,16) lens layout, tilt terms must be zero) on the byte loader of kb200_warp_u8hwc_forward (same `normalize`).
 * src (B,H,W,C) uint8 -> out (B,C,H,W) fp32.  C in {1,3}, W % 4 == 0, 4-byte aligned src; anything else returns
 * KB200_EUNSUPPORTED and the host converts the image and calls the fp32 path.  Forward only.  Equals
 * kb200_undistort_forward on the converted image bit for bit.  Status: emulator-verified, not yet run on hardware. */
int kb200_undistort_u8hwc_forward(const void* src_u8, const void* lens, void* out, int B, int C, int H, int W, int normalize,
                                  void* stream);

/* ------------------------------------------------------------------------------------------
 * filter2d core (filters/filter.py:136-150: F.pad + view + depthwise F.conv2d + view).
 *   x      (B,C,H,W)
 *   kernel (Bk,kh,kw) correlation taps, already flipped / normalised by the host
 *          (filter.py:123-129); plane (b,c) uses kernel b mod Bk (filter.py:131,141-142)
 *   same   1: 'same' (border-padded, out (B,C,H,W)); 0: 'valid' (out (B,C,H-kh+1,W-kw+1))
 * Backward: gx = adjoint of pad+correlate applied to gout; gkernel (Bk,kh,kw) fully overwritten.
 * ------------------------------------------------------------------------------------------ */
int kb200_filter2d_forward(const void* x, const void* kernel, void* out, int B, int C, int H, int W, int Bk,
                           int kh, int kw, int border, int same, int dtype, void* stream);
int kb200_filter2d_backward_input(const void* gout, const void* kernel, void* gx, int B, int C, int H, int W,
                                  int Bk, int kh, int kw, int border, int same, int dtype, void* stream);
size_t kb200_filter2d_backward_kernel_workspace_bytes(int B, int C, int H, int W, int Bk, int kh, int kw, int dtype);
int kb200_filter2d_backward_kernel(const void* gout, const void* x, void* gkernel, void* workspace, int B,
                                   int C, int H, int W, int Bk, int kh, int kw, int border, int same,
                                   int dtype, void* stream);

/* filter2d_separable (filter.py:205-207) in ONE pass over HBM: row pass (1 x kw, kernel_x) then
 * column pass (kh x 1, kernel_y) out of a shared-memory tile.  kernel_x (Bkx,kw), kernel_y (Bky,kh). */
int kb200_sepfilter_forward(const void* x, const void* kernel_x, const void* kernel_y, void* out, int B, int C,
                            int H, int W, int Bkx, int kw, int Bky, int kh, int border, int same, int dtype,
                            void* stream);

/* unsharp_mask (filters/unsharp.py:53-54): out = lerp(filter2d_separable(x), x, weight), the blend done in the epilogue
 * of the one-pass separable kernel instead of a separate pass over three full-size tensors.  Same arguments as
 * kb200_sepfilter_forward plus `weight` (torch.lerp semantics).  fp32, square odd kernels up to 11 taps,
 * constant / reflect / replicate, 'same': anything else returns KB200_EUNSUPPORTED (the host then blends with torch). */
int kb200_sepfilter_lerp_forward(const void* x, const void* kernel_x, const void* kernel_y, void* out, int B, int C, int H,
                                 int W, int Bkx, int kw, int Bky, int kh, int border, int same, double weight, int dtype,
                                 void* stream);

/* pyrdown (geometry/transform/pyramid.py:444-457: filter2d with the 5x5 pyramid taps, then F.interpolate(bilinear,
 * align_corners=False) onto exactly half the size) in ONE pass: the 2x2 average that the resampling reduces to at a
 * factor of two is the epilogue of the tiled 5x5 kernel, so the blurred full-size image never reaches HBM (4 B read +
 * 1 B written per input element instead of 8 + 5).  x (B,C,H,W), kernel (Bk,5,5) as in kb200_filter2d_forward,
 * out (B,C,H/2,W/2).  fp32, H even, W % 4 == 0, constant / reflect / replicate: anything else returns
 * KB200_EUNSUPPORTED and the host composes kb200_filter2d_forward with the resampling.
 * The Python layer calls it when KB200_FUSED_PYRDOWN=1 (the default). */
int kb200_pyrdown_forward(const void* x, const void* kernel, void* out, int B, int C, int H, int W, int Bk, int border,
                          int dtype, void* stream);

/* get_perspective_transform (geometry/transform/imgwarp.py:444-462: two unit-square-to-quad maps, a closed-form
 * 3x3 inverse, one bmm and a scale -- ~45 tiny torch launches) in one launch, for the RandomPerspective /
 * crop_and_resize callers (SURVEY.md 8f row 1).  points_src, points_dst: (B,4,2) x,y corners; H_out: (B,3,3)
 * with H[2,2] = 1.  `variant` as in kb200_warp_prelude.  No gradient: the host keeps the torch ops for that. */
int kb200_perspective_from_points(const void* points_src, const void* points_dst, void* H_out, int B, int dtype,
                                  int variant, void* stream);

/* get_rotation_matrix2d (geometry/transform/imgwarp.py:529-622: four eye_like, index assignments, deg2rad, cos, sin,
 * stack and three bmm -- ~35 tiny torch launches) in one launch, for rotate / scale / RandomAffine (SURVEY.md 8f rows
 * 1-2).  center (B,2) x,y; angle (B,) degrees; scale (B,2); M_out (B,2,3) = T(c) R S T(-c).  No gradient. */
int kb200_rotation_matrix2d(const void* center, const void* angle, const void* scale, void* M_out, int B, int dtype,
                            int variant, void* stream);

/* ------------------------------------------------------------------------------------------
 * Image derivatives (SURVEY.md 8f row 3): spatial_gradient / sobel (filters/sobel.py:32-74,134-167:
 * F.pad(replicate) + F.conv2d with a (nout,1,k,k) weight, then for sobel two slices + 5 elementwise
 * passes).  One kernel: the replicate border is a clamp on the tap index, all nout derivatives of a
 * pixel come out of one register window.
 *   x     (planes,H,W) device, planes = B*C
 *   taps  HOST pointer to nout*k*k doubles, [nout][k][k] correlation taps holding values exactly
 *         representable in `dtype` (the host builds and normalises them in that dtype:
 *         filters/kernels.py:504-528, :68-74); k in {3,5}, nout in {2,3}
 *   out   (planes,nout,H,W); with magnitude=1 (nout=2, k=3): (planes,H,W) = sqrt(gx*gx + gy*gy + eps)
 * Backward: gx (planes,H,W) = adjoint of (replicate pad, nout correlations) applied to
 * gout (planes,nout,H,W); deterministic gather.
 * ------------------------------------------------------------------------------------------ */
int kb200_spatial_gradient_forward(const void* x, const double* taps, void* out, int planes, int H, int W, int nout,
                                   int k, int magnitude, double eps, int dtype, void* stream);
int kb200_spatial_gradient_backward(const void* gout, const double* taps, void* gx, int planes, int H, int W,
                                    int nout, int k, int dtype, void* stream);

/* ------------------------------------------------------------------------------------------
 * SSIM index map (metrics/ssim.py:92-139: five filter2d_separable calls with a Gaussian window of sigma 1.5,
 * three product kernels and fourteen elementwise kernels) in ONE kernel: 8 B read + 4 B written per element.
 *   img1, img2 (planes,H,W) device; taps (K,) device Gaussian window (the same for rows and columns);
 *   out (planes,H,W) = ((2 mu1 mu2 + C1)(2 s12 + C2)) / ((mu1^2 + mu2^2 + C1)(s1 + s2 + C2) + eps),
 *   'reflect' border, 'same' size (the 'valid' variant is a crop of it).
 * fp32 and odd K <= 11 only: anything else returns KB200_EUNSUPPORTED and the host composes the map from
 * kb200_sepfilter_forward (which is also the differentiable path).
 * ------------------------------------------------------------------------------------------ */
int kb200_ssim_forward(const void* img1, const void* img2, const void* taps, void* out, int planes, int H, int W, int K,
                       double C1, double C2, double eps, int dtype, void* stream);

/* ------------------------------------------------------------------------------------------
 * Feature responses (feature/responses.py:39-282) in ONE kernel each: 4 B read + 4 B written per element.
 *   x        (planes,H,W) device, planes = B*C
 *   stencil  HOST pointer to nout*ks*ks doubles exact in fp32: (dx, dy) 3x3 for Harris / GFTT, (dxx, dxy, dyy) ks x ks
 *            for the Hessian (the taps of spatial_gradient, replicate border)
 *   blur_taps (blur_k,) device Gaussian taps of the structure-tensor blur (reflect border; Harris / GFTT only, else ignored)
 *   k        Harris k, rounded to fp32; k_ptr (device fp32) overrides it when not null
 *   s4       (planes / C,) device fp32 sigmas^4 multiplying each sample's response, or null
 *   out      (planes,H,W): kind 0 Harris det(M) - k tr(M)^2, kind 1 GFTT min(eig(M)), kind 2 Hessian dxx dyy - dxy^2
 * One rounding per reference op: bit-identical to the reference's composition over kb200_spatial_gradient_forward and
 * kb200_sepfilter_forward.  fp32 with W % 4 == 0, 3x3 stencils and blur_k = 7 (Harris, GFTT) or 3x3 / 5x5 stencils
 * (Hessian) only: anything else returns KB200_EUNSUPPORTED and the host composes the response.  Forward only.
 * ------------------------------------------------------------------------------------------ */
int kb200_feature_response_forward(const void* x, const double* stencil, const void* blur_taps, double k, const void* k_ptr,
                                   const void* s4, void* out, int planes, int C, int H, int W, int stencil_k, int blur_k,
                                   int kind, int dtype, void* stream);

/* ------------------------------------------------------------------------------------------
 * One octave of ScalePyramid (geometry/transform/pyramid.py:367-384: a reflect-bordered separable Gaussian per level,
 * each of the level before it, then torch.stack) in ONE kernel: 4 B read + 4 B written per element and level.
 *   x       (planes,H,W) device, the octave's seed (the input, its 2x upsample, or the bilinear octave seed)
 *   taps    HOST pointer to the taps of ksizes[0], ksizes[1], ... in that order, doubles exact in fp32
 *   ksizes  HOST pointer to L tap counts: ksizes[0] the initial blur of level 0 (0: level 0 is x itself), ksizes[l] the
 *           blur from level l-1 to level l
 *   out     (planes,L,H,W): every level of the octave
 * Each level is a row pass, then a column pass, with ascending taps, one FMA per tap from 0 and the reflect border of
 * the level it filters: bit-identical to L - 1 (or L) calls of kb200_sepfilter_forward.  fp32 with W % 4 == 0,
 * 16-byte aligned buffers, every tap count <= min(H, W), and one of the chains 13 | 11 13 17 21 25, 13 | 11 13 17 21,
 * 11 | 11 13 17 21 25, 0 | 11 13 17 21 25, 0 | 11 13 17 21 only: anything else returns KB200_EUNSUPPORTED and the
 * host composes the octave.  Forward only.
 * ------------------------------------------------------------------------------------------ */
int kb200_scale_octave_forward(const void* x, const double* taps, const int* ksizes, int L, void* out, int planes, int H, int W,
                               int dtype, void* stream);

/* ------------------------------------------------------------------------------------------
 * Non-maximum suppression (geometry/subpix/nms.py) in ONE kernel per call: 4 B read and 1 B (mask) or 4 B (values)
 * written per element, instead of one ATen kernel per neighbour comparison.
 *   x     fp32 source whose H x W planes are dense; sB, sC (and sL) are the element strides of b, c (and the level), so a
 *         permuted (B, C, L, H, W) view is read in place
 *   out   contiguous (B, C, H, W) / (B, C, L, H, W): uint8 0/1 masks, or fp32 x * mask (values = 1, mode = 1)
 * kb200_nms2d_forward: NonMaximaSuppression2d((k, k)) for odd k = 3..31; k = 3, 5, 7 compare with the k*k - 1 neighbours
 * and leave the (k - 1) / 2 border False, k >= 9 follows the reference's one-hot F.conv2d of the replicate-padded
 * image (0 joins the neighbour set; a window holding a non-finite texel is False).  Anything else returns
 * KB200_EUNSUPPORTED and the host composes the reference's op sequence.
 * kb200_nms3d_forward: NonMaximaSuppression3d((3, 3, 3)); mode 0 the maxima mask, 1 the maxima values, 2 nms3d_minmax's
 * maxima (out0) and minima (out1) masks.  Border levels, rows and columns are False.  Forward only.
 * ------------------------------------------------------------------------------------------ */
int kb200_nms2d_forward(const void* x, void* out, int B, int C, int H, int W, long long sB, long long sC, int k, int values, int dtype,
                        void* stream);
int kb200_nms3d_forward(const void* x, void* out0, void* out1, int B, int C, int L, int H, int W, long long sB, long long sC,
                        long long sL, int mode, int dtype, void* stream);

/* ------------------------------------------------------------------------------------------
 * Sub-pixel refinement of 3-D scale-space maxima (conv_quad_interp3d / iterative_quad_interp3d of
 * geometry/subpix/spatial_soft_argmax.py) in ONE kernel per call: 4 B read (5 B with a mask) and 16 B written per element,
 * with no host synchronisation, instead of a nonzero, index gathers and tens of small kernels per iteration.
 *   x       fp32 (B, C, L, H, W) whose H x W planes are dense; sB, sC, sL are its element strides, so a permuted
 *           (B, C, L, H, W) view is read in place
 *   mask    contiguous bool (B, C, L, H, W) NMS mask, or NULL: nms3d(x, (3, 3, 3), True) is computed in the kernel
 *   coords  contiguous (B, C, 3, L, H, W) [level, x, y]: the grid, refined at the maxima
 *   y       (B, C, L, H, W) at the element strides ysB .. ysW (those of x.clone()): x, refined at the maxima
 *   radius  the conv form's dilation radius (>= 1), or 0 for the iterative form
 *   max_shift, bonus  the Python floats rounded to fp32; add_bonus = (strict_maxima_bonus > 0)
 * L, H or W < 3 writes the grid and the copy only, as the reference returns them.  Forward only.
 * ------------------------------------------------------------------------------------------ */
int kb200_quad_interp3d_forward(const void* x, const void* mask, void* coords, void* y, int B, int C, int L, int H, int W, long long sB,
                                long long sC, long long sL, long long ysB, long long ysC, long long ysL, long long ysH,
                                long long ysW, int n_iters, int radius, float max_shift, float bonus, int add_bonus, int allow_scale,
                                int dtype, void* stream);

/* ------------------------------------------------------------------------------------------
 * Per-patch gradient histograms (feature/siftdesc.py SIFTDescriptor, feature/orientation.py
 * PatchDominantGradientOrientation) in ONE kernel per call: each patch is read once and D or 1 floats are written, instead
 * of about 100 (SIFT) or 290 (orientation) ATen kernels over the whole patch stack.
 *   x        fp32 (N, 1, P, P) patches with column stride 1; sB, sH are the batch and row element strides
 *   gk       contiguous fp32 P x P weighting (SIFT: the module's gk; orientation: its weighting)
 *   pk       contiguous fp32 K x K pooling weights (pk.weight); smooth: the 5 taps of angular_smooth.weight
 *   out      contiguous fp32 (N, A * S * S) descriptors or (N,) angles
 * Envelope: P <= 64, ksize <= 64 and A * S * S <= 1024 (SIFT), P <= 64 and 2 <= A <= 64 (orientation); KB200_EUNSUPPORTED outside it.
 * Each patch's result depends on that patch only (fixed-order sums, no atomics).  N = 0 launches nothing.  Forward only.
 * ------------------------------------------------------------------------------------------ */
int kb200_sift_describe_forward(const void* x, const void* gk, const void* pk, void* out, long long N, int P, long long sB, long long sH,
                                int num_ang_bins, int num_spatial_bins, int ksize, int stride, int pad, int rootsift, float clipval,
                                float eps, int dtype, void* stream);
int kb200_patch_orientation_forward(const void* x, const void* weighting, const void* smooth, void* out, long long N, int P, long long sB,
                                    long long sH, int num_ang_bins, float eps, int dtype, void* stream);

/* ------------------------------------------------------------------------------------------
 * LAF patch extraction (feature/laf.py extract_patches_from_pyramid / extract_patches_simple) in ONE kernel per call:
 * each patch picks its pyramid level, maps its PS x PS grid and samples every channel bilinearly with 'border' padding,
 * writing B * N * C * PS * PS floats once, instead of about 25 ATen kernels per (level, image) over all N patches.
 *   levels      n_levels pointers to fp32 (B_l, C, h_l, w_l) levels with column stride 1 (level 0 the image, then pyrdowns)
 *   level_dims  5 per level: h, w and the batch, channel and row element strides
 *   laf         contiguous fp32 (B, N, 2, 3); B <= every level's batch
 *   base        contiguous fp32 PS base-grid coordinates (affine_grid, align_corners=False)
 *   out         contiguous fp32 (B, N, C, PS, PS)
 * select_level = 0 samples level 0 only (extract_patches_simple).  A patch whose level is not among the n_levels given
 * (1 <= n_levels <= 32) is written as zeros.  Each output element is written once and depends on its patch only.
 * B * N = 0 launches nothing.  Forward only.
 * ------------------------------------------------------------------------------------------ */
int kb200_extract_patches_forward(const void* const* levels, const long long* level_dims, int n_levels, const void* laf, const void* base,
                                  void* out, long long B, long long N, int C, int PS, int normalize, int select_level, int dtype,
                                  void* stream);

/* ------------------------------------------------------------------------------------------
 * Affine shape (feature/affine_shape.py) in ONE kernel per call, one CTA per keypoint: the Baumberg second-moment matrix of
 * the weighted Sobel gradients, summed in fp64, with the reference's degenerate-shape test and max normalisation.
 * kb200_patch_affine_shape_forward (PatchAffineShapeEstimator):
 *   x          fp32 (N, 1, P, P) patches with column stride 1 (batch and row element strides sB, sH); P <= 64
 *   weighting  contiguous fp32 P x P
 *   out        contiguous fp32 (N, 3): (a, b, c) / max(a, b, c)
 * kb200_laf_affine_shape_forward (LAFAffineShapeEstimator with its default PatchAffineShapeEstimator):
 *   levels, level_dims, n_levels, base   as for kb200_extract_patches_forward: the levels of (B_l, 1, h_l, w_l) images
 *   laf        contiguous fp32 (B, N, 2, 3); B <= every level's batch
 *   weighting  contiguous fp32 PS x PS; PS <= 64
 *   out        contiguous fp32 (B, N, 2, 3): make_upright, the patch sampled at its level straight into shared memory
 *              (no patch stack), the moments, ellipse_to_laf (closed-form inverse), the rescale to the input's scale and,
 *              with preserve_orientation, the input's orientation; the centre copied.
 * N = 0 (B * N = 0) launches nothing.  Forward only.
 * ------------------------------------------------------------------------------------------ */
int kb200_patch_affine_shape_forward(const void* x, const void* weighting, void* out, long long N, int P, long long sB, long long sH, float eps,
                                     int dtype, void* stream);
int kb200_laf_affine_shape_forward(const void* const* levels, const long long* level_dims, int n_levels, const void* laf, const void* base,
                                   const void* weighting, void* out, long long B, long long N, int PS, float eps, int preserve_orientation,
                                   int dtype, void* stream);

/* ------------------------------------------------------------------------------------------
 * Diagnostics (used by tests/): counts elements where the shared-reciprocal division of the tiled
 * warp kernel differs from IEEE division in a way that could change a sampled pixel.  `count`
 * (device int, zeroed by the caller) is incremented atomically.
 * ------------------------------------------------------------------------------------------ */
int kb200_debug_fastdiv_mismatches(const float* num, const float* den, int n, int* count, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* KORNIA_B200_H */
