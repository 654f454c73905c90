/*
  magick_b200.h -- C-ABI of libmagickb200.so: ImageMagick's per-pixel hot path
  (separable / 2-D convolution, erode/dilate morphology, filtered resize,
  sRGB<->Lab/XYZ/linear colourspace) as hand-written sm_90a CUDA kernels.

  Plain pointers and sizes only.  No torch / CUDA types in the signatures (a
  CUDA stream is passed as void*).  Pixel buffers are the reference's own pixel
  cache layout for its default Q16-HDRI build (MagickCore/cache.c:5142,
  MagickCore/pixel.c:6158): tightly packed, row-major, channel-interleaved
  float32 Quantum, values 0..65535, `channels` floats per pixel:

      channels 1 = Gray, 2 = Gray+Alpha, 3 = RGB, 4 = RGBA (alpha last).

  Images with alpha give their colour channels the Blend trait exactly like
  MagickCore/pixel.c:6356-6381 (alpha-weighted convolution / resize).

  Every entry point names the reference interface it replaces.  Return value:
  0 (MB200_OK) on success, a negative MB200_E* code otherwise; the message is
  available from mb200_last_error() (thread-local).  There is NO CPU fallback:
  when no sm_90 device is usable the calls fail with MB200_ENODEVICE -- the
  MagickCore shim (imagemagick_b200/shim) then returns NULL so that the caller's
  stock CPU path runs, which is the accelerate hook contract of
  MagickCore/effect.c:783-787 and MagickCore/resize.c:3818-3826.
*/
#ifndef MAGICK_B200_H
#define MAGICK_B200_H

#include <stddef.h>

#if defined(__cplusplus)
extern "C" {
#endif

#if defined(_WIN32)
# define MB200_API
#else
# define MB200_API __attribute__((visibility("default")))
#endif

enum {
  MB200_OK = 0,
  MB200_EINVAL = -1,        /* bad argument */
  MB200_ENODEVICE = -2,     /* no usable CUDA device / wrong architecture */
  MB200_ECUDA = -3,         /* CUDA runtime error (see mb200_last_error) */
  MB200_ENOMEM = -4,
  MB200_EUNSUPPORTED = -5   /* valid in the reference but not implemented here:
                               the shim must fall back to the CPU path */
};

/* MagickCore/morphology.h:69-99 MorphologyMethod -- same numeric values */
typedef enum {
  MB200_UndefinedMorphology = 0,
  MB200_ConvolveMorphology = 1,
  MB200_CorrelateMorphology = 2,
  MB200_ErodeMorphology = 3,
  MB200_DilateMorphology = 4,
  MB200_ErodeIntensityMorphology = 5,
  MB200_DilateIntensityMorphology = 6,
  MB200_IterativeDistanceMorphology = 7,
  MB200_OpenMorphology = 8,
  MB200_CloseMorphology = 9,
  MB200_OpenIntensityMorphology = 10,
  MB200_CloseIntensityMorphology = 11,
  MB200_SmoothMorphology = 12,
  MB200_EdgeInMorphology = 13,
  MB200_EdgeOutMorphology = 14,
  MB200_EdgeMorphology = 15,
  MB200_TopHatMorphology = 16,
  MB200_BottomHatMorphology = 17,
  MB200_HitAndMissMorphology = 18,
  MB200_ThinningMorphology = 19,
  MB200_ThickenMorphology = 20,
  MB200_DistanceMorphology = 21,
  MB200_VoronoiMorphology = 22
} mb200_morphology_method;

/* MagickCore/resample.h:32-69 FilterType -- same numeric values */
typedef enum {
  MB200_UndefinedFilter = 0, MB200_PointFilter, MB200_BoxFilter, MB200_TriangleFilter,
  MB200_HermiteFilter, MB200_HannFilter, MB200_HammingFilter, MB200_BlackmanFilter,
  MB200_GaussianFilter, MB200_QuadraticFilter, MB200_CubicFilter, MB200_CatromFilter,
  MB200_MitchellFilter, MB200_JincFilter, MB200_SincFilter, MB200_SincFastFilter,
  MB200_KaiserFilter, MB200_WelchFilter, MB200_ParzenFilter, MB200_BohmanFilter,
  MB200_BartlettFilter, MB200_LagrangeFilter, MB200_LanczosFilter, MB200_LanczosSharpFilter,
  MB200_Lanczos2Filter, MB200_Lanczos2SharpFilter, MB200_RobidouxFilter,
  MB200_RobidouxSharpFilter, MB200_CosineFilter, MB200_SplineFilter,
  MB200_LanczosRadiusFilter, MB200_CubicSplineFilter, MB200_MagicKernelSharp2013Filter,
  MB200_MagicKernelSharp2021Filter, MB200_SentinelFilter
} mb200_filter_type;

/* MagickCore/colorspace.h:27-67 ColorspaceType -- same numeric values */
typedef enum {
  MB200_CMYColorspace = 1,
  MB200_CMYKColorspace = 2,           /* layout-changing: mb200_transform_colorspace_layout only */
  MB200_GRAYColorspace = 3,           /* layout-changing: mb200_transform_colorspace_layout only */
  MB200_HCLColorspace = 4,           /* hue / saturation family of the generic branch (colorspace-private.h:149-529, */
  MB200_HCLpColorspace = 5,           /* :801-1064): bit exact, HSI <= 1 ULP                                        */
  MB200_HSBColorspace = 6,
  MB200_HSIColorspace = 7,
  MB200_HSLColorspace = 8,
  MB200_HSVColorspace = 9,
  MB200_HWBColorspace = 10,
  MB200_LabColorspace = 11,
  MB200_LCHColorspace = 12,           /* polar Lab (alias of LCHab) and Luv: the hue of an achromatic pixel is */
  MB200_LCHabColorspace = 13,         /* rounding noise in the reference as well                               */
  MB200_LCHuvColorspace = 14,
  MB200_LogColorspace = 15,           /* table gather, colorspace.c:1055-1163 / :2391-2500 */
  MB200_LMSColorspace = 16,           /* XYZ-derived spaces of the generic branch: <= 1 ULP */
  MB200_LuvColorspace = 17,
  MB200_OHTAColorspace = 18,          /* LUT branch, colorspace.c:1229-1494 */
  MB200_Rec601YCbCrColorspace = 19,   /* LUT branch */
  MB200_Rec709YCbCrColorspace = 20,   /* LUT branch */
  MB200_RGBColorspace = 21,           /* linear RGB */
  MB200_sRGBColorspace = 23,
  MB200_xyYColorspace = 25,
  MB200_XYZColorspace = 26,
  MB200_YCbCrColorspace = 27,
  MB200_YCCColorspace = 28,           /* PhotoYCC, LUT branch :1347-1389 / :2681-2711, bit exact */
  MB200_YDbDrColorspace = 29,
  MB200_YIQColorspace = 30,
  MB200_YPbPrColorspace = 31,
  MB200_YUVColorspace = 32,
  MB200_LinearGRAYColorspace = 33,    /* layout-changing: mb200_transform_colorspace_layout only */
  MB200_JzazbzColorspace = 34,
  MB200_DisplayP3Colorspace = 35,
  MB200_Adobe98Colorspace = 36,
  MB200_ProPhotoColorspace = 37,
  MB200_OklabColorspace = 38,
  MB200_OklchColorspace = 39,
  MB200_CAT02LMSColorspace = 40
} mb200_colorspace;

/* Mirror of KernelInfo (MagickCore/morphology.h:102-130): a singly linked list
   of width x height double arrays, NaN == "not part of the neighbourhood",
   (x,y) the origin.  `type` is an mb200_kernel_type (needed only because the
   reference's 180-degree RotateKernelInfo is a no-op for some built-ins,
   MagickCore/morphology.c:4281-4305). */
typedef enum {
  MB200_UserDefinedKernel = 0, MB200_BlurKernel, MB200_GaussianKernel, MB200_DiskKernel,
  MB200_SquareKernel, MB200_DiamondKernel, MB200_OctagonKernel, MB200_PlusKernel,
  MB200_CrossKernel, MB200_RectangleKernel, MB200_UnityKernel, MB200_DoGKernel,
  MB200_LoGKernel, MB200_BinomialKernel,
  /* the rest of KernelInfoType (MagickCore/morphology.h:27-68): named convolution kernels, hit-and-miss lists, distances */
  MB200_CometKernel, MB200_LaplacianKernel, MB200_SobelKernel, MB200_FreiChenKernel, MB200_RobertsKernel,
  MB200_PrewittKernel, MB200_CompassKernel, MB200_KirschKernel, MB200_RingKernel, MB200_PeaksKernel, MB200_EdgesKernel,
  MB200_CornersKernel, MB200_DiagonalsKernel, MB200_LineEndsKernel, MB200_LineJunctionsKernel, MB200_RidgesKernel,
  MB200_ConvexHullKernel, MB200_ThinSEKernel, MB200_SkeletonKernel, MB200_ChebyshevKernel, MB200_ManhattanKernel,
  MB200_OctagonalKernel, MB200_EuclideanKernel
} mb200_kernel_type;

typedef struct mb200_kernel_info {
  int type;
  size_t width, height;
  long x, y;
  double *values;
  double minimum, maximum, negative_range, positive_range, angle;
  struct mb200_kernel_info *next;
} mb200_kernel_info;

/* ------------------------------------------------------------- runtime ---- */

/* Number of usable sm_90 (H100) devices (0 when there is no GPU / driver). */
MB200_API int mb200_device_count(void);
/* Bind the calling thread (and the library's per-device state) to `device`.
   One process per GPU is the intended deployment (imagemagick_b200.dist). */
MB200_API int mb200_set_device(int device);
MB200_API const char *mb200_last_error(void);
MB200_API const char *mb200_version(void);
/* Number of kernel launches issued by this library since process start
   (bench.py's "gpu_launches"). */
MB200_API unsigned long long mb200_launch_count(void);
/* Block until all work queued by this library on `stream` (NULL = the library's
   own stream for the current device) has finished. */
MB200_API int mb200_synchronize(void *stream);

/* Device pixel-cache staging (the CUDA analogue of AcquireMagickCLCacheInfo /
   GetAuthenticOpenCLBuffer, MagickCore/opencl.c:528-553, MagickCore/cache.c:1259). */
MB200_API int mb200_malloc(void **dev_ptr, size_t bytes);
MB200_API int mb200_free(void *dev_ptr);
MB200_API int mb200_malloc_host(void **host_ptr, size_t bytes);   /* pinned */
MB200_API int mb200_free_host(void *host_ptr);
/* Asynchronous on `stream` when the host memory is pinned; pageable memory is moved through the bounce ring
   (mb200_upload returns once the host buffer has been consumed, mb200_download when it holds the data). */
MB200_API int mb200_upload(void *dev_dst, const void *host_src, size_t bytes, void *stream);
MB200_API int mb200_download(void *host_dst, const void *dev_src, size_t bytes, void *stream);

/* Gives the memory cached in the library's private stream-ordered pool (operator temporaries of the
   current device) back to the driver, keeping at most `keep_bytes`.  The host application's default pool is
   never touched. */
MB200_API int mb200_trim(size_t keep_bytes);
/* Measures the FP64 FMA issue rate of the current device (FMA/s; 16 independent DFMA chains per thread):
   the co-limit of the FP64-accumulating convolution kernels (bench.py's second roofline entry). */
MB200_API int mb200_probe_fp64_fma_rate(double *fma_per_second);
/* Test / developer hook: force the generic kernels ("no_rank1", "no_morph_stream", "no_resize_stream",
   "resize_regular_h", "no_fused_unsharp", "no_resize_fused" = the two streaming passes of ResizeImage where the fused
   vertical + horizontal kernel would run, "resize_fused" = that kernel wherever it applies, also on images whose two-pass
   intermediate fits in L2, "conv_mma" = the FP64 mma.sync kernels of conv_mma.cu for
   RGBA 1-D passes: 1 whenever possible, 0 never, -1 automatic = float-in / float-out passes; initialised from the MB200_<NAME> environment variables).  mb200_get_option reads a switch back;
   "conv_mma_launches" counts the passes the mma.sync kernels have served since process start.
   The tuning knobs of DESIGN §10 are options too: "mma_strip" (>= 8, rounded up to a multiple of 8), "mma_minb" (3, 4),
   "mma_l2pf" (-1, 0, 1), "pair" (0, 1), "pair_async" (0, 1), "pair_async_col" (-1, 0, 1), "col_rot", "row_pair_rot"
   (>= 1), "row_rot" (>= 0), "resize_tma" (0, 1, 2), "resize_chunk" (8, 16), "resize_slots" (0, 2, 3), "resize_strip"
   (>= 0); the counts go up to 2^20.  Any other value is rejected with MB200_EINVAL (an invalid environment value is
   ignored: the default applies).  Launch counters per kernel family, readable like "conv_mma_launches":
   "conv_pair_launches", "conv_pair_async_launches", "conv_generic_launches", "resize_v_stream_launches",
   "resize_h_tma_launches", "resize_h_stream_launches", "resize_fused_launches", "resize_regular_launches",
   "resize_gather_launches", "adaptive_threshold_tile_launches", "adaptive_threshold_direct_launches" (with the switch
   "no_adaptive_tile", which sends AdaptiveThresholdImage to its direct family), "bounding_box_launches". */
MB200_API int mb200_set_option(const char *name, int value);
MB200_API int mb200_get_option(const char *name, int *value);

/* ------------------------------------------ pixel cache staged into HBM ---- */
/* Residency of HOST pixel caches in HBM -- the CUDA analogue of the reference's OpenCL cache plumbing:
     mb200_cache_attach        AcquireMagickCLCacheInfo      MagickCore/opencl.c:528-553
     (operators below)         GetAuthenticOpenCLBuffer      MagickCore/cache.c:1259-1292
     mb200_cache_sync          CopyOpenCLBuffer              MagickCore/cache.c:5341-5364 (sites :1710, :2771, :4079)
     mb200_cache_detach        RelinquishMagickCLCacheInfo   MagickCore/cache.c:978-984
   An attached buffer keeps one HBM copy for its lifetime.  The host-buffer operators find it by the buffer's
   base address: inputs whose HBM copy is current are not uploaded again, results are written to the HBM copy.
   EAGER mode (default): a result is copied to its host buffer before the operator returns, and an input's HBM
   copy is trusted only while it is the sole current copy -- always safe, no cooperation needed.
   LAZY mode (mb200_cache_set_lazy(1)): results stay in HBM until mb200_cache_sync(host) and resident inputs
   are not re-uploaded; the caller must call mb200_cache_sync before the host READS a buffer and
   mb200_cache_host_written after the host WRITES one (the three CopyOpenCLBuffer sites of cache.c are exactly
   those places; INTEGRATION.md shows the patch).  Unattached buffers are staged per call in either mode.
   Host memory that is pinned (mb200_malloc_host, cudaHostRegister, MB200_CACHE_REGISTER) moves at PCIe speed
   (55 GB/s); pageable memory goes through a threaded pinned bounce ring (49 / 44 GB/s up / down instead of
   cudaMemcpy's 9 / 19 GB/s). */
enum { MB200_CACHE_REGISTER = 1 };   /* pin the buffer with cudaHostRegister (67-450 ms per GiB, once) */
MB200_API int mb200_cache_attach(void *host_pixels, size_t bytes, int flags);
MB200_API int mb200_cache_detach(void *host_pixels);            /* drops the HBM copy WITHOUT syncing */
MB200_API int mb200_cache_sync(void *host_pixels);              /* HBM -> host if the HBM copy is newer */
MB200_API int mb200_cache_host_written(void *host_pixels);      /* the HBM copy is stale */
MB200_API int mb200_cache_resident(const void *host_pixels);    /* -1 unknown; bit 0: HBM copy current, bit 1: host copy current */
MB200_API int mb200_cache_set_lazy(int on);                     /* returns the previous mode */
/* uploads, upload bytes, downloads, download bytes, resident-input hits, bytes moved through the bounce ring */
MB200_API void mb200_cache_stats(unsigned long long out[6]);
MB200_API int mb200_copy_threads(void);

/* ------------------------------------------------------- kernel builders ---- */

/* AcquireKernelInfo (MagickCore/morphology.c:485): parses the reference's kernel
   strings -- "blur:RxS[+angle]", "gaussian:RxS", "dog:", "log:", "disk:R[,scale]",
   "square:", "diamond:", "octagon:", "plus:", "cross:", "rectangle:WxH+X+Y",
   "unity", "binomial:", user arrays "WxH+X+Y:v,v,..." and old-style "v,v,v,..." --
   and ';'-separated lists.  Returns NULL on a parse error / unsupported name. */
MB200_API mb200_kernel_info *mb200_acquire_kernel_info(const char *kernel_string);
/* AcquireKernelBuiltIn (MagickCore/morphology.c:950) with GeometryInfo rho,sigma,xi,psi. */
MB200_API mb200_kernel_info *mb200_acquire_kernel_builtin(int type, double rho, double sigma,
                                                         double xi, double psi);
MB200_API mb200_kernel_info *mb200_clone_kernel_info(const mb200_kernel_info *kernel);
MB200_API mb200_kernel_info *mb200_destroy_kernel_info(mb200_kernel_info *kernel);
/* ScaleKernelInfo (MagickCore/morphology.c:4571); flags: 1 = NormalizeValue,
   2 = CorrelateNormalizeValue. */
MB200_API void mb200_scale_kernel_info(mb200_kernel_info *kernel, double scaling_factor, int flags);
/* GetOptimalKernelWidth1D/2D (MagickCore/gem.c:262, :302). */
MB200_API size_t mb200_optimal_kernel_width_1d(double radius, double sigma);
MB200_API size_t mb200_optimal_kernel_width_2d(double radius, double sigma);

/* The kernels SharpenImage (MagickCore/effect.c:3991-4063) and EdgeImage (:1520-1570) build inline
   before calling ConvolveImage. */
MB200_API mb200_kernel_info *mb200_sharpen_kernel(double radius, double sigma);
MB200_API mb200_kernel_info *mb200_edge_kernel(double radius);
/* The anti-diagonal kernel EmbossImage (MagickCore/effect.c:1600-1665) builds inline. */
MB200_API mb200_kernel_info *mb200_emboss_kernel(double radius, double sigma);

/* MotionBlurImage's taps (GetMotionBlurKernel, MagickCore/effect.c:2316-2345) and integer offsets along
   `angle` (:2390-2398).  Returns the tap count; pass NULL arrays to query it. */
MB200_API long mb200_motion_blur_kernel(double radius, double sigma, double angle, double *taps,
    long *offset_x, long *offset_y, size_t max_taps);

/* Resize contribution table of one axis: exactly the start/stop/weights that
   HorizontalFilter / VerticalFilter (MagickCore/resize.c:3398-3443, :3614-3657)
   compute per output column/row.  weights is out_n * max_taps doubles (row o at
   weights[o*max_taps]); returns max_taps (>0) or a negative error.  Pass
   start/count/weights == NULL to only query max_taps. */
MB200_API long mb200_resize_contributions(int filter, size_t in_n, size_t out_n, double factor,
                                         long *start, int *count, double *weights,
                                         size_t max_taps);
/* The "filter:*" expert settings AcquireResizeFilter reads from the image artifacts (MagickCore/resize.c:999-1226), as
   values: the caller (the shim, with the reference's own StringToDouble / ParseCommandOption) does the string parsing.
   `set` says which fields are meaningful.  window + keep_filter restate :999-1043: a "filter:window" alone turns the
   weighting function into SincFast; with a truthy "filter:filter" the requested filter keeps its weighting function. */
enum { MB200_FO_WINDOW = 1, MB200_FO_SIGMA = 2, MB200_FO_KAISER_BETA = 4, MB200_FO_LOBES = 8, MB200_FO_BLUR = 16,
       MB200_FO_SUPPORT = 32, MB200_FO_WIN_SUPPORT = 64, MB200_FO_B = 128, MB200_FO_C = 256 };
typedef struct mb200_filter_options {
  unsigned set;
  int window;              /* FilterType of "filter:window" */
  int keep_filter;         /* "filter:filter" was a truthy string (:1000) */
  long lobes;              /* "filter:lobes" */
  double sigma;            /* "filter:sigma" (Gaussian) */
  double kaiser_beta;      /* "filter:alpha" / "filter:kaiser-beta" / pi * "filter:kaiser-alpha", last one wins (:1104-1117) */
  double blur, support, win_support, b, c;
} mb200_filter_options;
/* ... with expert settings (options == NULL: none) */
MB200_API long mb200_resize_contributions_ex(int filter, const mb200_filter_options *options, size_t in_n, size_t out_n,
                                            double factor, long *start, int *count, double *weights, size_t max_taps);
MB200_API double mb200_resize_filter_weight_ex(int filter, const mb200_filter_options *options, double x);
MB200_API double mb200_resize_filter_support_ex(int filter, const mb200_filter_options *options);
/* GetResizeFilterWeight / GetResizeFilterSupport (MagickCore/resize.c:1690, :1656). */
MB200_API double mb200_resize_filter_weight(int filter, double x);
MB200_API double mb200_resize_filter_support(int filter);

/* ---- DistortImage / RotateImage (MagickCore/distort.c:1754, :2954) through resample.c's EWA sampler ----
   The planner runs on the host without a device: GenerateCoefficients (distort.c:380-960) for Affine (1),
   AffineProjection (2), ScaleRotateTranslate (3), Perspective (4), PerspectiveProjection (5) and RigidAffine (19) --
   all reduce to an affine (6 coefficients) or a perspective (9) reverse map -- and the output geometry: bestfit
   bounds (:1827-1990), a "distort:viewport" given as values, and "distort:scale" (:2393-2410, NaN = not set).  The
   caller allocates dst from plan->columns x plan->rows.  MB200_EUNSUPPORTED: another method; MB200_EINVAL: the
   reference's argument errors (too few / many arguments, a zero scale, an unsolvable matrix, a scale below 0.1). */
#define MB200_RESAMPLE_LUT 1024
typedef enum { MB200_DistortAffineMap = 0, MB200_DistortPerspectiveMap = 1 } mb200_distort_map;
typedef struct mb200_distort_params {
  int map;                       /* mb200_distort_map */
  double coeff[9];               /* output -> source: affine c0..c5; perspective c0..c7 and the ground sign c8 */
  size_t columns, rows;          /* the output image */
  long page_x, page_y;           /* the output's page offset (geometry.x / y) */
  double output_scaling;         /* 1 / |distort:scale| */
  int bestfit;                   /* the source's page is subtracted from each sample point (:2853-2856) */
  long src_page_x, src_page_y;
} mb200_distort_params;
MB200_API int mb200_distort_plan(int method, const double *arguments, size_t number_arguments, int bestfit,
    size_t width, size_t height, long page_x, long page_y, const long *viewport /* w, h, x, y or NULL */,
    double scale, mb200_distort_params *plan);
/* RotateImage's angle reduction (:2976-2988); MB200_EUNSUPPORTED where the reference takes IntegralRotateImage. */
MB200_API int mb200_rotate_plan(double degrees, size_t width, size_t height, long page_x, long page_y,
    mb200_distort_params *plan);

/* The source image's resample settings.  filter: its FilterType (Undefined = Robidoux; Point is MB200_EUNSUPPORTED,
   it interpolates every pixel); filter_options: "filter:*" settings or NULL; virtual_pixel: Undefined (0),
   Background (1), Edge (3), Transparent (7), Black (9), Gray (10), White (11); interpolate: Undefined (0) or
   Bilinear (5); background / matte: the colours as doubles (rgba), matte_alpha != 0 when the matte colour has an
   alpha trait.  On a gray image the background must be gray (the reference re-lays a gray image out to sRGB
   otherwise) and its blue component is the gray value. */
typedef struct mb200_resample_options {
  int filter;
  const mb200_filter_options *filter_options;
  int virtual_pixel;
  int interpolate;
  double background[4];
  double matte[4];
  int matte_alpha;
} mb200_resample_options;
/* The cylindrical weight table of SetResampleFilter (resample.c:1246-1300): lut[MB200_RESAMPLE_LUT], *support. */
MB200_API int mb200_resample_filter_lut(int filter, const mb200_filter_options *options, double *lut, double *support);

/* ---- The orientation and crop operators of MagickCore/transform.c and shear.c: pure data movement ----
   mb200_geometry_plan runs on the host without a device.  It restates the output geometry and page of
     CropImage (transform.c:542)       args: width, height, x, y (the RectangleInfo; width / height 0 = the page's)
     ShaveImage (transform.c:1641)     args: width, height
     FlipImage, FlopImage (:1194, :1329), TransposeImage, TransverseImage (:2127, :2265)   no args
     IntegralRotateImage (shear.c:700) args: rotations (taken mod 4 as a size_t, so -1 is 3)
     RollImage (transform.c:1546)      args: x_offset, y_offset
   in the reference's arithmetic and order, and the map out(x, y) = in(map(x, y)) the kernel runs.  MB200_EUNSUPPORTED
   where the reference returns no image of the operation's own (it warns "GeometryDoesNotContainImage": a crop outside
   the virtual canvas, which it answers with a transparent 1x1 image, a crop of zero area, a shave of half the image or
   more) and for IntegralRotateImage by 0 (a CloneImage); MB200_EINVAL: an empty image, another op. */
typedef enum {
  MB200_GeometryCrop = 0, MB200_GeometryShave = 1, MB200_GeometryFlip = 2, MB200_GeometryFlop = 3,
  MB200_GeometryTranspose = 4, MB200_GeometryTransverse = 5, MB200_GeometryIntegralRotate = 6, MB200_GeometryRoll = 7
} mb200_geometry_op;
/* The dihedral transforms of the map: bit 0 mirrors the source x, bit 1 the source y, bit 2 swaps the axes first. */
typedef enum {
  MB200_MapIdentity = 0, MB200_MapFlop = 1, MB200_MapFlip = 2, MB200_MapRotate180 = 3,
  MB200_MapTranspose = 4, MB200_MapRotate270 = 5, MB200_MapRotate90 = 6, MB200_MapTransverse = 7
} mb200_geometry_map;
typedef struct mb200_page { size_t width, height; long x, y; } mb200_page;   /* the image's RectangleInfo page */
typedef struct mb200_geometry_params {
  int map;                       /* mb200_geometry_map */
  size_t columns, rows;          /* the output image */
  mb200_page page;               /* the output's page */
  long src_x, src_y;             /* the source rectangle's origin (its size is the output's, swapped by bit 2) */
  long roll_x, roll_y;           /* RollImage's offsets, in [0, columns) x [0, rows): out(x, y) = in(x - roll_x, ...) */
} mb200_geometry_params;
MB200_API int mb200_geometry_plan(int op, size_t columns, size_t rows, const mb200_page *page, const long *args,
    mb200_geometry_params *plan);

/* ---- GetImageBoundingBox (MagickCore/attribute.c:391) and TrimImage (transform.c:2412) ----
   The image's settings the bounding box reads: its fuzz, the "trim:edges" artifact as a bitmask of the edges it names
   (MB200_TRIM_EDGES_UNSET when the artifact is not set; 0 when it names none of the four), and its colourspace (CMYK
   adds the black term to the fuzzy comparison and needs 4 or 5 channels, HCL / HCLp / HSB / HSI / HSL / HSV measure the
   first channel as a hue arc, anything else compares plainly).  "trim:percent-background" selects another algorithm
   (GetEdgeBoundingBox) that is not served here. */
typedef enum {
  MB200_TrimEdgeNorth = 1, MB200_TrimEdgeEast = 2, MB200_TrimEdgeSouth = 4, MB200_TrimEdgeWest = 8
} mb200_trim_edge;
#define MB200_TRIM_EDGES_UNSET (-1)
typedef struct mb200_trim_options {
  double fuzz;                   /* image->fuzz, in quantum units */
  int edges;                     /* mb200_trim_edge bits, or MB200_TRIM_EDGES_UNSET */
  int colorspace;                /* mb200_colorspace */
} mb200_trim_options;
/* MagickCore/geometry.h GravityType -- same numeric values */
typedef enum {
  MB200_UndefinedGravity = 0, MB200_NorthWestGravity = 1, MB200_NorthGravity = 2, MB200_NorthEastGravity = 3,
  MB200_WestGravity = 4, MB200_CenterGravity = 5, MB200_EastGravity = 6, MB200_SouthWestGravity = 7,
  MB200_SouthGravity = 8, MB200_SouthEastGravity = 9
} mb200_gravity;
/* The host half of GetImageBoundingBox, without a device.  `summaries` holds 4 words per row, all 0 when nothing in the
   row mismatches: [0] columns - the first x not fuzzy-equivalent to the top-left pixel, [1] 1 + the last x not
   equivalent to the top-right pixel, [2] nonzero when any x is not equivalent to the bottom-left pixel, [3] columns -
   the first x not equivalent to the bottom-right pixel.  *box receives what the reference's single-threaded row loop
   (:487-551) computes from the initial bounds `edges` gives, after its final arithmetic (:553-560, in size_t, so a
   one-column image can give width 2).  *warning (may be NULL) is set to 1 where the reference warns
   "GeometryDoesNotContainImage" -- the loop left a zero width or height, and the box is returned as it is -- and to 0
   otherwise: the final arithmetic can itself give a zero side, without the warning.  MB200_EINVAL: no buffer, an empty
   image, a bad `edges`. */
MB200_API int mb200_bounding_box_from_rows(const unsigned *summaries, size_t columns, size_t rows, int edges,
    mb200_page *box, int *warning);
/* TrimImage's geometry (:2445-2509) for a bounding box `box` of a columns x rows image with page `page`: the box grown
   to `min_size` (width, height; NULL: no "trim:minSize") under `gravity` when both of its sides are smaller, offset by
   the page, then the CropImage plan of mb200_geometry_plan.  MB200_EUNSUPPORTED for a zero box (the reference returns a
   transparent 1x1 clone) and wherever the crop plan declines. */
MB200_API int mb200_trim_plan(size_t columns, size_t rows, const mb200_page *page, const mb200_page *box, int gravity,
    const size_t *min_size, mb200_geometry_params *plan);

/* --------------------------------------- device-resident operators (HBM) ---- */
/* src/dst are DEVICE pointers (from mb200_malloc or any CUDA allocation, e.g. a
   torch tensor's data_ptr()); they must not alias unless stated.  `stream` is a
   cudaStream_t passed as void* (NULL = library stream).  Calls are asynchronous
   with respect to the host unless a `changed` result is requested. */

/* MorphologyPrimitive (MagickCore/morphology.c:2566-3227) for ONE kernel:
   method in {Convolve, Erode, Dilate}.  *changed (host, may be NULL) receives the
   reference's return value (pixels changed).  Width-1 Convolve kernels take the
   reference's column path semantics (:2654-2807). */
MB200_API int mb200_morphology_primitive_dev(const float *src, float *dst, size_t width,
    size_t height, int channels, int method, const mb200_kernel_info *kernel, double bias,
    long long *changed, void *stream);

/* MorphologyImage / MorphologyApply (MagickCore/morphology.c:4129, :3634) with the
   default compose (re-iterate kernel lists): iterations (<0 = until unchanged),
   compound methods Open / Close / Smooth, Correlate, and -- for single kernels -- the
   "difference" methods EdgeIn / EdgeOut / Edge / TopHat / BottomHat, whose final
   CompositeImage(..., DifferenceCompositeOp, ...) step (:3995-4012) runs as one point
   kernel (bit exact).  HitAndMiss / Thinning / Thicken / Distance / Voronoi / the
   *Intensity methods return MB200_EUNSUPPORTED; Distance and Voronoi have their own
   entry point, mb200_morphology_direct_image_dev. */
MB200_API int mb200_morphology_image_dev(const float *src, float *dst, size_t width,
    size_t height, int channels, int method, long iterations,
    const mb200_kernel_info *kernel, double bias, void *stream);

/* MorphologyImage with the directly applied methods, Distance and Voronoi (MagickCore/morphology.c:3736-3776,
   MorphologyPrimitiveDirect :3242-3623): one forward and one reverse sweep, whatever the iteration count and bias, with
   the head kernel of the list only.  Bit exact.  Every channel is swept (a `-channel` selection is put back with
   mb200_restore_channels_dev).  Voronoi replaces the swept alpha with the source's, ClampPixel(QuantumRange*QuantumScale*a),
   clamps the other channels to [0, QuantumRange], and leaves the image's alpha trait at Copy (the caller's to record);
   on an image without alpha its result needs one more channel, so it returns MB200_EUNSUPPORTED.  MB200_EINVAL: a method
   other than Distance / Voronoi, no kernel, or an origin outside the kernel; MB200_EUNSUPPORTED also for kernels the
   wavefront cannot hold (more than 1 024 non-NaN cells in a pass, more than 32 rows on one side of the origin, or rings
   beyond shared memory).  Both are checked before the device is touched. */
MB200_API int mb200_morphology_direct_image_dev(const float *src, float *dst, size_t width, size_t height,
    int channels, int method, const mb200_kernel_info *kernel, void *stream);

/* DistortImage's sampling loop (MagickCore/distort.c:2474-2890) for a plan from mb200_distort_plan /
   mb200_rotate_plan: one thread per output pixel runs the map, the perspective validity and horizon blend, and
   ResamplePixelColor (resample.c:315-670) -- the miss test, the limit fallbacks, the EWA parallelogram scan over the
   weight table and the interpolated fallback -- in the reference's order with unfused double operations: bit exact.
   dst (plan->columns x plan->rows x channels) must not alias src.  MB200_EUNSUPPORTED, before the device is touched
   and with dst untouched: the Point filter, interpolate methods other than Undefined / Bilinear, virtual-pixel
   methods other than the six above, and a perspective map on an image without alpha whose horizon blend band
   crosses the output (the reference's blend there reads an alpha sum carried along the row). */
MB200_API int mb200_distort_image_dev(const float *src, size_t width, size_t height, int channels, float *dst,
    const mb200_distort_params *plan, const mb200_resample_options *options, void *stream);

/* The map of a plan from mb200_geometry_plan: dst (plan->columns x plan->rows x channels, 1-5 channels) receives the
   source samples as 32-bit words, so every bit pattern (NaN payloads, -0, denormals) is kept.  dst must not alias src.
   MB200_EINVAL, before the device is touched: a map or source rectangle that does not fit the source image. */
MB200_API int mb200_geometry_image_dev(const float *src, size_t width, size_t height, int channels, float *dst,
    const mb200_geometry_params *plan, void *stream);

/* GetImageBoundingBox (MagickCore/attribute.c:391) of `src` (1-5 channels: gray, gray + alpha, RGB, RGBA, or CMYK and
   CMYKA when options->colorspace is CMYK): one scan for the row summaries of mb200_bounding_box_from_rows, with
   IsFuzzyEquivalencePixelInfo (pixel.c:6028) restated in double, then that function.  Bit exact, with the reference's
   single-threaded result on images of any height; *warning (may be NULL) as there.  Synchronises `stream` to return
   *box.  MB200_EINVAL, before the device is touched: bad options or a channel count the colourspace does not have;
   MB200_EUNSUPPORTED: images wider than 2^32 - 1. */
MB200_API int mb200_bounding_box_dev(const float *src, size_t width, size_t height, int channels,
    const mb200_trim_options *options, mb200_page *box, int *warning, void *stream);

/* ConvolveImage (MagickCore/effect.c:1170) */
MB200_API int mb200_convolve_image_dev(const float *src, float *dst, size_t width, size_t height,
    int channels, const mb200_kernel_info *kernel, void *stream);
/* BlurImage (MagickCore/effect.c:765) == AccelerateBlurImage (accelerate-private.h:36) */
MB200_API int mb200_blur_image_dev(const float *src, float *dst, size_t width, size_t height,
    int channels, double radius, double sigma, void *stream);
/* GaussianBlurImage (MagickCore/effect.c:1709) */
MB200_API int mb200_gaussian_blur_image_dev(const float *src, float *dst, size_t width,
    size_t height, int channels, double radius, double sigma, void *stream);
/* UnsharpMaskImage (MagickCore/effect.c:4256) == AccelerateUnsharpMaskImage (:46) */
MB200_API int mb200_unsharp_mask_image_dev(const float *src, float *dst, size_t width,
    size_t height, int channels, double radius, double sigma, double gain, double threshold,
    void *stream);
/* SharpenImage (MagickCore/effect.c:3991) and EdgeImage (:1520): ConvolveImage with the kernel above */
MB200_API int mb200_sharpen_image_dev(const float *src, float *dst, size_t width, size_t height,
    int channels, double radius, double sigma, void *stream);
MB200_API int mb200_edge_image_dev(const float *src, float *dst, size_t width, size_t height,
    int channels, double radius, void *stream);
/* EqualizeImage (MagickCore/enhance.c:2040; the reference's hook is AccelerateEqualizeImage, accelerate-private.h), in place:
   histogram on the device, the 65 536-entry map on the host in the reference's order, table lookup on the device --
   bit exact.  sync_channels != 0: the channel mask carries SyncChannels (the default mask does): one histogram of the
   pixel intensity for all channels; 0: one histogram per channel.  Synchronises `stream`. */
MB200_API int mb200_equalize_image_dev(float *buf, size_t width, size_t height, int channels, int sync_channels,
    void *stream);
/* EmbossImage (MagickCore/effect.c:1600): ConvolveImage with mb200_emboss_kernel, then EqualizeImage. */
MB200_API int mb200_emboss_image_dev(const float *src, float *dst, size_t width, size_t height, int channels,
    double radius, double sigma, void *stream);
/* StatisticImage (MagickCore/statistic.c:2918): `type` is a StatisticType (statistic.h:141-151: 1 Gradient, 2 Maximum,
   3 Mean, 4 Median, 5 Minimum, 6 Mode, 7 Nonpeak, 8 RootMeanSquare, 9 StandardDeviation, 10 Contrast) over a
   window_width x window_height neighbourhood, bit exact. */
MB200_API int mb200_statistic_image_dev(const float *src, float *dst, size_t width, size_t height, int channels,
    int type, size_t window_width, size_t window_height, void *stream);
/* RotationalBlurImage (MagickCore/effect.c:3129) == AccelerateRotationalBlurImage (accelerate-private.h), bit exact. */
MB200_API int mb200_rotational_blur_image_dev(const float *src, float *dst, size_t width, size_t height, int channels,
    double angle, void *stream);
/* BilateralBlurImage (MagickCore/effect.c:821), odd window sizes (even ones return MB200_EUNSUPPORTED), bit exact. */
MB200_API int mb200_bilateral_blur_image_dev(const float *src, float *dst, size_t width, size_t height, int channels,
    size_t window_width, size_t window_height, double intensity_sigma, double spatial_sigma, void *stream);
/* AdaptiveBlurImage (MagickCore/effect.c:128) / AdaptiveSharpenImage (:447): EdgeImage -> AutoLevelImage -> BlurImage ->
   AutoLevelImage gives the edge map that selects a kernel size per pixel; every stage in the reference's operation
   order, bit exact. */
MB200_API int mb200_adaptive_blur_image_dev(const float *src, float *dst, size_t width, size_t height, int channels,
    double radius, double sigma, void *stream);
MB200_API int mb200_adaptive_sharpen_image_dev(const float *src, float *dst, size_t width, size_t height, int channels,
    double radius, double sigma, void *stream);
/* SelectiveBlurImage (MagickCore/effect.c:3406): contrast-gated Gaussian (threshold in quantum units), bit exact. */
MB200_API int mb200_selective_blur_image_dev(const float *src, float *dst, size_t width, size_t height, int channels,
    double radius, double sigma, double threshold, void *stream);
/* MotionBlurImage (MagickCore/effect.c:2347) == AccelerateMotionBlurImage (accelerate-private.h). */
MB200_API int mb200_motion_blur_image_dev(const float *src, float *dst, size_t width, size_t height,
    int channels, double radius, double sigma, double angle, void *stream);
/* DespeckleImage (MagickCore/effect.c:1308) == AccelerateDespeckleImage (accelerate-private.h): the 16 Hulls of every
   channel (alpha included) over a zero border, bit exact.  Timings of these three (8192^2 RGBA, one H100 80GB HBM3 at
   400 W): Despeckle 20.2 ms, LocalContrast 10x12.5 12.2 ms, WaveletDenoise 11.7 ms (DESIGN.md §5.7). */
MB200_API int mb200_despeckle_image_dev(const float *src, float *dst, size_t width, size_t height, int channels,
    void *stream);
/* LocalContrastImage (MagickCore/effect.c:2013) == AccelerateLocalContrastImage, bit exact (a pixel whose luma is 0
   gives NaN in R, G and B, as in the reference).  MB200_EUNSUPPORTED where the kernel width
   (ssize_t) (max(width,height)*0.002*|radius|) exceeds width - 1: the reference then reads padding it never wrote. */
MB200_API int mb200_local_contrast_image_dev(const float *src, float *dst, size_t width, size_t height, int channels,
    double radius, double strength, void *stream);
/* WaveletDenoiseImage (MagickCore/visual-effects.c:3515) on R, G, B (gray), alpha untouched, bit exact.  The reference's
   hook AccelerateWaveletDenoiseImage drops `softness`; this takes it.  MB200_EUNSUPPORTED below 32 columns or rows
   (HatTransform's level-4 step reads outside the line there). */
MB200_API int mb200_wavelet_denoise_image_dev(const float *src, float *dst, size_t width, size_t height, int channels,
    double threshold, double softness, void *stream);
/* ResizeImage (MagickCore/resize.c:3761) == AccelerateResizeImage (:43).  filter
   UndefinedFilter applies the reference's own default choice (:3806-3816). */
MB200_API int mb200_resize_image_ex_dev(const float *src, size_t width, size_t height, int channels, float *dst,
                                       size_t out_width, size_t out_height, int filter,
                                       const mb200_filter_options *options, void *stream);
MB200_API int mb200_resize_image_dev(const float *src, size_t width, size_t height, int channels,
    float *dst, size_t out_width, size_t out_height, int filter, void *stream);
/* SampleImage (MagickCore/resize.c:3907): nearest-sample gather with the default sampling offset
   (0.5 - MagickEpsilon; the "sample:offset" artifact is the shim's decline), bit exact. */
MB200_API int mb200_sample_image_dev(const float *src, size_t width, size_t height, int channels,
    float *dst, size_t out_width, size_t out_height, void *stream);
/* ScaleImage (MagickCore/resize.c:4106): box scaling.  The reference's sequential (span, scale) state machines are
   simulated on the host (mb200_scale_contributions) into per-output term lists; the gather kernel accumulates them in
   the reference's order with unfused double operations: bit exact, reductions and enlargements alike. */
MB200_API int mb200_scale_image_dev(const float *src, size_t width, size_t height, int channels,
    float *dst, size_t out_width, size_t out_height, void *stream);
MB200_API long mb200_scale_contributions(int axis, size_t in_n, size_t out_n, long *offsets, int *index,
    double *weight, size_t max_terms);
/* ThumbnailImage (MagickCore/resize.c:4591-4650), pixel path only: SampleImage to 4x the target when both
   integer reduction factors exceed 4, ResizeImage(BoxFilter) to 2x when they exceed 2, then
   ResizeImage(`filter` = image->filter; UndefinedFilter selects LanczosSharp like the reference).  The
   profile stripping and Thumb::* properties the reference adds afterwards are left to the caller. */
MB200_API int mb200_thumbnail_image_dev(const float *src, size_t width, size_t height, int channels,
    float *dst, size_t columns, size_t rows, int filter, void *stream);
/* TransformImageColorspace (MagickCore/colorspace.c:1751), in place on `buf`. */
MB200_API int mb200_transform_colorspace_dev(float *buf, size_t width, size_t height,
    int channels, int from_colorspace, int to_colorspace, void *stream);
/* ... with the image settings the reference reads inside sRGBTransformImage / TransformsRGBImage, as values (the shim
   parses them with the reference's own functions): the "color:illuminant" artifact (colorspace.c:761-773, :2093-2105) =
   the reference white of Lab, LCH, LCHab, LCHuv and Luv; the "white-luminance" property (:996, :2331) of Jzazbz; the
   "film-gamma", "reference-black" and "reference-white" properties (:1085-1095, :2416-2426) of Log.  (Log's "gamma"
   property, :1081, cannot be set on an image: SetImageProperty diverts that key to image->gamma, property.c:4583.)
   options == NULL or a clear `set` bit: the reference's default. */
typedef enum {                          /* MagickCore/color.h:40-54 IlluminantType -- same numeric values */
  MB200_AIlluminant = 0, MB200_BIlluminant, MB200_CIlluminant, MB200_D50Illuminant, MB200_D55Illuminant,
  MB200_D65Illuminant, MB200_D75Illuminant, MB200_EIlluminant, MB200_F2Illuminant, MB200_F7Illuminant, MB200_F11Illuminant
} mb200_illuminant;
enum { MB200_CO_ILLUMINANT = 1, MB200_CO_WHITE_LUMINANCE = 2, MB200_CO_FILM_GAMMA = 4, MB200_CO_REFERENCE_BLACK = 8,
       MB200_CO_REFERENCE_WHITE = 16 };
typedef struct mb200_colorspace_options {
  unsigned set;
  int illuminant;                      /* mb200_illuminant */
  double white_luminance;
  double film_gamma, reference_black, reference_white;    /* reference_black / _white within 0..1024 */
} mb200_colorspace_options;
MB200_API int mb200_transform_colorspace_ex_dev(float *buf, size_t width, size_t height, int channels,
    int from_colorspace, int to_colorspace, const mb200_colorspace_options *options, void *stream);
/* The colourspaces that change the channel layout of the pixel cache: GRAY and LinearGRAY (gray[, alpha]) and CMYK
   (cyan, magenta, yellow, black[, alpha]); every other space is 3 channels (+ alpha).  The in-place entry points above
   return MB200_EUNSUPPORTED for any pair involving them.  mb200_colorspace_channels gives the channel count of a space. */
MB200_API int mb200_colorspace_channels(int colorspace, int has_alpha);
/* TransformImageColorspace (colorspace.c:1751) out of place: `src` (src_channels, tagged from_colorspace) -> `dst`
   (dst_channels, tagged to_colorspace); `src` is never written and must not overlap `dst`.  Legs: sRGB -> GRAY
   (:901-957) / LinearGRAY (:843-900), GRAY / LinearGRAY -> sRGB (:2171-2291, R = G = B = the reference's weighted sum of
   the gray sample), sRGB <-> CMYK (:778-842, :2110-2170); every other pair goes through sRGB with the in-place legs (any
   pair the in-place entry points serve is served here too).  Alpha is carried over.  Bit exact for the GRAY and CMYK
   legs, <= 1 ULP for the LinearGRAY ones; hops add the error of the in-place leg.  Channel counts off the layout rule
   give MB200_EINVAL, a space without a leg (scRGB, Transparent, ...) MB200_EUNSUPPORTED; `dst` is untouched on every
   failure. */
MB200_API int mb200_transform_colorspace_layout_dev(const float *src, int src_channels, float *dst, int dst_channels,
    size_t width, size_t height, int from_colorspace, int to_colorspace, const mb200_colorspace_options *options,
    void *stream);
/* The host-built tables behind the Log and YCC legs (no device needed): the 65536-entry `logmap` of colorspace.c:1100-1106
   (forward != 0) / :2431-2440 (inverse) for the given film settings, and the 1389-entry PhotoYCC table of :1828. */
MB200_API int mb200_log_colorspace_table(int forward, const mb200_colorspace_options *options, float *table65536);
MB200_API int mb200_ycc_table(float *table1389);

/* Threshold point operators of MagickCore/threshold.c, in place on `buf`, bit exact.
   BilevelImage (:805): every channel (alpha included) := intensity <= threshold ? 0 : QuantumRange,
   intensity = GetPixelIntensity (pixel.c:2356, Rec709Luma; the gray sample for Gray / Gray+Alpha).
   A non-gray image is re-tagged sRGB by the reference (:827); the caller owns that tag. */
MB200_API int mb200_bilevel_image_dev(float *buf, size_t width, size_t height, int channels,
    double threshold, void *stream);
/* BlackThresholdImage (:927) / WhiteThresholdImage (:2518).  `thresholds` is the reference's
   geometry string "v[,v[,v[,v]]][%]" = red[,green[,blue[,alpha]]] (missing green/blue default to
   red, alpha to 100, '%' scales all by QuantumRange/100, :955-985).  Gray images (which the
   reference first promotes to sRGB, :949), linear-RGB images (`colorspace` == MB200_RGBColorspace:
   the intensity then needs EncodePixelGamma) and other geometry syntax return MB200_EUNSUPPORTED. */
MB200_API int mb200_black_threshold_image_dev(float *buf, size_t width, size_t height, int channels,
    int colorspace, const char *thresholds, void *stream);
MB200_API int mb200_white_threshold_image_dev(float *buf, size_t width, size_t height, int channels,
    int colorspace, const char *thresholds, void *stream);
/* ClampImage (:1087): ClampPixel on every channel (HDRI: below 0 -> 0, >= QuantumRange -> QuantumRange). */
MB200_API int mb200_clamp_image_dev(float *buf, size_t width, size_t height, int channels, void *stream);
/* AdaptiveThresholdImage (:182), out of place `src` -> `dst` (no overlap), bit exact: every channel of `update_mask`
   := (double) centre <= mean ? 0 : QuantumRange, mean = S / (double) (width*height) + bias, where S is the reference's
   running double sum of the width x height window (origin -(width/2), -(height/2); edge virtual pixels), updated in the
   reference's order along each row (a NaN or +-inf that enters it stays for the rest of the row).  The other channels
   (the Copy trait) copy the source.  `bias` is in quantum units (the CLI's `-lat WxH+b%` passes QuantumRange*b/100).
   width == 0 or height == 0 copies `src`.  Windows wider or taller than MB200_ADAPTIVE_THRESHOLD_MAX_WINDOW give
   MB200_EUNSUPPORTED with `dst` untouched. */
#define MB200_ADAPTIVE_THRESHOLD_MAX_WINDOW 4096
MB200_API int mb200_adaptive_threshold_image_dev(const float *src, float *dst, size_t width, size_t height, int channels,
    size_t window_width, size_t window_height, double bias, unsigned update_mask, void *stream);
/* MagickCore/threshold.h AutoThresholdMethod -- same numeric values (Undefined means OTSU) */
typedef enum {
  MB200_UndefinedThresholdMethod = 0, MB200_KapurThresholdMethod, MB200_OTSUThresholdMethod,
  MB200_TriangleThresholdMethod
} mb200_auto_threshold_method;
/* AutoThresholdImage (:660), in place, default channel mask: the 256-bin histogram of
   ScaleQuantumToChar(ClampToQuantum(intensity)), the threshold of `method` computed on the host in the reference's order
   with the same libm calls, then BilevelImage at QuantumRange*threshold/100.  `threshold_percent` receives the threshold
   (the "auto-threshold:threshold" property is its "%g%%").  Bit exact.  Images of 2^32 pixels or more give
   MB200_EUNSUPPORTED. */
MB200_API int mb200_auto_threshold_image_dev(float *buf, size_t width, size_t height, int channels, int method,
    double *threshold_percent, void *stream);
/* RangeThresholdImage (:2377), in place on the channels of `update_mask`: the five-way branch of :2446-2464 on the
   pixel's intensity (per_channel == 0: the default channel mask) or on the channel's own sample (per_channel != 0: a
   `-channel` selection).  Bit exact.  Gray images (1-2 channels), which the reference first transforms to sRGB, give
   MB200_EUNSUPPORTED: transform them with mb200_transform_colorspace_layout_dev first. */
MB200_API int mb200_range_threshold_image_dev(float *buf, size_t width, size_t height, int channels, double low_black,
    double low_white, double high_white, double high_black, int per_channel, unsigned update_mask, void *stream);
/* PerceptibleImage (:2092), in place: PerceptibleThreshold (:2080) on the channels of `update_mask`.  Bit exact. */
MB200_API int mb200_perceptible_image_dev(float *buf, size_t width, size_t height, int channels, double epsilon,
    unsigned update_mask, void *stream);

/* In-place point operators of MagickCore/enhance.c and statistic.c (the reference's in-place accelerate hooks,
   accelerate-private.h:50-60), on `buf`.  Gray images (1 or 2 channels) give R, G and B the gray sample; where the three
   results differ the blue one is written, as in the reference.  Alpha is untouched except by FunctionImage.
   ContrastImage (enhance.c:1370): HSB brightness pushed along a sine (sharpen != 0) or pulled back (0); <= 1 ULP. */
MB200_API int mb200_contrast_image_dev(float *buf, size_t width, size_t height, int channels, int sharpen, void *stream);
/* ModulateImage (enhance.c:3461) with the geometry "B,S,H" already parsed into percentages, `colorspace` the
   "modulate:colorspace" artifact (HCL, HCLp, HSB, HSI, HSL, HSV, HWB, LCH, LCHab, LCHuv; any other value is HSL) and
   `illuminant` a value of mb200_illuminant: the "color:illuminant" artifact, used by the LCH spaces (for an unparsable
   artifact the reference uses D65 and HSL; the caller passes those).  Bit exact in HCL, HCLp, HSB, HSL, HSV and HWB, <= 1 ULP in HSI,
   LCHab and LCHuv (except the hue noise of achromatic pixels when the chroma is scaled, DESIGN.md §5.8).  The re-tag of an
   image whose colourspace is not sRGB-compatible (:3681) is the caller's. */
MB200_API int mb200_modulate_image_dev(float *buf, size_t width, size_t height, int channels, double percent_brightness,
    double percent_saturation, double percent_hue, int colorspace, int illuminant, void *stream);
/* MagickCore/pixel.h:110-120 PixelIntensityMethod -- same numeric values */
typedef enum {
  MB200_UndefinedPixelIntensityMethod = 0, MB200_AveragePixelIntensityMethod, MB200_BrightnessPixelIntensityMethod,
  MB200_LightnessPixelIntensityMethod, MB200_MSPixelIntensityMethod, MB200_Rec601LumaPixelIntensityMethod,
  MB200_Rec601LuminancePixelIntensityMethod, MB200_Rec709LumaPixelIntensityMethod,
  MB200_Rec709LuminancePixelIntensityMethod, MB200_RMSPixelIntensityMethod
} mb200_pixel_intensity_method;
/* GrayscaleImage (enhance.c:2474): the intensity of R, G, B by `method` into channel 0; the other channels are left as
   they are.  The Luma methods (and Undefined) encode the gamma of a linear-RGB image (`image_colorspace` ==
   MB200_RGBColorspace), the Luminance methods decode that of an sRGB one.  The caller does the rest of the reference's
   hook branch (:2503-2511): image->intensity, GrayscaleType, and SetImageColorspace(GRAY, or LinearGRAY for the
   Luminance methods), which keeps channel 0 (and alpha).  Bit exact without a gamma step, <= 1 ULP with one. */
MB200_API int mb200_grayscale_image_dev(float *buf, size_t width, size_t height, int channels, int method,
    int image_colorspace, void *stream);
/* MagickCore/statistic.h:130-137 MagickFunction -- same numeric values */
typedef enum {
  MB200_UndefinedFunction = 0, MB200_ArcsinFunction, MB200_ArctanFunction, MB200_PolynomialFunction,
  MB200_SinusoidFunction
} mb200_function;
#define MB200_MAX_FUNCTION_PARAMETERS 32
/* FunctionImage (statistic.c:1064) on the channels whose bit is set in `update_mask` (the Update trait: alpha is one of
   them by default; a `-channel` selection clears the others).  At most MB200_MAX_FUNCTION_PARAMETERS parameters (more:
   MB200_EUNSUPPORTED, `buf` untouched).  Polynomial and Undefined bit exact, Sinusoid / Arcsin / Arctan <= 1 ULP. */
MB200_API int mb200_function_image_dev(float *buf, size_t width, size_t height, int channels, int function,
    size_t number_parameters, const double *parameters, unsigned update_mask, void *stream);
/* The level and stretch operators of enhance.c, in place.  `update_mask`: bit c = channel c has the Update trait (all
   channels, alpha included, by default).  `per_channel`: the image's channel mask is not AllChannels (a `-channel`
   selection, even one that leaves every trait at its default).  Bad arguments give MB200_EINVAL, unsupported cases
   MB200_EUNSUPPORTED; both leave `buf` untouched.
   ContrastStretchImage (enhance.c:1544; NormalizeImage is black 0.02 N, white 0.99 N for N pixels): one intensity
   histogram (Rec709Luma, no gamma step: the caller declines linear images and other intensity methods) for every
   channel, or one per channel with `per_channel`; black / white bins per channel ([4], unused entries 0) are returned
   for the "histogram:contrast-stretch" property.  IdentifyImageType's gray re-layout (SetImageColorspace(GRAY) of a
   gray-valued image) is the caller's, before the call: see mb200_identify_gray_dev.  Bit exact.  Reads the histogram
   back, so it synchronises `stream`.  Images of 2^32 pixels or more: MB200_EUNSUPPORTED. */
MB200_API int mb200_contrast_stretch_image_dev(float *buf, size_t width, size_t height, int channels, double black_point,
    double white_point, int per_channel, unsigned update_mask, float *black, float *white, void *stream);
/* LinearStretchImage (enhance.c:3347): one intensity histogram, black / white bins by its own search (returned for the
   "histogram:linear-stretch" property), then LevelImage(black, white, 1) on the Update channels.  Bit exact.
   Synchronises `stream`; 2^32 pixels or more: MB200_EUNSUPPORTED. */
MB200_API int mb200_linear_stretch_image_dev(float *buf, size_t width, size_t height, int channels, double black_point,
    double white_point, unsigned update_mask, double *black_bin, double *white_bin, void *stream);
/* LevelImage (enhance.c:2913, with its closing ClampImage) and LevelizeImage (:3062, no clamp) on the Update channels.
   Bit exact at gamma 1, <= 1 ULP otherwise (CUDA pow).  Asynchronous. */
MB200_API int mb200_level_image_dev(float *buf, size_t width, size_t height, int channels, double black_point,
    double white_point, double gamma, unsigned update_mask, void *stream);
MB200_API int mb200_levelize_image_dev(float *buf, size_t width, size_t height, int channels, double black_point,
    double white_point, double gamma, unsigned update_mask, void *stream);
/* MinMaxStretchImage (histogram.c:927; AutoLevelImage is black 0, white 0, gamma 1): GetImageRange, each row seeded by
   its first sample of channel 0, then LevelImage(min + black, max - white, gamma) when the two differ by MagickEpsilon
   or more.  With `per_channel` the Update colour channels one at a time in channel order (range, then level); alpha is
   never levelled there, as in the reference.  The per-channel loop takes the gray / RGB layout (colour channels at
   offsets 0-2, alpha last); a CMYK image's K would be levelled by the reference and is the caller's to decline.  The decision is taken on the device: asynchronous.  Bit exact at gamma 1. */
MB200_API int mb200_minmax_stretch_image_dev(float *buf, size_t width, size_t height, int channels, double black,
    double white, double gamma, int per_channel, unsigned update_mask, void *stream);
/* GammaImage (enhance.c:2322): nothing for gamma 1; otherwise the reference's 65 536-entry table (built on the host with
   libm; all zeros for gamma 0) on the Update channels.  Bit exact.  The caller multiplies image->gamma.  Nothing is read
   back, but the table is a pageable upload, which CUDA orders after the work already queued on `stream`: the call
   returns once that work is done and the table is on the device. */
MB200_API int mb200_gamma_image_dev(float *buf, size_t width, size_t height, int channels, double gamma,
    unsigned update_mask, void *stream);
/* IdentifyImageGray's pixel scan (attribute.c:1564-1626; IsPixelGray / IsPixelMonochrome on channels 0-2, or the gray
   sample three times for 1-2 channels): *type = 0 not gray, 1 grayscale, 2 bilevel.  Synchronises `stream`. */
MB200_API int mb200_identify_gray_dev(const float *buf, size_t width, size_t height, int channels, int *type,
    void *stream);

/* Copy-trait channels.  With a `-channel` selection the reference hands the unselected channels through from the
   operator's source (MagickCore/morphology.c:2733-2737, effect.c:4346-4350); ResizeImage takes the nearest source sample
   of each pass (resize.c:3697-3707).  The operators above compute every channel; these point passes put the Copy channels
   back into `dst` (bit c of update_mask set = channel c is updated by the operator).  Valid for the operators whose
   selected channels do not depend on the selection: Blur, GaussianBlur, Convolve, the non-difference morphology methods,
   UnsharpMask, Sharpen, Edge and Resize. */
MB200_API int mb200_restore_channels_dev(float *dst, const float *src, size_t width, size_t height, int channels,
    unsigned update_mask, void *stream);
MB200_API int mb200_resize_copy_channels_dev(const float *src, size_t width, size_t height, int channels, float *dst,
    size_t out_width, size_t out_height, int filter, unsigned update_mask, void *stream);

/* ---------------------------------------------- host-buffer operators ---- */
/* Same operators on HOST buffers: stage into HBM, run, copy back, synchronise.
   These are what the MagickCore shim calls with the pixel-cache pointers
   (GetVirtualPixels / GetAuthenticPixels, MagickCore/cache.c:3257, :1490). */
MB200_API int mb200_blur_image(const float *src, float *dst, size_t width, size_t height,
    int channels, double radius, double sigma);
MB200_API int mb200_gaussian_blur_image(const float *src, float *dst, size_t width, size_t height,
    int channels, double radius, double sigma);
MB200_API int mb200_convolve_image(const float *src, float *dst, size_t width, size_t height,
    int channels, const mb200_kernel_info *kernel);
MB200_API int mb200_morphology_image(const float *src, float *dst, size_t width, size_t height,
    int channels, int method, long iterations, const mb200_kernel_info *kernel, double bias);
MB200_API int mb200_morphology_direct_image(const float *src, float *dst, size_t width, size_t height,
    int channels, int method, const mb200_kernel_info *kernel);
MB200_API int mb200_unsharp_mask_image(const float *src, float *dst, size_t width, size_t height,
    int channels, double radius, double sigma, double gain, double threshold);
MB200_API int mb200_distort_image(const float *src, size_t width, size_t height, int channels, float *dst,
    const mb200_distort_params *plan, const mb200_resample_options *options);
MB200_API int mb200_geometry_image(const float *src, size_t width, size_t height, int channels, float *dst,
    const mb200_geometry_params *plan);
MB200_API int mb200_bounding_box(const float *src, size_t width, size_t height, int channels,
    const mb200_trim_options *options, mb200_page *box, int *warning);
MB200_API int mb200_sharpen_image(const float *src, float *dst, size_t width, size_t height, int channels,
    double radius, double sigma);
MB200_API int mb200_edge_image(const float *src, float *dst, size_t width, size_t height, int channels,
    double radius);
MB200_API int mb200_motion_blur_image(const float *src, float *dst, size_t width, size_t height, int channels,
    double radius, double sigma, double angle);
MB200_API int mb200_restore_channels(float *dst, const float *src, size_t width, size_t height, int channels,
    unsigned update_mask);
MB200_API int mb200_resize_copy_channels(const float *src, size_t width, size_t height, int channels, float *dst,
    size_t out_width, size_t out_height, int filter, unsigned update_mask);
MB200_API int mb200_statistic_image(const float *src, float *dst, size_t width, size_t height, int channels, int type,
    size_t window_width, size_t window_height);
MB200_API int mb200_rotational_blur_image(const float *src, float *dst, size_t width, size_t height, int channels,
    double angle);
MB200_API int mb200_bilateral_blur_image(const float *src, float *dst, size_t width, size_t height, int channels,
    size_t window_width, size_t window_height, double intensity_sigma, double spatial_sigma);
MB200_API int mb200_adaptive_blur_image(const float *src, float *dst, size_t width, size_t height, int channels,
    double radius, double sigma);
MB200_API int mb200_adaptive_sharpen_image(const float *src, float *dst, size_t width, size_t height, int channels,
    double radius, double sigma);
MB200_API int mb200_selective_blur_image(const float *src, float *dst, size_t width, size_t height, int channels,
    double radius, double sigma, double threshold);
MB200_API int mb200_despeckle_image(const float *src, float *dst, size_t width, size_t height, int channels);
MB200_API int mb200_local_contrast_image(const float *src, float *dst, size_t width, size_t height, int channels,
    double radius, double strength);
MB200_API int mb200_wavelet_denoise_image(const float *src, float *dst, size_t width, size_t height, int channels,
    double threshold, double softness);
MB200_API int mb200_equalize_image(float *buf, size_t width, size_t height, int channels, int sync_channels);
MB200_API int mb200_emboss_image(const float *src, float *dst, size_t width, size_t height, int channels,
    double radius, double sigma);
MB200_API int mb200_resize_image_ex(const float *src, size_t width, size_t height, int channels, float *dst,
                                   size_t out_width, size_t out_height, int filter, const mb200_filter_options *options);
MB200_API int mb200_resize_image(const float *src, size_t width, size_t height, int channels,
    float *dst, size_t out_width, size_t out_height, int filter);
MB200_API int mb200_sample_image(const float *src, size_t width, size_t height, int channels,
    float *dst, size_t out_width, size_t out_height);
MB200_API int mb200_scale_image(const float *src, size_t width, size_t height, int channels,
    float *dst, size_t out_width, size_t out_height);
MB200_API int mb200_thumbnail_image(const float *src, size_t width, size_t height, int channels,
    float *dst, size_t columns, size_t rows, int filter);
MB200_API int mb200_transform_colorspace(float *buf, size_t width, size_t height, int channels,
    int from_colorspace, int to_colorspace);
MB200_API int mb200_transform_colorspace_ex(float *buf, size_t width, size_t height, int channels,
    int from_colorspace, int to_colorspace, const mb200_colorspace_options *options);
MB200_API int mb200_transform_colorspace_layout(const float *src, int src_channels, float *dst, int dst_channels,
    size_t width, size_t height, int from_colorspace, int to_colorspace, const mb200_colorspace_options *options);
MB200_API int mb200_bilevel_image(float *buf, size_t width, size_t height, int channels, double threshold);
MB200_API int mb200_black_threshold_image(float *buf, size_t width, size_t height, int channels,
    int colorspace, const char *thresholds);
MB200_API int mb200_white_threshold_image(float *buf, size_t width, size_t height, int channels,
    int colorspace, const char *thresholds);
MB200_API int mb200_clamp_image(float *buf, size_t width, size_t height, int channels);
MB200_API int mb200_adaptive_threshold_image(const float *src, float *dst, size_t width, size_t height, int channels,
    size_t window_width, size_t window_height, double bias, unsigned update_mask);
MB200_API int mb200_auto_threshold_image(float *buf, size_t width, size_t height, int channels, int method,
    double *threshold_percent);
MB200_API int mb200_range_threshold_image(float *buf, size_t width, size_t height, int channels, double low_black,
    double low_white, double high_white, double high_black, int per_channel, unsigned update_mask);
MB200_API int mb200_perceptible_image(float *buf, size_t width, size_t height, int channels, double epsilon,
    unsigned update_mask);
MB200_API int mb200_contrast_image(float *buf, size_t width, size_t height, int channels, int sharpen);
MB200_API int mb200_modulate_image(float *buf, size_t width, size_t height, int channels, double percent_brightness,
    double percent_saturation, double percent_hue, int colorspace, int illuminant);
MB200_API int mb200_grayscale_image(float *buf, size_t width, size_t height, int channels, int method,
    int image_colorspace);
MB200_API int mb200_function_image(float *buf, size_t width, size_t height, int channels, int function,
    size_t number_parameters, const double *parameters, unsigned update_mask);
MB200_API int mb200_contrast_stretch_image(float *buf, size_t width, size_t height, int channels, double black_point,
    double white_point, int per_channel, unsigned update_mask, float *black, float *white);
MB200_API int mb200_linear_stretch_image(float *buf, size_t width, size_t height, int channels, double black_point,
    double white_point, unsigned update_mask, double *black_bin, double *white_bin);
MB200_API int mb200_level_image(float *buf, size_t width, size_t height, int channels, double black_point,
    double white_point, double gamma, unsigned update_mask);
MB200_API int mb200_levelize_image(float *buf, size_t width, size_t height, int channels, double black_point,
    double white_point, double gamma, unsigned update_mask);
MB200_API int mb200_minmax_stretch_image(float *buf, size_t width, size_t height, int channels, double black,
    double white, double gamma, int per_channel, unsigned update_mask);
MB200_API int mb200_gamma_image(float *buf, size_t width, size_t height, int channels, double gamma,
    unsigned update_mask);
MB200_API int mb200_identify_gray(const float *buf, size_t width, size_t height, int channels, int *type);

#if defined(__cplusplus)
}
#endif
#endif /* MAGICK_B200_H */
