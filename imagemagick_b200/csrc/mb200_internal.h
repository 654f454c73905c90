// mb200_internal.h -- shared declarations inside libmagickb200 (not installed).
#pragma once

#include "../../include/magick_b200.h"

#include <cstddef>
#include <cstdint>
#include <memory>

struct CUmemPoolHandle_st;      // cudaMemPool_t == CUmemPoolHandle_st * (driver_types.h)

// resize_filter.cpp: the source sample a Copy-trait channel takes for every output of one axis (resize.c:3697-3707)
extern "C" int mb200_resize_nearest(int filter, size_t in_n, size_t out_n, double factor, long *nearest);

namespace mb200 {

// ---- error plumbing (runtime.cu) -------------------------------------------
int fail(int code, const char *fmt, ...);       // records thread-local message, returns code
int cuda_fail(int cuda_error, const char *what); // wraps a cudaError_t
void count_launch(unsigned n = 1);

// ---- run-time options (runtime.cu, DESIGN §10) ---------------------------------
// Initialised from the environment (an invalid value falls back to the default), settable with
// mb200_set_option("<name>").  Callers take a snapshot per call.
struct TuningKnobs {
  int mma_strip, mma_minb, mma_l2pf, conv_mma, mma_wide;              // conv_mma.cu
  int pair, pair_async, pair_async_col, col_rot, row_pair_rot, row_rot;   // conv1d.cu
  int resize_tma, resize_chunk, resize_slots, resize_strip;           // resize_stream.cu
  // switches (0 / 1) that force the generic paths, or opt in to a slower one, in api.cu
  int no_rank1, no_morph_stream, no_resize_stream, resize_regular_h, no_fused_unsharp;
  int resize_fused, no_resize_fused;                                   // force the fused / the two-pass ResizeImage
  int conv2d_rows;                                                     // morph2d.cu: 0 automatic, else 8 / 4 / 2
  int no_adaptive_tile;                                                // threshold.cu: force the direct family
};
TuningKnobs tuning_knobs();

// ---- per-family launch counters (runtime.cu): bumped where a family's kernel is launched, never on a decline -------
enum LaunchFamily {
  kConvMma, kConvMmaWide,                                              // conv_mma.cu (a wide launch counts in both)
  kConvPair, kConvPairAsync, kConvGeneric,                             // conv1d.cu
  kResizeVStream, kResizeHTma, kResizeHStream, kResizeFused,           // resize_stream.cu
  kResizeRegular, kResizeGather,                                       // resize.cu
  kConv2dDenseR8, kConv2dDenseR4, kConv2dDenseR2, kMorph2d, kMinmax2d, // morph2d.cu
  kMorphStream,                                                        // morph_stream.cu
  kMorphDirect,                                                        // morph_direct.cu
  kDistort,                                                            // distort.cu
  kGeometry,                                                           // geometry.cu
  kAdaptiveThresholdTile, kAdaptiveThresholdDirect,                    // threshold.cu
  kBoundingBox,                                                        // trim.cu
  kLaunchFamilies
};
void count_family(LaunchFamily family);

// ---- per-device state (runtime.cu) -----------------------------------------
struct DeviceState;
int ensure_device();                     // lazily initialises the current device; 0 or error
void *default_stream();                  // library-owned stream of the current device
int scratch(void **ptr, size_t bytes, int slot);   // grow-only device scratch buffers
int sm_count();
size_t l2_bytes();                       // L2 cache size of the current device (cudaDevAttrL2CacheSize)
// The library's PRIVATE stream-ordered memory pool of the current device (temporaries of the operators).  The host
// application's default pool is left alone; mb200_trim() gives the cached memory back.
::CUmemPoolHandle_st *temp_pool();

// ---- pixel-cache staging (cache.cu) ------------------------------------------
// copy_h2d returns once the host buffer has been consumed (the copy itself may still be in flight on `stream`);
// copy_d2h returns when the host buffer holds the data.  Pinned / registered / managed host memory is copied
// directly, pageable memory through the threaded pinned bounce ring.
int copy_h2d(void *dev, const void *host, size_t bytes, void *stream);
int copy_d2h(void *host, const void *dev, size_t bytes, void *stream);
struct StageRef {
  void *entry = nullptr;     // residency-registry entry when the host buffer is an attached pixel cache
  void *dev = nullptr;       // HBM copy to run the operator on
  void *host = nullptr;
  size_t bytes = 0;
  bool temporary = false;    // dev is a stream-ordered temporary (unattached host buffer)
};
int stage_input(const void *host, size_t bytes, void *stream, StageRef *out);
int stage_output(void *host, size_t bytes, void *stream, StageRef *out);
int finish_output(StageRef *ref, void *stream);
void release_stage(StageRef *ref, void *stream);

// ---- kernel helpers (kernel_info.cpp) --------------------------------------
void rotate_kernel_info(mb200_kernel_info *k, double angle);
struct KernelInfoFree {
  void operator()(mb200_kernel_info *k) const { mb200_destroy_kernel_info(k); }
};
using KernelList = std::unique_ptr<mb200_kernel_info, KernelInfoFree>;     // owns a whole kernel list
// BlurImage's kernel list "blur:RxS;blur:RxS+90" (effect.c:788); null when out of memory
KernelList blur_kernel_pair(double radius, double sigma);

// ---- channel traits (pixel.c:6356-6381) ------------------------------------
inline bool has_alpha(int channels) { return channels == 2 || channels == 4; }

// ---- device launchers -------------------------------------------------------
// All take device pointers and a cudaStream_t (as void*).  Return 0 / MB200_E*.

// conv1d.cu: one 1-D convolution pass (width-1 or height-1 kernel) with the
// reference's edge clamp, reflected taps and alpha blending.  taps[] is in window
// order (tap t multiplies the source sample at offset t - origin_offset).
// axis 0 = along x (row path, morphology.c:2815), axis 1 = along y (column path :2654).
// d_changed: device counter (may be null) incremented per changed channel value.
// epilogue: UnsharpMaskImage's point pass (effect.c:4358-4364) fused into the output stage when the RGBA pair kernels
// run the pass (*epilogue_fused tells; otherwise the caller runs launch_unsharp_combine afterwards).
struct UnsharpEpilogue { const float *source; double gain, quantum_threshold; };
int launch_conv1d(const float *src, float *dst, size_t width, size_t height, int channels,
                  int axis, const double *taps_window_order, int ntaps, int origin_offset,
                  double bias, double gamma_scale, unsigned long long *d_changed, void *stream,
                  int io = 0,    // io: 0 float->float, 1 float->raw double sums, 2 raw double sums->float (RGBA only)
                  const UnsharpEpilogue *epilogue = nullptr, bool *epilogue_fused = nullptr);

// conv_mma.cu: the same pass on the FP64 matrix path (mma.sync m8n8k4) for RGBA images, bias 0, <= 33 taps; src / dst are
// float4 pixels (io 0), double4 sums out (io 1) or in (io 2).  MB200_EUNSUPPORTED => use launch_conv1d's DFMA kernels.
int launch_conv_mma(const void *src, void *dst, size_t width, size_t height, int axis, const double *taps_window_order,
                    int ntaps, int origin_offset, void *stream, int io, const UnsharpEpilogue *epilogue,
                    bool *epilogue_fused);

// conv2d.cu: general 2-D convolution / erode / dilate (MorphologyPrimitive row path)
int launch_morph2d(const float *src, float *dst, size_t width, size_t height, int channels,
                   int method, const double *kernel_window_order, int kw, int kh, int ox, int oy,
                   double bias, double gamma_scale, unsigned long long *d_changed, void *stream);

// morph_stream.cu: erode / dilate for the built-in structuring elements, register streaming
// (MB200_EUNSUPPORTED => shape not in the table; use launch_morph2d)
int launch_morph_stream(const float *src, float *dst, size_t width, size_t height, int channels, int method,
                        const double *kernel_window_order, int kw, int kh, int ox, int oy, void *stream);

// morph_direct.cu: MorphologyApply's Distance / Voronoi branch (the two sequential sweeps of MorphologyPrimitiveDirect
// and Voronoi's alpha epilogue).  The check runs on the host before anything is allocated (MB200_EINVAL: another method,
// no kernel, an origin outside it; MB200_EUNSUPPORTED: Voronoi without alpha, a kernel too large for the wavefront);
// the launcher takes a temporary of the image's size for the forward pass.
int morphology_direct_check(int channels, int method, const mb200_kernel_info *kernel);
int launch_morphology_direct(const float *src, float *tmp, float *dst, size_t width, size_t height, int channels,
                             int method, const mb200_kernel_info *kernel, void *stream);

// distort.cu: DistortImage's sampling loop for a plan of distort_plan.cpp.  The check runs on the host before anything
// is touched (MB200_EINVAL / MB200_EUNSUPPORTED as documented at mb200_distort_image_dev); the launch is one kernel.
int distort_check(size_t width, size_t height, int channels, const mb200_distort_params *plan,
                  const mb200_resample_options *options);
int launch_distort(const float *src, size_t width, size_t height, int channels, float *dst,
                   const mb200_distort_params *plan, const mb200_resample_options *options, void *stream);

// geometry.cu: the orientation and crop operators for a plan of geometry_plan.cpp.  The check runs on the host before
// anything is touched (MB200_EINVAL: a plan that does not fit the source); the launch is one kernel.
int geometry_check(size_t width, size_t height, int channels, const mb200_geometry_params *plan);
int launch_geometry(const float *src, size_t width, size_t height, int channels, float *dst,
                    const mb200_geometry_params *plan, void *stream);

// trim.cu: GetImageBoundingBox's scan into d_rows (height x 4 words, the format of mb200_bounding_box_from_rows).  The
// check runs on the host before anything is touched; the launch is one memset and one kernel.
int bounding_box_check(size_t width, size_t height, int channels, const mb200_trim_options *options);
int launch_bounding_box(const float *src, size_t width, size_t height, int channels, const mb200_trim_options *options,
                        unsigned *d_rows, void *stream);

// ---- resize axis tables (resize_tables.cpp) ---------------------------------
// One axis of ResizeImage, planned on the host and resident on one device: the reference's contribution lists
// (tap-major), and what the specialised kernels need on top of them.
#define MB200_RESIZE_MAX_SEGMENTS 8
struct ResizeAxis {
  int device = -1, filter = 0;
  mb200_filter_options options{};     // expert settings the table was built with (all zero: none)
  size_t in_n = 0, out_n = 0;
  long taps = 0;
  // max_span: widest source span of any aligned block of 32 outputs (tile width of the tiled horizontal kernel)
  int max_span = 0, reg_stride = 0, reg_taps = 0;
  int *d_start = nullptr, *d_count = nullptr;
  double *d_weights = nullptr;
  double *d_wreg = nullptr;           // [out_n][reg_taps] when the interior is regular (integer-ratio reduction)
  // streaming kernels (resize_stream.cu): runs of outputs with bit-identical weights, and the
  // complement (borders, short runs) that stays with the gather kernels
  int nseg = 0, seg_o[MB200_RESIZE_MAX_SEGMENTS], seg_n[MB200_RESIZE_MAX_SEGMENTS], seg_src[MB200_RESIZE_MAX_SEGMENTS];
  double *d_wsets = nullptr;
  int nborder = 0;
  int *d_border = nullptr;
  // fused V+H kernel (resize_stream.cu): the runs cut into tiles of tile_w (this axis used as x) / tile_h (as y) outputs
  int *d_tiles_x = nullptr, *d_tiles_y = nullptr;
  int ntiles_x = 0, ntiles_y = 0;
  unsigned char *d_is_border = nullptr;       // [out_n]: output lies outside the runs
  ResizeAxis() = default;
  ResizeAxis(const ResizeAxis &) = delete;
  ResizeAxis &operator=(const ResizeAxis &) = delete;
  ~ResizeAxis();              // frees on the owning device; cudaFree waits for launches that still read the buffers
};
// The tables of (current device, filter, options, in_n, out_n), from a bounded cache shared by all threads.  The
// returned reference keeps the tables alive while the caller's launches are queued, even if they are evicted meanwhile.
int resize_axis_tables(int filter, const mb200_filter_options *options, size_t in_n, size_t out_n, double factor,
                       std::shared_ptr<const ResizeAxis> *out);

// resize.cu: one axis of ResizeImage on the gather kernels; `regular` allows the regular-stride kernels (when the
// axis has them).
int launch_resize_axis(const float *src, size_t width, size_t height, int channels, float *dst, int axis,
                       const ResizeAxis &t, bool regular, void *stream);

// resize_stream.cu: streaming kernels for the runs of outputs with bit-identical weights (integer-ratio
// reductions, RGBA); extra CTAs of the same launch gather the outputs outside the runs.
int launch_resize_stream(const float *src, size_t width, size_t height, float *dst, int axis, const ResizeAxis &t,
                         void *stream);

// Fused vertical + horizontal pass for equal integer reductions on both axes (RGBA): tile lists of both axes' runs,
// the two-pass path's contribution / border lists for the outputs outside the runs.
void resize_fused_tile(int stride, int taps, int *tile_w, int *tile_h);
int launch_resize_fused(const float *src, size_t width, size_t height, float *dst, const ResizeAxis &x,
                        const ResizeAxis &y, void *stream);

// colorspace.cu
int launch_colorspace(float *buf, size_t npixels, int channels, int from, int to, const mb200_colorspace_options *options,
                      void *stream);
// whether launch_colorspace has a leg between `colorspace` and sRGB (sRGB itself included)
bool colorspace_served(int colorspace);

// layout.cu: TransformImageColorspace to / from GRAY, LinearGRAY and CMYK, out of place (src is never written); the
// channel counts follow mb200_colorspace_channels.  Every decline is reported before anything is launched.
int colorspace_layout_check(const void *src, int src_channels, const void *dst, int dst_channels, size_t width,
                            size_t height, int from, int to, const mb200_colorspace_options *options);
int launch_colorspace_layout(const float *src, int src_channels, float *dst, int dst_channels, size_t npixels, int from,
                             int to, const mb200_colorspace_options *options, void *stream);

// hexcone.cu: HCL, HCLp, HSB, HSI, HSL, HSV, HWB (one leg: sRGB -> space or space -> sRGB), in place
bool is_hexcone_colorspace(int cs);
int launch_hexcone_leg(float *buf, size_t npixels, int channels, int space, bool forward, void *stream);

// pointwise.cu
int launch_unsharp_combine(const float *src, float *blur_inout, size_t n, double gain,
                           double quantum_threshold, void *stream);

// Copy-trait channels (a `-channel` selection): dst[c] = src[c] for the channels NOT in update_mask; the resize form takes
// the nearest source sample of each axis (resize.c:3697-3707)
int launch_restore_channels(float *dst, const float *src, size_t npixels, int channels, unsigned update_mask, void *stream);
int launch_resize_copy_channels(float *dst, const float *src, size_t w, size_t ow, size_t oh, int channels, const int *d_nearest_x,
                                const int *d_nearest_y, unsigned update_mask, void *stream);

// CompositeImage(canvas, source, DifferenceCompositeOp) for same-size images (Edge/TopHat/BottomHat), in place on canvas
int launch_composite_difference(float *canvas, const float *source, size_t npixels, int channels, void *stream);
// ... LightenCompositeOp: the union of the results of a HitAndMiss kernel list (morphology.c:3722, :4044-4046)
int launch_composite_lighten(float *canvas, const float *source, size_t npixels, int channels, void *stream);

// MotionBlurImage (effect.c:2347): taps + integer offsets from the host, gather along the blur direction
int launch_motion_blur(const float *src, float *dst, size_t w, size_t h, int channels, const double *taps, const long *ox,
                       const long *oy, int width, void *stream);

// stencils.cu: StatisticImage (statistic.c:2918), RotationalBlurImage (effect.c:3129), BilateralBlurImage (effect.c:821)
int launch_statistic(const float *src, float *dst, size_t w, size_t h, int channels, int type, size_t width, size_t height,
                     void *stream);
int launch_rotational_blur(const float *src, float *dst, size_t w, size_t h, int channels, double angle, void *stream);
int launch_bilateral_blur(const float *src, float *dst, size_t w, size_t h, int channels, size_t width, size_t height,
                          double intensity_sigma, double spatial_sigma, void *stream);
// AdaptiveBlurImage (effect.c:128) / AdaptiveSharpenImage (:447): edge map + per-pixel kernel size, bit exact
int launch_adaptive(const float *src, float *dst, size_t w, size_t h, int channels, double radius, double sigma, int sharpen,
                    void *stream);
// SelectiveBlurImage (effect.c:3406)
int launch_selective_blur(const float *src, float *dst, size_t w, size_t h, int channels, double radius, double sigma,
                          double threshold, void *stream);

// hooks.cu: DespeckleImage (effect.c:1308), LocalContrastImage (effect.c:2013), WaveletDenoiseImage
// (visual-effects.c:3515), bit exact.  The temporaries are the caller's: despeckle `tmp` one image; local contrast `luma`
// and `inter` one float plane each; wavelet `planes` 3 * (channels >= 3 ? 3 : 1) float planes.  The *_supported checks
// are the declines (MB200_EUNSUPPORTED where the reference reads memory it never wrote), run before anything is allocated.
int launch_despeckle(const float *src, float *dst, float *tmp, size_t w, size_t h, int channels, void *stream);
int local_contrast_supported(size_t w, size_t h, double radius);
int launch_local_contrast(const float *src, float *dst, float *luma, float *inter, size_t w, size_t h, int channels,
                          double radius, double strength, void *stream);
int wavelet_denoise_supported(size_t w, size_t h);
int launch_wavelet_denoise(const float *src, float *dst, float *planes, size_t w, size_t h, int channels, double threshold,
                           double softness, void *stream);

// ScaleImage (resize.c:4106): CSR contribution lists of both axes (mb200_scale_contributions), bit exact
int launch_scale(const float *src, size_t w, size_t h, int channels, float *dst, size_t ow, size_t oh, const int *d_xoff,
                 const int *d_xidx, const double *d_xwt, const int *d_yoff, const int *d_yidx, const double *d_ywt, void *stream);

// SampleImage (resize.c:3907): nearest-sample gather, bit exact
int launch_sample(const float *src, size_t w, size_t h, int channels, float *dst, size_t ow, size_t oh, void *stream);

// equalize.cu: EqualizeImage (enhance.c:2040) in place; sync_channels = the channel mask carries SyncChannels (the
// default): one intensity-driven histogram for all channels.  Synchronises the stream (host step between the kernels).
int launch_equalize(float *buf, size_t npixels, int channels, int sync_channels, void *stream);

// enhance.cu: ContrastImage (enhance.c:1370), ModulateImage (:3461), GrayscaleImage (:2474; channel 0 only) and
// FunctionImage (statistic.c:1064) in place, arguments already checked
int launch_contrast(float *buf, size_t npixels, int channels, bool sharpen, void *stream);
int launch_modulate(float *buf, size_t npixels, int channels, double percent_brightness, double percent_saturation,
                    double percent_hue, int colorspace, int illuminant, void *stream);
int launch_grayscale(float *buf, size_t npixels, int channels, int method, int image_colorspace, void *stream);
int launch_function(float *buf, size_t npixels, int channels, int function, size_t n, const double *params,
                    unsigned update_mask, void *stream);

// level.cu: the level and stretch operators of enhance.c in place, arguments already checked.  contrast / linear stretch
// read the histogram back (synchronise the stream); identify_gray reads one flag word back.
int launch_level(float *buf, size_t npixels, int channels, double black, double white, double gamma, unsigned update_mask,
                 bool levelize, void *stream);
int launch_minmax_stretch(float *buf, size_t width, size_t height, int channels, double black, double white, double gamma,
                          bool per_channel, unsigned update_mask, void *stream);
int launch_contrast_stretch(float *buf, size_t width, size_t height, int channels, double black_point, double white_point,
                            bool per_channel, unsigned update_mask, float *black, float *white, void *stream);
int launch_linear_stretch(float *buf, size_t width, size_t height, int channels, double black_point, double white_point,
                          unsigned update_mask, double *black_bin, double *white_bin, void *stream);
int launch_gamma(float *buf, size_t npixels, int channels, double gamma, unsigned update_mask, void *stream);
int launch_identify_gray(const float *buf, size_t npixels, int channels, int *type, void *stream);

// threshold.c point operators in place; op: 0 bilevel (t[0]), 1 black, 2 white (t = r,g,b,a), 3 clamp (every channel);
// 4 range (t = low black, low white, high white, high black, QuantumRange*PerceptibleReciprocal(lw-lb),
// QuantumRange*PerceptibleReciprocal(hb-hw); per_channel: the sample instead of the intensity), 5 perceptible (t[0] =
// epsilon) on the channels of update_mask
int launch_threshold(float *buf, size_t npixels, int channels, int op, const double *thresholds, void *stream,
                     unsigned update_mask = 0xfu, bool per_channel = false);
// AutoThresholdImage's histogram (threshold.c:717-735): 256 bins of ScaleQuantumToChar(ClampToQuantum(intensity)), read
// back (synchronises the stream)
int auto_threshold_histogram(const float *buf, size_t npixels, int channels, unsigned counts[256], void *stream);
// threshold.cu: AutoThresholdImage's threshold (percent) of `method` from that histogram, in the reference's arithmetic
double auto_threshold_percent(const unsigned counts[256], int method);
// threshold.cu: AdaptiveThresholdImage (threshold.c:182) out of place on the channels of update_mask (the others copy)
int launch_adaptive_threshold(const float *src, float *dst, size_t width, size_t height, int channels, size_t w, size_t h,
                              double bias, unsigned update_mask, void *stream);

}  // namespace mb200
