// pointwise.cu -- per-sample epilogues.
//
// unsharp combine: the point pass of UnsharpMaskImage (MagickCore/effect.c:4310-4384):
//   d = p - blur;  out = (|2d| < QuantumRange*threshold) ? p : p + gain*d     (double -> float)
// applied to every channel (all carry the Update trait on the accelerated path).
//
// threshold point operators of MagickCore/threshold.c (see threshold_kernel below).
#include "mb200_internal.h"
#include "conv_common.cuh"

#include <cuda_runtime.h>

namespace mb200 {
namespace {

__global__ void __launch_bounds__(256) unsharp_kernel(const float4 *__restrict__ src, float4 *__restrict__ blur,
                                                      size_t n4, double gain, double qthreshold) {
  const size_t i = static_cast<size_t>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= n4) return;
  const float4 p = __ldg(src + i);
  float4 b = blur[i];
  // unfused double operations in the reference's order (conv_common.cuh): `p + gain * d` contracted into an FMA differs from
  // the reference's mul + add by one float ULP in ~0.2 % of the samples when gain is not a short binary fraction
  auto one = [&](float pv, float bv) -> float { return unsharp_point(pv, bv, gain, qthreshold); };
  b.x = one(p.x, b.x); b.y = one(p.y, b.y); b.z = one(p.z, b.z); b.w = one(p.w, b.w);
  blur[i] = b;
}

__global__ void __launch_bounds__(256) unsharp_tail_kernel(const float *__restrict__ src, float *__restrict__ blur,
                                                           size_t begin, size_t n, double gain, double qthreshold) {
  const size_t i = begin + static_cast<size_t>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= n) return;
  blur[i] = unsharp_point(src[i], blur[i], gain, qthreshold);
}

// threshold.c point operators, in place (BilevelImage :805, BlackThresholdImage :927, WhiteThresholdImage
// :2518, ClampImage :1087).  Every channel (alpha included) is compared through the pixel's intensity
// (pixel.c:2356, Rec709Luma on an sRGB / gray image), evaluated exactly as the reference does: three
// products summed left to right in double with no contraction, so the comparison -- and therefore the
// result -- is bit-identical.  op: 0 bilevel, 1 black, 2 white, 3 clamp, on every channel; 4 RangeThresholdImage
// (:2377) and 5 PerceptibleImage (:2092) on the channels of `update`.
struct ThresholdArgs {
  double t[6];     // bilevel, perceptible: t[0]; black / white: red, green, blue, alpha; range: see launch_threshold
  int op;
  unsigned update;
  bool per_channel;
};

template <int CH>
__global__ void __launch_bounds__(256) threshold_kernel(float *__restrict__ buf, size_t npixels, const ThresholdArgs a) {
  const size_t i = static_cast<size_t>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= npixels) return;
  float v[CH];
  if (CH == 4) {
    const float4 t = reinterpret_cast<const float4 *>(buf)[i];
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[CH - 1] = t.w;
  } else {
#pragma unroll
    for (int c = 0; c < CH; ++c) v[c] = buf[i * CH + c];
  }
  constexpr double kQR = 65535.0;
  if (a.op == 3) {                                     // ClampPixel (pixel-accessor.h:35-46, HDRI)
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const double p = static_cast<double>(v[c]);
      if (p < 0.0) v[c] = 0.0f;
      else if (p >= kQR) v[c] = 65535.0f;
    }
  } else if (a.op == 5) {                              // PerceptibleThreshold (:2080)
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      if (!((a.update >> c) & 1u)) continue;
      const double q = static_cast<double>(v[c]), sign = q < 0.0 ? -1.0 : 1.0;
      if (!(__dmul_rn(sign, q) >= a.t[0])) v[c] = static_cast<float>(__dmul_rn(sign, a.t[0]));
    }
  } else {
    const double red = static_cast<double>(v[0]);
    double pixel = red;
    if (CH > 1) {
      const double green = CH >= 3 ? static_cast<double>(v[1]) : red;
      const double blue = CH >= 3 ? static_cast<double>(v[CH >= 3 ? 2 : 0]) : red;
      pixel = __dadd_rn(__dadd_rn(__dmul_rn(0.212656, red), __dmul_rn(0.715158, green)), __dmul_rn(0.072186, blue));
    }
    if (a.op == 4) {                                   // :2446-2464, ClampToQuantum = the float cast (HDRI)
#pragma unroll
      for (int c = 0; c < CH; ++c) {
        if (!((a.update >> c) & 1u)) continue;
        if (a.per_channel) pixel = static_cast<double>(v[c]);
        if (pixel < a.t[0]) v[c] = 0.0f;
        else if (pixel >= a.t[0] && pixel < a.t[1]) v[c] = static_cast<float>(__dmul_rn(a.t[4], __dsub_rn(pixel, a.t[0])));
        else if (pixel >= a.t[1] && pixel <= a.t[2]) v[c] = 65535.0f;
        else if (pixel > a.t[2] && pixel <= a.t[3]) v[c] = static_cast<float>(__dmul_rn(a.t[5], __dsub_rn(a.t[3], pixel)));
        else v[c] = 0.0f;
      }
    } else {
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const bool is_alpha = (CH == 2 || CH == 4) && c == CH - 1;
      const double t = a.op == 0 ? a.t[0] : (is_alpha ? a.t[3] : a.t[c < 3 ? c : 0]);
      if (a.op == 0) v[c] = pixel <= t ? 0.0f : 65535.0f;
      else if (a.op == 1) { if (pixel < t) v[c] = 0.0f; }
      else { if (pixel > t) v[c] = 65535.0f; }
    }
    }
  }
  if (CH == 4) reinterpret_cast<float4 *>(buf)[i] = make_float4(v[0], v[1], v[2], v[CH - 1]);
  else {
#pragma unroll
    for (int c = 0; c < CH; ++c) buf[i * CH + c] = v[c];
  }
}

// CompositeImage(canvas, source, DifferenceCompositeOp, clip_to_self, 0, 0) as MorphologyApply calls it for
// the Edge / TopHat / BottomHat methods (morphology.c:3995-4012; composite.c:2377-3562 with the default
// compose:sync / compose:clamp): same-size images, default channel traits.  Evaluated in the reference's
// operation order with unfused double arithmetic => bit exact.
//   Sa, Da = QS*alpha (1 without alpha);  alpha = RoundToUnity(Sa+Da-Sa*Da);  gamma = PerceptibleReciprocal(alpha)
//   colour: QR*gamma*(Sca+Dca-2*min(Sca*Da,Dca*Sa)), Sca = QS*Sa*Sc, Dca = QS*Da*Dc;  alpha: QR*|Sa-Da|;  ClampPixel.
// OP 1 = LightenCompositeOp, the union MorphologyApply forms over a HitAndMiss kernel list (morphology.c:3722, :4044;
// composite.c:3110-3124): colour (Sca*Da > Dca*Sa) ? QR*(Sca+Dca*(1-Sa)) : QR*(Dca+Sca*(1-Da)), alpha QR*alpha.
template <int CH, int OP>
__global__ void __launch_bounds__(256) difference_kernel(float *__restrict__ canvas, const float *__restrict__ source,
                                                         size_t npixels) {
  const size_t i = static_cast<size_t>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= npixels) return;
  constexpr bool kAlpha = (CH == 2 || CH == 4);
  constexpr double kQR = 65535.0, kQS = 1.0 / 65535.0, kEps = 1.0e-12;
  float q[CH], p[CH];
  if (CH == 4) {
    const float4 a = reinterpret_cast<const float4 *>(canvas)[i], b = __ldg(reinterpret_cast<const float4 *>(source) + i);
    q[0] = a.x; q[1] = a.y; q[2] = a.z; q[CH - 1] = a.w;
    p[0] = b.x; p[1] = b.y; p[2] = b.z; p[CH - 1] = b.w;
  } else {
#pragma unroll
    for (int c = 0; c < CH; ++c) { q[c] = canvas[i * CH + c]; p[c] = __ldg(source + i * CH + c); }
  }
  const double Sa = __dmul_rn(kQS, kAlpha ? static_cast<double>(p[CH - 1]) : 65535.0);
  const double Da = __dmul_rn(kQS, kAlpha ? static_cast<double>(q[CH - 1]) : 65535.0);
  double alpha = __dsub_rn(__dadd_rn(Sa, Da), __dmul_rn(Sa, Da));
  alpha = alpha < 0.0 ? 0.0 : (alpha > 1.0 ? 1.0 : alpha);
  const double sign = alpha < 0.0 ? -1.0 : 1.0;
  const double gamma = __dmul_rn(sign, alpha) >= kEps ? __ddiv_rn(1.0, alpha) : __ddiv_rn(sign, kEps);
  float out[CH];
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    double pixel;
    if (kAlpha && c == CH - 1) pixel = OP == 1 ? __dmul_rn(kQR, alpha) : __dmul_rn(kQR, fabs(__dsub_rn(Sa, Da)));
    else {
      const double Sca = __dmul_rn(__dmul_rn(kQS, Sa), static_cast<double>(p[c]));
      const double Dca = __dmul_rn(__dmul_rn(kQS, Da), static_cast<double>(q[c]));
      const double a = __dmul_rn(Sca, Da), b = __dmul_rn(Dca, Sa);
      if (OP == 1)
        pixel = a > b ? __dmul_rn(kQR, __dadd_rn(Sca, __dmul_rn(Dca, __dsub_rn(1.0, Sa))))
                      : __dmul_rn(kQR, __dadd_rn(Dca, __dmul_rn(Sca, __dsub_rn(1.0, Da))));
      else
        pixel = __dmul_rn(__dmul_rn(kQR, gamma), __dsub_rn(__dadd_rn(Sca, Dca), __dmul_rn(2.0, a < b ? a : b)));
    }
    out[c] = pixel < 0.0 ? 0.0f : (pixel >= kQR ? 65535.0f : static_cast<float>(pixel));
  }
  if (CH == 4) reinterpret_cast<float4 *>(canvas)[i] = make_float4(out[0], out[1], out[2], out[CH - 1]);
  else {
#pragma unroll
    for (int c = 0; c < CH; ++c) canvas[i * CH + c] = out[c];
  }
}

// SampleImage (MagickCore/resize.c:3907-4090): nearest-sample gather.  The source column / row of an output is
// (ssize_t) (((j + 0.5 - MagickEpsilon) * in_n) / out_n) in double (:3973, :3996) -- single IEEE operations, so the
// device evaluates the identical expression instead of reading offset tables.  Bit exact.
template <int CH>
__global__ void __launch_bounds__(256) sample_kernel(const float *__restrict__ src, float *__restrict__ dst, int w, int h,
                                                     int ow, int oh) {
  const int x = blockIdx.x * 256 + threadIdx.x;
  const int y = blockIdx.y;
  if (x >= ow) return;
  constexpr double kOffset = 0.5 - 1.0e-12;
  const long xo = static_cast<long>(__ddiv_rn(__dmul_rn(__dadd_rn(static_cast<double>(x), kOffset), static_cast<double>(w)),
                                               static_cast<double>(ow)));
  const long yo = static_cast<long>(__ddiv_rn(__dmul_rn(__dadd_rn(static_cast<double>(y), kOffset), static_cast<double>(h)),
                                               static_cast<double>(oh)));
  const float *p = src + (static_cast<size_t>(yo) * w + static_cast<size_t>(xo)) * CH;
  float *q = dst + (static_cast<size_t>(y) * ow + x) * CH;
  if (CH == 4) *reinterpret_cast<float4 *>(q) = __ldg(reinterpret_cast<const float4 *>(p));
  else {
#pragma unroll
    for (int c = 0; c < CH; ++c) q[c] = __ldg(p + c);
  }
}

// MotionBlurImage (MagickCore/effect.c:2347-2560): `width` taps of a one-sided Gaussian walked along the blur angle
// from every output pixel (integer offsets, edge-replicated source), alpha-weighted blend for the colour channels of
// images with alpha.  Host builds taps and offsets with the reference's arithmetic (effect.c:2316-2345, :2390-2398);
// the device accumulates in the reference's order with unfused double operations and an IEEE division, so the
// result is the reference's double value rounded once to float.
constexpr int kMaxMotionTaps = 129;
struct MotionArgs {
  double k[kMaxMotionTaps];
  short ox[kMaxMotionTaps], oy[kMaxMotionTaps];
  int width;
};

template <int CH>
__global__ void __launch_bounds__(128) motion_blur_kernel(const float *__restrict__ src, float *__restrict__ dst, int w,
                                                          int h, const MotionArgs a) {
  const int x = blockIdx.x * 128 + threadIdx.x;
  const int y = blockIdx.y;
  if (x >= w) return;
  constexpr bool kAlpha = (CH == 2 || CH == 4);
  constexpr double kQS = 1.0 / 65535.0, kEps = 1.0e-12;
  double pixel[CH], gamma = 0.0;
#pragma unroll
  for (int c = 0; c < CH; ++c) pixel[c] = 0.0;
  for (int j = 0; j < a.width; ++j) {
    const int xx = min(max(x + a.ox[j], 0), w - 1), yy = min(max(y + a.oy[j], 0), h - 1);
    const float *r = src + (static_cast<size_t>(yy) * w + xx) * CH;
    float v[CH];
    if (CH == 4) { const float4 t = __ldg(reinterpret_cast<const float4 *>(r)); v[0] = t.x; v[1] = t.y; v[2] = t.z; v[CH - 1] = t.w; }
    else {
#pragma unroll
      for (int c = 0; c < CH; ++c) v[c] = __ldg(r + c);
    }
    const double kj = a.k[j];
    if (kAlpha) {
      const double ka = __dmul_rn(kj, __dmul_rn(kQS, static_cast<double>(v[CH - 1])));       /* (*k)*alpha */
#pragma unroll
      for (int c = 0; c < CH - 1; ++c) pixel[c] = __dadd_rn(pixel[c], __dmul_rn(ka, static_cast<double>(v[c])));
      gamma = __dadd_rn(gamma, ka);
      pixel[CH - 1] = __dadd_rn(pixel[CH - 1], __dmul_rn(kj, static_cast<double>(v[CH - 1])));
    } else {
#pragma unroll
      for (int c = 0; c < CH; ++c) pixel[c] = __dadd_rn(pixel[c], __dmul_rn(kj, static_cast<double>(v[c])));
    }
  }
  float o[CH];
  if (kAlpha) {
    const double sign = gamma < 0.0 ? -1.0 : 1.0;
    const double g = __dmul_rn(sign, gamma) >= kEps ? __ddiv_rn(1.0, gamma) : __ddiv_rn(sign, kEps);
#pragma unroll
    for (int c = 0; c < CH - 1; ++c) o[c] = static_cast<float>(__dmul_rn(g, pixel[c]));
    o[CH - 1] = static_cast<float>(pixel[CH - 1]);
  } else {
#pragma unroll
    for (int c = 0; c < CH; ++c) o[c] = static_cast<float>(pixel[c]);
  }
  float *q = dst + (static_cast<size_t>(y) * w + x) * CH;
  if (CH == 4) *reinterpret_cast<float4 *>(q) = make_float4(o[0], o[1], o[2], o[CH - 1]);
  else {
#pragma unroll
    for (int c = 0; c < CH; ++c) q[c] = o[c];
  }
}

}  // namespace

int launch_motion_blur(const float *src, float *dst, size_t w, size_t h, int channels, const double *taps, const long *ox,
                       const long *oy, int width, void *stream) {
  if (width < 1 || width > kMaxMotionTaps) return fail(MB200_EUNSUPPORTED, "motion blur: %d taps (max %d)", width, kMaxMotionTaps);
  if (w > 0x3fffffffull || h > 65535ull) return fail(MB200_EUNSUPPORTED, "motion blur: image too large for this kernel");
  MotionArgs a{};
  a.width = width;
  for (int j = 0; j < width; ++j) {
    if (ox[j] < -32768 || ox[j] > 32767 || oy[j] < -32768 || oy[j] > 32767) return fail(MB200_EUNSUPPORTED, "motion blur: offset range");
    a.k[j] = taps[j]; a.ox[j] = static_cast<short>(ox[j]); a.oy[j] = static_cast<short>(oy[j]);
  }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  dim3 grid(static_cast<unsigned>((w + 127) / 128), static_cast<unsigned>(h));
  const int W = static_cast<int>(w), H = static_cast<int>(h);
  switch (channels) {
    case 1: motion_blur_kernel<1><<<grid, 128, 0, s>>>(src, dst, W, H, a); break;
    case 2: motion_blur_kernel<2><<<grid, 128, 0, s>>>(src, dst, W, H, a); break;
    case 3: motion_blur_kernel<3><<<grid, 128, 0, s>>>(src, dst, W, H, a); break;
    case 4:
      if (((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) != 0)
        return fail(MB200_EINVAL, "motion blur: RGBA buffers must be 16-byte aligned");
      motion_blur_kernel<4><<<grid, 128, 0, s>>>(src, dst, W, H, a);
      break;
    default: return fail(MB200_EINVAL, "motion blur: 1..4 channels");
  }
  count_launch();
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "motion blur launch");
  return MB200_OK;
}

int launch_sample(const float *src, size_t w, size_t h, int channels, float *dst, size_t ow, size_t oh, void *stream) {
  if (w > 0x3fffffffull || h > 0x3fffffffull || ow > 0x3fffffffull || oh > 65535ull * 1ull * 65535ull)
    return fail(MB200_EINVAL, "sample: image too large");
  if (oh > 65535) return fail(MB200_EUNSUPPORTED, "sample: more than 65535 output rows");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  dim3 grid(static_cast<unsigned>((ow + 255) / 256), static_cast<unsigned>(oh));
  const int W = static_cast<int>(w), H = static_cast<int>(h), OW = static_cast<int>(ow), OH = static_cast<int>(oh);
  switch (channels) {
    case 1: sample_kernel<1><<<grid, 256, 0, s>>>(src, dst, W, H, OW, OH); break;
    case 2: sample_kernel<2><<<grid, 256, 0, s>>>(src, dst, W, H, OW, OH); break;
    case 3: sample_kernel<3><<<grid, 256, 0, s>>>(src, dst, W, H, OW, OH); break;
    case 4:
      if (((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) != 0)
        return fail(MB200_EINVAL, "sample: RGBA buffers must be 16-byte aligned");
      sample_kernel<4><<<grid, 256, 0, s>>>(src, dst, W, H, OW, OH);
      break;
    default: return fail(MB200_EINVAL, "sample: 1..4 channels");
  }
  count_launch();
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "sample launch");
  return MB200_OK;
}

template <int OP>
int launch_composite(float *canvas, const float *source, size_t npixels, int channels, void *stream) {
  if (npixels == 0) return MB200_OK;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t blocks = (npixels + 255) / 256;
  if (blocks > 0x7fffffffull) return fail(MB200_EINVAL, "composite: image too large");
  const unsigned grid = static_cast<unsigned>(blocks);
  switch (channels) {
    case 1: difference_kernel<1, OP><<<grid, 256, 0, s>>>(canvas, source, npixels); break;
    case 2: difference_kernel<2, OP><<<grid, 256, 0, s>>>(canvas, source, npixels); break;
    case 3: difference_kernel<3, OP><<<grid, 256, 0, s>>>(canvas, source, npixels); break;
    case 4:
      if (((reinterpret_cast<uintptr_t>(canvas) | reinterpret_cast<uintptr_t>(source)) & 15) != 0)
        return fail(MB200_EINVAL, "composite: RGBA buffers must be 16-byte aligned");
      difference_kernel<4, OP><<<grid, 256, 0, s>>>(canvas, source, npixels);
      break;
    default: return fail(MB200_EINVAL, "composite: 1..4 channels");
  }
  count_launch();
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "composite launch");
  return MB200_OK;
}

int launch_composite_difference(float *canvas, const float *source, size_t npixels, int channels, void *stream) {
  return launch_composite<0>(canvas, source, npixels, channels, stream);
}
int launch_composite_lighten(float *canvas, const float *source, size_t npixels, int channels, void *stream) {
  return launch_composite<1>(canvas, source, npixels, channels, stream);
}

int launch_threshold(float *buf, size_t npixels, int channels, int op, const double *thresholds, void *stream,
                     unsigned update_mask, bool per_channel) {
  if (npixels == 0) return MB200_OK;
  ThresholdArgs a{};
  for (int k = 0; k < (op == 4 ? 6 : 4); ++k) a.t[k] = thresholds ? thresholds[k] : 0.0;
  a.op = op;
  a.update = update_mask;
  a.per_channel = per_channel;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t blocks = (npixels + 255) / 256;
  if (blocks > 0x7fffffffull) return fail(MB200_EINVAL, "threshold: image too large");
  const unsigned grid = static_cast<unsigned>(blocks);
  const bool aligned = (reinterpret_cast<uintptr_t>(buf) & 15) == 0;
  switch (channels) {
    case 1: threshold_kernel<1><<<grid, 256, 0, s>>>(buf, npixels, a); break;
    case 2: threshold_kernel<2><<<grid, 256, 0, s>>>(buf, npixels, a); break;
    case 3: threshold_kernel<3><<<grid, 256, 0, s>>>(buf, npixels, a); break;
    case 4:
      if (!aligned) return fail(MB200_EINVAL, "threshold: RGBA buffers must be 16-byte aligned");
      threshold_kernel<4><<<grid, 256, 0, s>>>(buf, npixels, a);
      break;
    default: return fail(MB200_EINVAL, "threshold: 1..4 channels");
  }
  count_launch();
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "threshold launch");
  return MB200_OK;
}

// Channels outside a `-channel` selection carry the Copy trait: every operator of the path hands them through from its
// source (morphology.c:2733-2737, effect.c:4346-4350; resize.c:3697-3707 takes the NEAREST source sample of each pass).
// The kernels compute all channels; these point passes put the Copy channels back.  update_mask bit c = channel c is updated.
namespace {
template <int CH>
__global__ void __launch_bounds__(256) restore_channels_kernel(float *__restrict__ dst, const float *__restrict__ src, size_t npixels,
                                                               unsigned update_mask) {
  const size_t i = static_cast<size_t>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= npixels) return;
#pragma unroll
  for (int c = 0; c < CH; ++c)
    if (!(update_mask >> c & 1u)) dst[i * CH + c] = __ldg(src + i * CH + c);
}

template <int CH>
__global__ void __launch_bounds__(256) resize_copy_channels_kernel(float *__restrict__ dst, const float *__restrict__ src, int w, int ow,
                                                                   int oh, const int *__restrict__ nearest_x,
                                                                   const int *__restrict__ nearest_y, unsigned update_mask) {
  const int x = blockIdx.x * 256 + threadIdx.x, y = blockIdx.y;
  if (x >= ow || y >= oh) return;
  const size_t s = (static_cast<size_t>(__ldg(nearest_y + y)) * w + __ldg(nearest_x + x)) * CH;
  const size_t d = (static_cast<size_t>(y) * ow + x) * CH;
#pragma unroll
  for (int c = 0; c < CH; ++c)
    if (!(update_mask >> c & 1u)) dst[d + c] = __ldg(src + s + c);
}
}  // namespace

int launch_restore_channels(float *dst, const float *src, size_t npixels, int channels, unsigned update_mask, void *stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t blocks = (npixels + 255) / 256;
  if (blocks == 0 || blocks > 0x7fffffffull) return fail(MB200_EINVAL, "restore channels: bad image size");
  const unsigned grid = static_cast<unsigned>(blocks);
  switch (channels) {
    case 1: restore_channels_kernel<1><<<grid, 256, 0, s>>>(dst, src, npixels, update_mask); break;
    case 2: restore_channels_kernel<2><<<grid, 256, 0, s>>>(dst, src, npixels, update_mask); break;
    case 3: restore_channels_kernel<3><<<grid, 256, 0, s>>>(dst, src, npixels, update_mask); break;
    case 4: restore_channels_kernel<4><<<grid, 256, 0, s>>>(dst, src, npixels, update_mask); break;
    default: return fail(MB200_EINVAL, "restore channels: 1..4 channels");
  }
  count_launch();
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? MB200_OK : cuda_fail(e, "restore channels launch");
}

int launch_resize_copy_channels(float *dst, const float *src, size_t w, size_t ow, size_t oh, int channels, const int *d_nearest_x,
                                const int *d_nearest_y, unsigned update_mask, void *stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (oh > 65535) return fail(MB200_EUNSUPPORTED, "resize copy channels: more than 65535 output rows");
  dim3 grid(static_cast<unsigned>((ow + 255) / 256), static_cast<unsigned>(oh));
  const int W = static_cast<int>(w), OW = static_cast<int>(ow), OH = static_cast<int>(oh);
  switch (channels) {
    case 1: resize_copy_channels_kernel<1><<<grid, 256, 0, s>>>(dst, src, W, OW, OH, d_nearest_x, d_nearest_y, update_mask); break;
    case 2: resize_copy_channels_kernel<2><<<grid, 256, 0, s>>>(dst, src, W, OW, OH, d_nearest_x, d_nearest_y, update_mask); break;
    case 3: resize_copy_channels_kernel<3><<<grid, 256, 0, s>>>(dst, src, W, OW, OH, d_nearest_x, d_nearest_y, update_mask); break;
    case 4: resize_copy_channels_kernel<4><<<grid, 256, 0, s>>>(dst, src, W, OW, OH, d_nearest_x, d_nearest_y, update_mask); break;
    default: return fail(MB200_EINVAL, "resize copy channels: 1..4 channels");
  }
  count_launch();
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? MB200_OK : cuda_fail(e, "resize copy channels launch");
}

// ScaleImage (resize.c:4106): thread = output pixel; out = fold over its column list of (fold over its row list of the
// premultiplied source samples), both folds as acc = acc + w * v with unfused double operations starting from 0 -- the
// reference's y_vector / pixel accumulation -- then the alpha division of :4482-4503.  Bit exact.
namespace {
struct ScaleArgs {
  const float *src;
  float *dst;
  int w, h, ow, oh;
  const int *xoff, *xidx, *yoff, *yidx;     // CSR lists of both axes (device)
  const double *xwt, *ywt;
};

template <int CH>
__global__ void __launch_bounds__(128) scale_kernel(const ScaleArgs a) {
  const int t = blockIdx.x * 128 + threadIdx.x, y = blockIdx.y;
  if (t >= a.ow) return;
  constexpr bool kAlpha = (CH == 2 || CH == 4);
  constexpr double kQS = 1.0 / 65535.0, kEps = 1.0e-12;
  const int x0 = __ldg(a.xoff + t), x1 = __ldg(a.xoff + t + 1), y0 = __ldg(a.yoff + y), y1 = __ldg(a.yoff + y + 1);
  double pixel[CH];
#pragma unroll
  for (int c = 0; c < CH; ++c) pixel[c] = 0.0;
  for (int j = x0; j < x1; ++j) {
    const int x = __ldg(a.xidx + j);
    double col[CH];
#pragma unroll
    for (int c = 0; c < CH; ++c) col[c] = 0.0;
    for (int k = y0; k < y1; ++k) {
      const float *p = a.src + (static_cast<size_t>(__ldg(a.yidx + k)) * a.w + x) * CH;
      const double wy = __ldg(a.ywt + k);
      float v[CH];
      if (CH == 4) { const float4 q = __ldg(reinterpret_cast<const float4 *>(p)); v[0] = q.x; v[1] = q.y; v[2] = q.z; v[CH - 1] = q.w; }
      else {
#pragma unroll
        for (int c = 0; c < CH; ++c) v[c] = __ldg(p + c);
      }
      const double alpha = kAlpha ? __dmul_rn(kQS, static_cast<double>(v[CH - 1])) : 1.0;
#pragma unroll
      for (int c = 0; c < CH; ++c) {
        const double xv = (kAlpha && c != CH - 1) ? __dmul_rn(alpha, static_cast<double>(v[c])) : static_cast<double>(v[c]);
        col[c] = __dadd_rn(col[c], __dmul_rn(wy, xv));
      }
    }
    const double wx = __ldg(a.xwt + j);
#pragma unroll
    for (int c = 0; c < CH; ++c) pixel[c] = __dadd_rn(pixel[c], __dmul_rn(wx, col[c]));
  }
  float o[CH];
  if (kAlpha) {
    const double g = __dmul_rn(kQS, pixel[CH - 1]);
    const double sign = g < 0.0 ? -1.0 : 1.0;
    const double r = __dmul_rn(sign, g) >= kEps ? __ddiv_rn(1.0, g) : __ddiv_rn(sign, kEps);
#pragma unroll
    for (int c = 0; c < CH - 1; ++c) o[c] = static_cast<float>(__dmul_rn(r, pixel[c]));
    o[CH - 1] = static_cast<float>(pixel[CH - 1]);
  } else {
#pragma unroll
    for (int c = 0; c < CH; ++c) o[c] = static_cast<float>(pixel[c]);
  }
  float *q = a.dst + (static_cast<size_t>(y) * a.ow + t) * CH;
  if (CH == 4) *reinterpret_cast<float4 *>(q) = make_float4(o[0], o[1], o[2], o[CH - 1]);
  else {
#pragma unroll
    for (int c = 0; c < CH; ++c) q[c] = o[c];
  }
}
}  // namespace

int launch_scale(const float *src, size_t w, size_t h, int channels, float *dst, size_t ow, size_t oh, const int *d_xoff,
                 const int *d_xidx, const double *d_xwt, const int *d_yoff, const int *d_yidx, const double *d_ywt, void *stream) {
  if (w > 0x3fffffffull || h > 0x3fffffffull || ow > 0x3fffffffull) return fail(MB200_EINVAL, "scale: image too large");
  if (oh > 65535) return fail(MB200_EUNSUPPORTED, "scale: more than 65535 output rows");
  if (channels == 4 && ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) != 0)
    return fail(MB200_EINVAL, "scale: RGBA buffers must be 16-byte aligned");
  ScaleArgs a{src, dst, static_cast<int>(w), static_cast<int>(h), static_cast<int>(ow), static_cast<int>(oh),
              d_xoff, d_xidx, d_yoff, d_yidx, d_xwt, d_ywt};
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  dim3 grid(static_cast<unsigned>((ow + 127) / 128), static_cast<unsigned>(oh));
  switch (channels) {
    case 1: scale_kernel<1><<<grid, 128, 0, s>>>(a); break;
    case 2: scale_kernel<2><<<grid, 128, 0, s>>>(a); break;
    case 3: scale_kernel<3><<<grid, 128, 0, s>>>(a); break;
    case 4: scale_kernel<4><<<grid, 128, 0, s>>>(a); break;
    default: return fail(MB200_EINVAL, "scale: 1..4 channels");
  }
  count_launch();
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? MB200_OK : cuda_fail(e, "scale launch");
}

int launch_unsharp_combine(const float *src, float *blur_inout, size_t n, double gain, double quantum_threshold,
                           void *stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const bool aligned = ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(blur_inout)) & 15) == 0;
  const size_t n4 = aligned ? n / 4 : 0;
  if (n4) {
    unsharp_kernel<<<static_cast<unsigned>((n4 + 255) / 256), 256, 0, s>>>(
        reinterpret_cast<const float4 *>(src), reinterpret_cast<float4 *>(blur_inout), n4, gain, quantum_threshold);
    count_launch();
  }
  if (n4 * 4 < n) {
    const size_t rest = n - n4 * 4;
    unsharp_tail_kernel<<<static_cast<unsigned>((rest + 255) / 256), 256, 0, s>>>(src, blur_inout, n4 * 4, n, gain,
                                                                                 quantum_threshold);
    count_launch();
  }
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "unsharp launch");
  return MB200_OK;
}

}  // namespace mb200
