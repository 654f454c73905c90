// stencils.cu -- the neighbourhood operators next to the convolution path (SURVEY 8f rank 4):
//   StatisticImage       MagickCore/statistic.c:2918-3160   (Gradient, Maximum, Mean, Median, Minimum, Mode, Nonpeak,
//                                                             RootMeanSquare, StandardDeviation, Contrast)
//   RotationalBlurImage  MagickCore/effect.c:3129-3400
//   BilateralBlurImage   MagickCore/effect.c:821-1165
//   SelectiveBlurImage   MagickCore/effect.c:3406-3700
//   AdaptiveBlurImage / AdaptiveSharpenImage   MagickCore/effect.c:128-416 / :447-735
// One thread per output pixel, all channels of the pixel in one pass over the window (the per-channel accumulation
// order of the reference -- window order, sequential double adds -- is kept, and every operation is an UNFUSED IEEE double
// operation, so the results are bit-identical to the reference's).  Neighbours are fetched through the read-only path
// (float4 for RGBA); the windows of adjacent threads overlap almost completely, so L1 / L2 serve the re-reads.  These
// are first, untuned versions (correctness first; DESIGN.md lists their measured throughput).
#include "launch.cuh"

#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <vector>

namespace mb200 {
namespace {

constexpr double kQS = 1.0 / 65535.0, kEps = 1.0e-12;

template <int CH>
__device__ __forceinline__ void load_pixel(const float *__restrict__ src, size_t index, float (&v)[CH]) {
  const float *r = src + index * CH;
  if (CH == 4) {
    const float4 t = __ldg(reinterpret_cast<const float4 *>(r));
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[CH - 1] = t.w;
  } else {
#pragma unroll
    for (int c = 0; c < CH; ++c) v[c] = __ldg(r + c);
  }
}

template <int CH>
__device__ __forceinline__ void store_pixel(float *__restrict__ dst, size_t index, const float (&o)[CH]) {
  float *q = dst + index * CH;
  if (CH == 4) *reinterpret_cast<float4 *>(q) = make_float4(o[0], o[1], o[2], o[CH - 1]);
  else {
#pragma unroll
    for (int c = 0; c < CH; ++c) q[c] = o[c];
  }
}

// PerceptibleReciprocal (pixel-accessor.h:242-254) with IEEE division
__device__ __forceinline__ double perceptible_reciprocal(double x) {
  const double sign = x < 0.0 ? -1.0 : 1.0;
  return __dmul_rn(sign, x) >= kEps ? __ddiv_rn(1.0, x) : __ddiv_rn(sign, kEps);
}

// GetPixelIntensity, Rec709Luma on an sRGB / gray image (pixel.c:2356): see threshold_kernel (pointwise.cu)
template <int CH>
__device__ __forceinline__ double pixel_intensity(const float (&v)[CH]) {
  const double red = static_cast<double>(v[0]);
  if (CH == 1) return red;
  const double green = CH >= 3 ? static_cast<double>(v[CH >= 3 ? 1 : 0]) : red;
  const double blue = CH >= 3 ? static_cast<double>(v[CH >= 3 ? 2 : 0]) : red;
  return __dadd_rn(__dadd_rn(__dmul_rn(0.212656, red), __dmul_rn(0.715158, green)), __dmul_rn(0.072186, blue));
}

// ------------------------------------------------------------------------------------------------ StatisticImage
// MagickAbsoluteValue (image-private.h:45): unlike fabs it keeps -0 (Contrast of a one-level window of negative samples)
__device__ __forceinline__ double magick_absolute_value(double x) { return x < 0.0 ? -x : x; }

__device__ __forceinline__ unsigned scale_quantum_to_short(float q) {      // quantum-private.h (HDRI)
  if (!(q > 0.0f)) return 0u;
  if (q >= 65535.0f) return 65535u;
  return static_cast<unsigned>(q + 0.5f);
}

// The element of sorted index k among the ScaleQuantumToShort values of channel c over the W x H window at (x0, y0),
// edge replicated: a 16-bit radix select (one pass over the window per bit) -- what the reference reads off its skip list.
template <int CH>
__device__ __forceinline__ unsigned window_select(const float *__restrict__ src, int w, int h, int x0, int y0, int W, int H,
                                                  int c, unsigned k) {
  unsigned prefix = 0;
  for (int bit = 15; bit >= 0; --bit) {
    const unsigned himask = bit == 15 ? 0u : (0xffffu << (bit + 1)) & 0xffffu;
    unsigned zeros = 0;
    for (int v = 0; v < H; ++v) {
      const size_t row = static_cast<size_t>(min(max(y0 + v, 0), h - 1)) * w;
      for (int u = 0; u < W; ++u) {
        const unsigned s = scale_quantum_to_short(__ldg(src + (row + min(max(x0 + u, 0), w - 1)) * CH + c));
        zeros += ((s & himask) == prefix && !(s >> bit & 1u)) ? 1u : 0u;
      }
    }
    if (k >= zeros) { k -= zeros; prefix |= 1u << bit; }
  }
  return prefix;
}

// type: statistic.h:141-151 (1 Gradient, 2 Maximum, 3 Mean, 4 Median, 5 Minimum, 6 Mode, 7 Nonpeak, 8 RootMeanSquare,
// 9 StandardDeviation, 10 Contrast).  The window's top-left corner is (x - W/2, y - H/2), edge replicated (:3012-3020).
template <int CH>
__global__ void __launch_bounds__(128) statistic_kernel(const float *__restrict__ src, float *__restrict__ dst, int w, int h,
                                                        int type, int W, int H) {
  const int x = blockIdx.x * 128 + threadIdx.x, y = blockIdx.y;
  if (x >= w) return;
  const int x0 = x - W / 2, y0 = y - H / 2;
  float o[CH];
  if (type == 4) {
    // Median: the reference inserts ScaleQuantumToShort(value) into a skip list and returns the element at sorted index
    // length/2 (:2784, :2878) -- a 16-bit radix select over the window gives the same element without storing it.
    if (W == 3 && H == 3) {
      // 3x3 (`-median 1`, by far the most common window): the nine samples are loaded once and the element of sorted
      // index 4 comes out of the 19-exchange median network (checked on all 512 0/1 inputs), per channel.
      unsigned s[9][CH];
#pragma unroll
      for (int v = 0; v < 3; ++v) {
        const size_t row = static_cast<size_t>(min(max(y0 + v, 0), h - 1)) * w;
#pragma unroll
        for (int u = 0; u < 3; ++u) {
          float p[CH];
          load_pixel<CH>(src, row + min(max(x0 + u, 0), w - 1), p);
#pragma unroll
          for (int c = 0; c < CH; ++c) s[v * 3 + u][c] = scale_quantum_to_short(p[c]);
        }
      }
#define MB200_SORT2(a, b) { const unsigned lo_ = min(s[a][c], s[b][c]); s[b][c] = max(s[a][c], s[b][c]); s[a][c] = lo_; }
#pragma unroll
      for (int c = 0; c < CH; ++c) {
        MB200_SORT2(1, 2) MB200_SORT2(4, 5) MB200_SORT2(7, 8) MB200_SORT2(0, 1) MB200_SORT2(3, 4) MB200_SORT2(6, 7)
        MB200_SORT2(1, 2) MB200_SORT2(4, 5) MB200_SORT2(7, 8) MB200_SORT2(0, 3) MB200_SORT2(5, 8) MB200_SORT2(4, 7)
        MB200_SORT2(3, 6) MB200_SORT2(1, 4) MB200_SORT2(2, 5) MB200_SORT2(4, 7) MB200_SORT2(4, 2) MB200_SORT2(6, 4)
        MB200_SORT2(4, 2)
        o[c] = static_cast<float>(s[4][c]);
      }
#undef MB200_SORT2
      store_pixel<CH>(dst, static_cast<size_t>(y) * w + x, o);
      return;
    }
    const unsigned n = static_cast<unsigned>(W) * static_cast<unsigned>(H);
#pragma unroll
    for (int c = 0; c < CH; ++c) o[c] = static_cast<float>(static_cast<double>(window_select<CH>(src, w, h, x0, y0, W, H, c, n >> 1)));
    store_pixel<CH>(dst, static_cast<size_t>(y) * w + x, o);
    return;
  }
  if (type == 6) {
    // Mode (GetModePixelList :2809): the reference walks the distinct 16-bit values of the window in ascending order and
    // keeps the first one whose count is strictly the greatest.  Same walk here without the list: one pass over the window
    // per distinct value finds the next larger value and its count (<= W*H passes, the window stays in L1).
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const unsigned n = static_cast<unsigned>(W) * static_cast<unsigned>(H);
      unsigned mode = 65536u, best = 0u, seen = 0u;
      int current = -1;
      while (seen < n) {
        unsigned value = 0x10000u, count = 0u;
        for (int v = 0; v < H; ++v) {
          const size_t row = static_cast<size_t>(min(max(y0 + v, 0), h - 1)) * w;
          for (int u = 0; u < W; ++u) {
            const unsigned s = scale_quantum_to_short(__ldg(src + (row + min(max(x0 + u, 0), w - 1)) * CH + c));
            if (static_cast<int>(s) > current) {
              if (s < value) { value = s; count = 1u; }
              else if (s == value) ++count;
            }
          }
        }
        if (count == 0u) break;                  // cannot happen while seen < n; keeps the loop finite regardless
        if (count > best) { best = count; mode = value; }
        seen += count;
        current = static_cast<int>(value);
      }
      o[c] = static_cast<float>(static_cast<double>(mode));
    }
    store_pixel<CH>(dst, static_cast<size_t>(y) * w + x, o);
    return;
  }
  if (type == 7) {
    // Nonpeak (GetNonpeakPixelList :2843): the median's value, unless it is the smallest distinct value of the window and
    // a larger one exists (then that one), or the largest and a smaller one exists (then that one).
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const unsigned n = static_cast<unsigned>(W) * static_cast<unsigned>(H);
      const unsigned median = window_select<CH>(src, w, h, x0, y0, W, H, c, n >> 1);
      int previous = -1, next = -1;
      for (int v = 0; v < H; ++v) {
        const size_t row = static_cast<size_t>(min(max(y0 + v, 0), h - 1)) * w;
        for (int u = 0; u < W; ++u) {
          const int s = static_cast<int>(scale_quantum_to_short(__ldg(src + (row + min(max(x0 + u, 0), w - 1)) * CH + c)));
          if (s < static_cast<int>(median)) previous = max(previous, s);
          if (s > static_cast<int>(median)) next = next < 0 ? s : min(next, s);
        }
      }
      unsigned color = median;
      if (previous < 0 && next >= 0) color = static_cast<unsigned>(next);
      else if (previous >= 0 && next < 0) color = static_cast<unsigned>(previous);
      o[c] = static_cast<float>(static_cast<double>(color));
    }
    store_pixel<CH>(dst, static_cast<size_t>(y) * w + x, o);
    return;
  }
  double minimum[CH], maximum[CH], sum[CH], sum_squared[CH];
  double area = 0.0;
  bool first = true;
  for (int v = 0; v < H; ++v) {
    const size_t row = static_cast<size_t>(min(max(y0 + v, 0), h - 1)) * w;
    for (int u = 0; u < W; ++u) {
      float p[CH];
      load_pixel<CH>(src, row + min(max(x0 + u, 0), w - 1), p);
      area = __dadd_rn(area, 1.0);
#pragma unroll
      for (int c = 0; c < CH; ++c) {
        const double value = static_cast<double>(p[c]);
        if (first) { minimum[c] = value; maximum[c] = value; sum[c] = 0.0; sum_squared[c] = 0.0; }
        if (value < minimum[c]) minimum[c] = value;
        if (value > maximum[c]) maximum[c] = value;
        sum[c] = __dadd_rn(sum[c], value);
        sum_squared[c] = __dadd_rn(sum_squared[c], __dmul_rn(value, value));
      }
      first = false;
    }
  }
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    double pixel;
    switch (type) {
      case 1: pixel = magick_absolute_value(__dsub_rn(maximum[c], minimum[c])); break;
      case 2: pixel = maximum[c]; break;
      case 5: pixel = minimum[c]; break;
      case 8: pixel = __dsqrt_rn(__ddiv_rn(sum_squared[c], area)); break;
      case 9: {                                              // sqrt(ss/area - (sum/area*sum/area)), left to right
        const double m = __ddiv_rn(__dmul_rn(__ddiv_rn(sum[c], area), sum[c]), area);
        pixel = __dsqrt_rn(__dsub_rn(__ddiv_rn(sum_squared[c], area), m));
        break;
      }
      case 10: pixel = magick_absolute_value(__dmul_rn(__dsub_rn(maximum[c], minimum[c]), perceptible_reciprocal(__dadd_rn(maximum[c], minimum[c])))); break;
      default: pixel = __ddiv_rn(sum[c], area); break;
    }
    o[c] = static_cast<float>(pixel);
  }
  store_pixel<CH>(dst, static_cast<size_t>(y) * w + x, o);
}

// ------------------------------------------------------------------------------------------- RotationalBlurImage
// n samples on the arc through the pixel about the image centre; cos / sin tables from the host (libm, like the
// reference); every `step`-th sample, step = blur_radius / radius clamped to [1, n-1] (:3246-3262).
template <int CH>
__global__ void __launch_bounds__(128) rotational_blur_kernel(const float *__restrict__ src, float *__restrict__ dst, int w,
                                                              int h, const double *__restrict__ cos_theta,
                                                              const double *__restrict__ sin_theta, int n, double cx, double cy,
                                                              double blur_radius) {
  const int x = blockIdx.x * 128 + threadIdx.x, y = blockIdx.y;
  if (x >= w) return;
  constexpr bool kAlpha = (CH == 2 || CH == 4);
  const double dx = __dsub_rn(static_cast<double>(x), cx), dy = __dsub_rn(static_cast<double>(y), cy);
  // hypot(dx, dy): dx, dy are multiples of 0.5 of moderate size, dx*dx + dy*dy is exact, so the correctly rounded square
  // root IS the correctly rounded hypot glibc returns
  const double radius = __dsqrt_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)));
  int step = 1;
  if (radius != 0.0) {
    const double ratio = __ddiv_rn(blur_radius, radius);
    step = ratio >= static_cast<double>(n) ? n - 1 : static_cast<int>(ratio);
    if (step == 0) step = 1;
    else if (step >= n) step = n - 1;
  }
  double pixel[CH], gamma = 0.0, count = 0.0;
#pragma unroll
  for (int c = 0; c < CH; ++c) pixel[c] = 0.0;
  for (int j = 0; j < n; j += step) {
    const double ct = __ldg(cos_theta + j), st = __ldg(sin_theta + j);
    // (ssize_t) (cx + dx*cos - dy*sin + 0.5): truncation toward zero, then edge replication
    const double fx = __dadd_rn(__dsub_rn(__dadd_rn(cx, __dmul_rn(dx, ct)), __dmul_rn(dy, st)), 0.5);
    const double fy = __dadd_rn(__dadd_rn(__dadd_rn(cy, __dmul_rn(dx, st)), __dmul_rn(dy, ct)), 0.5);
    const int xx = min(max(static_cast<int>(fx), 0), w - 1), yy = min(max(static_cast<int>(fy), 0), h - 1);
    float r[CH];
    load_pixel<CH>(src, static_cast<size_t>(yy) * w + xx, r);
    count = __dadd_rn(count, 1.0);
    if (kAlpha) {
      const double alpha = __dmul_rn(kQS, static_cast<double>(r[CH - 1]));
#pragma unroll
      for (int c = 0; c < CH - 1; ++c) pixel[c] = __dadd_rn(pixel[c], __dmul_rn(alpha, static_cast<double>(r[c])));
      gamma = __dadd_rn(gamma, alpha);
      pixel[CH - 1] = __dadd_rn(pixel[CH - 1], static_cast<double>(r[CH - 1]));
    } else {
#pragma unroll
      for (int c = 0; c < CH; ++c) pixel[c] = __dadd_rn(pixel[c], static_cast<double>(r[c]));
    }
  }
  float o[CH];
  const double plain = perceptible_reciprocal(count);
  if (kAlpha) {
    const double g = perceptible_reciprocal(gamma);
#pragma unroll
    for (int c = 0; c < CH - 1; ++c) o[c] = static_cast<float>(__dmul_rn(g, pixel[c]));
    o[CH - 1] = static_cast<float>(__dmul_rn(plain, pixel[CH - 1]));
  } else {
#pragma unroll
    for (int c = 0; c < CH; ++c) o[c] = static_cast<float>(__dmul_rn(plain, pixel[c]));
  }
  store_pixel<CH>(dst, static_cast<size_t>(y) * w + x, o);
}

// -------------------------------------------------------------------------------------------- BilateralBlurImage
// 8-bit intensity plane (ScaleQuantumToChar of the float-converted intensity, :1017-1030): one pre-pass instead of an
// intensity evaluation per tap.
__device__ __forceinline__ unsigned scale_quantum_to_char(float q) {       // quantum.h:113-124 (HDRI)
  if (!(q > 0.0f)) return 0u;
  const float s = q / 257.0f;
  if (s >= 255.0f) return 255u;
  return static_cast<unsigned>(s + 0.5f);
}

template <int CH>
__global__ void __launch_bounds__(256) intensity8_kernel(const float *__restrict__ src, unsigned char *__restrict__ out, size_t n) {
  const size_t i = static_cast<size_t>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= n) return;
  float v[CH];
  load_pixel<CH>(src, i, v);
  out[i] = static_cast<unsigned char>(scale_quantum_to_char(static_cast<float>(pixel_intensity<CH>(v))));
}

// weight(k) = intensity_gaussian[I(r_k) - I(p) + 255] * spatial_gaussian[k]; r_k = (x + mid_x - u, y + mid_y - v), the
// reference's reflected window index (:1060-1070); colour channels of images with alpha normalise by
// sum w * (QS*alpha(p)) * (QS*alpha(r)) while accumulating w * r unweighted (:1108-1125), as written there.
template <int CH>
__global__ void __launch_bounds__(128) bilateral_kernel(const float *__restrict__ src, const unsigned char *__restrict__ i8,
                                                        float *__restrict__ dst, int w, int h, int W, int H,
                                                        const double *__restrict__ intensity_gaussian,
                                                        const double *__restrict__ spatial_gaussian) {
  const int x = blockIdx.x * 128 + threadIdx.x, y = blockIdx.y;
  if (x >= w) return;
  constexpr bool kAlpha = (CH == 2 || CH == 4);
  const int midx = W / 2, midy = H / 2;
  const size_t centre = static_cast<size_t>(y) * w + x;
  const int ip = i8[centre];
  double palpha = 1.0;
  if (kAlpha) palpha = __dmul_rn(kQS, static_cast<double>(__ldg(src + centre * CH + CH - 1)));
  double pixel[CH], gamma_plain = 0.0, gamma_blend = 0.0;
#pragma unroll
  for (int c = 0; c < CH; ++c) pixel[c] = 0.0;
  int k = 0;
  for (int v = 0; v < H; ++v) {
    const size_t row = static_cast<size_t>(min(max(y + midy - v, 0), h - 1)) * w;
    for (int u = 0; u < W; ++u, ++k) {
      const size_t idx = row + min(max(x + midx - u, 0), w - 1);
      const int d = static_cast<int>(__ldg(i8 + idx)) - ip;
      const double wt = __dmul_rn(__ldg(intensity_gaussian + d + 255), __ldg(spatial_gaussian + k));
      float r[CH];
      load_pixel<CH>(src, idx, r);
#pragma unroll
      for (int c = 0; c < CH; ++c) pixel[c] = __dadd_rn(pixel[c], __dmul_rn(wt, static_cast<double>(r[c])));
      gamma_plain = __dadd_rn(gamma_plain, wt);
      if (kAlpha)
        gamma_blend = __dadd_rn(gamma_blend, __dmul_rn(__dmul_rn(wt, palpha), __dmul_rn(kQS, static_cast<double>(r[CH - 1]))));
    }
  }
  float o[CH];
  const double gp = perceptible_reciprocal(gamma_plain);
  const double gb = kAlpha ? perceptible_reciprocal(gamma_blend) : gp;
#pragma unroll
  for (int c = 0; c < CH; ++c) o[c] = static_cast<float>(__dmul_rn((kAlpha && c != CH - 1) ? gb : gp, pixel[c]));
  store_pixel<CH>(dst, centre, o);
}

// -------------------------------------------------------------------------------------------- SelectiveBlurImage
// Double intensity plane (one pre-pass): the reference compares the centre's double intensity with, for the alpha-blended
// colour channels, the neighbour's double intensity (:3657) and, for the others, the neighbour's intensity in its GRAY
// clone (:3629), which gray_clone_intensity derives from the same plane.
template <int CH>
__global__ void __launch_bounds__(256) intensity_plane_kernel(const float *__restrict__ src, double *__restrict__ out, size_t n) {
  const size_t i = static_cast<size_t>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= n) return;
  float v[CH];
  load_pixel<CH>(src, i, v);
  out[i] = pixel_intensity<CH>(v);
}

// GetPixelIntensity of the GRAY clone's pixel, from the pixel's double intensity li.  The clone stores li rounded to
// float (colorspace.c:943-945); a gray image is not transformed, and its li is already its sample.  With alpha the clone
// keeps two channels, so the intensity weighs its sample as (g, g, g) again (pixel.c:2366) -- for a gray image that is
// li itself.
template <int CH>
__device__ __forceinline__ double gray_clone_intensity(double li) {
  if (CH == 2) return li;
  const float g[2] = {static_cast<float>(li), 0.0f};
  return CH == 4 ? pixel_intensity<2>(g) : static_cast<double>(g[0]);
}

// window top-left (x - j, y - j), j = (width-1)/2, edge replicated; taps in window order, unfused.
template <int CH>
__global__ void __launch_bounds__(128) selective_blur_kernel(const float *__restrict__ src, const double *__restrict__ lum,
                                                             float *__restrict__ dst, int w, int h, int W,
                                                             const double *__restrict__ taps, double threshold) {
  const int x = blockIdx.x * 128 + threadIdx.x, y = blockIdx.y;
  if (x >= w) return;
  constexpr bool kAlpha = (CH == 2 || CH == 4);
  const int j = (W - 1) / 2;
  const size_t centre = static_cast<size_t>(y) * w + x;
  const double intensity = lum[centre];
  double plain[CH], blend[CH], gamma_plain = 0.0, gamma_blend = 0.0;
#pragma unroll
  for (int c = 0; c < CH; ++c) plain[c] = blend[c] = 0.0;
  int k = 0;
  for (int v = 0; v < W; ++v) {
    const size_t row = static_cast<size_t>(min(max(y - j + v, 0), h - 1)) * w;
    for (int u = 0; u < W; ++u, ++k) {
      const size_t idx = row + min(max(x - j + u, 0), w - 1);
      const double li = __ldg(lum + idx);
      const bool take_plain = fabs(__dsub_rn(gray_clone_intensity<CH>(li), intensity)) < threshold;
      const bool take_blend = kAlpha && fabs(__dsub_rn(li, intensity)) < threshold;
      if (!take_plain && !take_blend) continue;
      const double t = __ldg(taps + k);
      float r[CH];
      load_pixel<CH>(src, idx, r);
      if (take_plain) {
        gamma_plain = __dadd_rn(gamma_plain, t);
        if (kAlpha) plain[CH - 1] = __dadd_rn(plain[CH - 1], __dmul_rn(t, static_cast<double>(r[CH - 1])));
        else {
#pragma unroll
          for (int c = 0; c < CH; ++c) plain[c] = __dadd_rn(plain[c], __dmul_rn(t, static_cast<double>(r[c])));
        }
      }
      if (take_blend) {
        const double ta = __dmul_rn(t, __dmul_rn(kQS, static_cast<double>(r[CH - 1])));
        gamma_blend = __dadd_rn(gamma_blend, ta);
#pragma unroll
        for (int c = 0; c < CH - 1; ++c) blend[c] = __dadd_rn(blend[c], __dmul_rn(ta, static_cast<double>(r[c])));
      }
    }
  }
  float p[CH], o[CH];
  load_pixel<CH>(src, centre, p);
  const bool keep_plain = fabs(gamma_plain) < kEps, keep_blend = fabs(gamma_blend) < kEps;
  const double gp = perceptible_reciprocal(gamma_plain), gb = perceptible_reciprocal(gamma_blend);
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    if (kAlpha && c != CH - 1) o[c] = keep_blend ? p[c] : static_cast<float>(__dmul_rn(gb, blend[c]));
    else o[c] = keep_plain ? p[c] : static_cast<float>(__dmul_rn(gp, plain[c]));
  }
  store_pixel<CH>(dst, centre, o);
}

// ------------------------------------------------------------------- AdaptiveBlurImage / AdaptiveSharpenImage
// The operator picks a kernel SIZE per pixel from an edge map (EdgeImage -> AutoLevelImage -> BlurImage -> AutoLevelImage),
// so a one-ULP difference in that map could select a different kernel for a pixel.  Its stages therefore do not use the
// FMA-contracted streaming kernels: exact_convolve_kernel evaluates ConvolveMorphology (morphology.c:2897-2979, and the
// column path :2654-2807, which for kernels without NaN cells is the same arithmetic) with unfused IEEE operations in the
// reference's cell order, and the whole pipeline is bit-identical to the reference's.
//   cells[] is already reflected (cells[v*kw+u] = values[kw*kh-1-(v*kw+u)]), (ox, oy) = (kw-x-1, kh-y-1).
template <int CH>
__global__ void __launch_bounds__(128) exact_convolve_kernel(const float *__restrict__ src, float *__restrict__ dst, int w, int h,
                                                             const double *__restrict__ cells, int kw, int kh, int ox, int oy) {
  const int x = blockIdx.x * 128 + threadIdx.x, y = blockIdx.y;
  if (x >= w) return;
  constexpr bool kAlpha = (CH == 2 || CH == 4);
  double pixel[CH], gamma = 0.0;
#pragma unroll
  for (int c = 0; c < CH; ++c) pixel[c] = 0.0;
  int k = 0;
  for (int v = 0; v < kh; ++v) {
    const size_t row = static_cast<size_t>(min(max(y - oy + v, 0), h - 1)) * w;
    for (int u = 0; u < kw; ++u, ++k) {
      const double kv = __ldg(cells + k);
      float p[CH];
      load_pixel<CH>(src, row + min(max(x - ox + u, 0), w - 1), p);
      if (kAlpha) {
        const double ak = __dmul_rn(__dmul_rn(kQS, static_cast<double>(p[CH - 1])), kv);      // alpha * kv
        gamma = __dadd_rn(gamma, ak);
#pragma unroll
        for (int c = 0; c < CH - 1; ++c) pixel[c] = __dadd_rn(pixel[c], __dmul_rn(ak, static_cast<double>(p[c])));
        pixel[CH - 1] = __dadd_rn(pixel[CH - 1], __dmul_rn(kv, static_cast<double>(p[CH - 1])));
      } else {
#pragma unroll
        for (int c = 0; c < CH; ++c) pixel[c] = __dadd_rn(pixel[c], __dmul_rn(kv, static_cast<double>(p[c])));
      }
    }
  }
  float o[CH];
  const double g = kAlpha ? perceptible_reciprocal(gamma) : 1.0;
#pragma unroll
  for (int c = 0; c < CH; ++c) o[c] = static_cast<float>(__dmul_rn((kAlpha && c != CH - 1) ? g : 1.0, pixel[c]));
  store_pixel<CH>(dst, static_cast<size_t>(y) * w + x, o);
}

// The adaptive stage (effect.c:279-372): j from the edge map's intensity, then the (width - j)^2 window in plain order.
// kernels[] holds the pyramid back to back, offsets[j / 2] the start of kernel[j].
template <int CH>
__global__ void __launch_bounds__(128) adaptive_kernel(const float *__restrict__ src, const float *__restrict__ edge,
                                                       float *__restrict__ dst, int w, int h, int width,
                                                       const double *__restrict__ kernels, const int *__restrict__ offsets) {
  const int x = blockIdx.x * 128 + threadIdx.x, y = blockIdx.y;
  if (x >= w) return;
  constexpr bool kAlpha = (CH == 2 || CH == 4);
  const size_t centre = static_cast<size_t>(y) * w + x;
  float r[CH];
  load_pixel<CH>(edge, centre, r);
  const double t = ceil(__dsub_rn(__dmul_rn(static_cast<double>(width), __dsub_rn(1.0, __dmul_rn(kQS, pixel_intensity<CH>(r)))), 0.5));
  int j = t != t ? 0 : (t <= 0.0 ? 0 : (t >= static_cast<double>(width) ? width : static_cast<int>(t)));   // CastDoubleToLong + clip
  if ((j & 1) != 0) --j;
  const int size = width - j, x0 = x - size / 2, y0 = y - size / 2;
  const double *k = kernels + __ldg(offsets + (j >> 1));
  double pixel[CH], gamma_plain = 0.0, gamma_blend = 0.0;
#pragma unroll
  for (int c = 0; c < CH; ++c) pixel[c] = 0.0;
  for (int v = 0; v < size; ++v) {
    const size_t row = static_cast<size_t>(min(max(y0 + v, 0), h - 1)) * w;
    for (int u = 0; u < size; ++u, ++k) {
      const double kv = __ldg(k);
      float p[CH];
      load_pixel<CH>(src, row + min(max(x0 + u, 0), w - 1), p);
      gamma_plain = __dadd_rn(gamma_plain, kv);
      if (kAlpha) {
        const double ka = __dmul_rn(kv, __dmul_rn(kQS, static_cast<double>(p[CH - 1])));      // (*k) * alpha
        gamma_blend = __dadd_rn(gamma_blend, ka);
#pragma unroll
        for (int c = 0; c < CH - 1; ++c) pixel[c] = __dadd_rn(pixel[c], __dmul_rn(ka, static_cast<double>(p[c])));
        pixel[CH - 1] = __dadd_rn(pixel[CH - 1], __dmul_rn(kv, static_cast<double>(p[CH - 1])));
      } else {
#pragma unroll
        for (int c = 0; c < CH; ++c) pixel[c] = __dadd_rn(pixel[c], __dmul_rn(kv, static_cast<double>(p[c])));
      }
    }
  }
  float o[CH];
  const double gp = perceptible_reciprocal(gamma_plain), gb = kAlpha ? perceptible_reciprocal(gamma_blend) : gp;
#pragma unroll
  for (int c = 0; c < CH; ++c) o[c] = static_cast<float>(__dmul_rn((kAlpha && c != CH - 1) ? gb : gp, pixel[c]));
  store_pixel<CH>(dst, centre, o);
}

int check_image(const float *src, float *dst, size_t w, size_t h, int channels, const char *what) {
  if (!src || !dst || w == 0 || h == 0 || w > 0x3fffffffull || h > 65535ull * 32768ull) return fail(MB200_EINVAL, "%s: bad geometry", what);
  if (h > 65535) return fail(MB200_EUNSUPPORTED, "%s: more than 65535 rows", what);
  if (channels < 1 || channels > 4) return fail(MB200_EINVAL, "%s: 1..4 channels", what);
  if (channels == 4 && !aligned16(src, dst)) return fail(MB200_EINVAL, "%s: RGBA buffers must be 16-byte aligned", what);
  return MB200_OK;
}

}  // namespace

int launch_statistic(const float *src, float *dst, size_t w, size_t h, int channels, int type, size_t width, size_t height,
                     void *stream) {
  int rc = check_image(src, dst, w, h, channels, "statistic");
  if (rc) return rc;
  if (type < 1 || type > 10) return fail(MB200_EINVAL, "statistic type %d", type);
  const size_t W = width > 1 ? width : 1, H = height > 1 ? height : 1;
  if (W > 255 || H > 255) return fail(MB200_EUNSUPPORTED, "statistic: window larger than 255");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  dim3 grid(static_cast<unsigned>((w + 127) / 128), static_cast<unsigned>(h));
  const int iw = static_cast<int>(w), ih = static_cast<int>(h), iW = static_cast<int>(W), iH = static_cast<int>(H);
  return with_channels(channels, "statistic", [&](auto ch) {
    statistic_kernel<ch()><<<grid, 128, 0, s>>>(src, dst, iw, ih, type, iW, iH);
    return launch_status("statistic launch");
  });
}

int launch_rotational_blur(const float *src, float *dst, size_t w, size_t h, int channels, double angle, void *stream) {
  int rc = check_image(src, dst, w, h, channels, "rotational blur");
  if (rc) return rc;
  // effect.c:3177-3203: centre, blur radius, sample count and the cos / sin tables
  const double kPi = 3.14159265358979323846264338327950288419716939937510;
  const double cx = static_cast<double>(w - 1) / 2.0, cy = static_cast<double>(h - 1) / 2.0;
  const double blur_radius = std::hypot(cx, cy);
  const double rad = kPi * angle / 180.0;
  const size_t n = static_cast<size_t>(std::fabs(4.0 * rad * std::sqrt(blur_radius) + 2UL));
  if (n < 2 || n > (1u << 20)) return fail(MB200_EUNSUPPORTED, "rotational blur: %zu samples per pixel", n);
  const double theta = rad / static_cast<double>(n - 1), offset = theta * static_cast<double>(n - 1) / 2.0;
  std::vector<double> tables(2 * n);
  for (size_t k = 0; k < n; ++k) {
    tables[k] = std::cos(theta * static_cast<double>(static_cast<long>(k)) - offset);
    tables[n + k] = std::sin(theta * static_cast<double>(static_cast<long>(k)) - offset);
  }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  StreamAlloc table(s);
  if ((rc = table.upload(tables.data(), tables.size() * sizeof(double), "rotational blur: table upload"))) return rc;
  const double *d_tables = table.as<double>();
  dim3 grid(static_cast<unsigned>((w + 127) / 128), static_cast<unsigned>(h));
  const int iw = static_cast<int>(w), ih = static_cast<int>(h), in = static_cast<int>(n);
  return with_channels(channels, "rotational blur", [&](auto ch) {
    rotational_blur_kernel<ch()><<<grid, 128, 0, s>>>(src, dst, iw, ih, d_tables, d_tables + n, in, cx, cy, blur_radius);
    return launch_status("rotational blur launch");
  });
}

int launch_bilateral_blur(const float *src, float *dst, size_t w, size_t h, int channels, size_t width, size_t height,
                          double intensity_sigma, double spatial_sigma, void *stream) {
  int rc = check_image(src, dst, w, h, channels, "bilateral blur");
  if (rc) return rc;
  const size_t W = width > 1 ? width : 1, H = height > 1 ? height : 1;
  if ((W % 2) == 0 || (H % 2) == 0)
    return fail(MB200_EUNSUPPORTED, "bilateral blur: even window sizes (the reference's reflected index leaves the window it fetched)");
  if (W > 255 || H > 255) return fail(MB200_EUNSUPPORTED, "bilateral blur: window larger than 255");
  // BlurGaussian (effect.c:808-819) tables: 511 intensity differences, W*H distances from the window centre
  auto reciprocal = [](double x) { const double sign = x < 0.0 ? -1.0 : 1.0; return sign * x >= kEps ? 1.0 / x : sign / kEps; };
  const double k2Pi = 6.28318530717958647692528676655900576839433879875020;
  auto blur_gaussian = [&](double x, double sigma) {
    return std::exp(-(x * x) * reciprocal(2.0 * sigma * sigma)) * reciprocal(k2Pi * sigma * sigma);
  };
  std::vector<double> tables(512 + W * H);
  for (int v = -255; v <= 255; ++v) tables[v + 255] = blur_gaussian(static_cast<double>(v), intensity_sigma);
  tables[511] = 0.0;
  size_t n = 512;
  const long midx = static_cast<long>(W) / 2, midy = static_cast<long>(H) / 2;
  for (long v = 0; v < static_cast<long>(H); ++v)
    for (long u = 0; u < static_cast<long>(W); ++u) {
      const double dx = 0.0 - static_cast<double>(u - midx), dy = 0.0 - static_cast<double>(v - midy);
      tables[n++] = blur_gaussian(std::sqrt(dx * dx + dy * dy), spatial_sigma);
    }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  StreamAlloc table(s), plane(s);
  if ((rc = table.upload(tables.data(), tables.size() * sizeof(double), "bilateral blur: table upload"))) return rc;
  if ((rc = plane.alloc(w * h, "bilateral blur: intensity plane"))) return rc;
  const double *d_tables = table.as<double>();
  unsigned char *d_i8 = plane.as<unsigned char>();
  const size_t npix = w * h;
  const unsigned pgrid = static_cast<unsigned>((npix + 255) / 256);
  dim3 grid(static_cast<unsigned>((w + 127) / 128), static_cast<unsigned>(h));
  const int iw = static_cast<int>(w), ih = static_cast<int>(h), iW = static_cast<int>(W), iH = static_cast<int>(H);
  return with_channels(channels, "bilateral blur", [&](auto ch) {
    intensity8_kernel<ch()><<<pgrid, 256, 0, s>>>(src, d_i8, npix);
    bilateral_kernel<ch()><<<grid, 128, 0, s>>>(src, d_i8, dst, iw, ih, iW, iH, d_tables, d_tables + 512);
    return launch_status("bilateral blur launch", 2);
  });
}

int launch_selective_blur(const float *src, float *dst, size_t w, size_t h, int channels, double radius, double sigma,
                          double threshold, void *stream) {
  int rc = check_image(src, dst, w, h, channels, "selective blur");
  if (rc) return rc;
  const size_t W = mb200_optimal_kernel_width_1d(radius, sigma);
  if (W > 255) return fail(MB200_EUNSUPPORTED, "selective blur: window larger than 255");
  // effect.c:3467-3478: exp(-(u^2+v^2)/(2 s^2)) / (2 pi s^2), not normalised (gamma does that per pixel)
  const double kPi = 3.14159265358979323846264338327950288419716939937510;
  const double sg = std::fabs(sigma) < kEps ? kEps : sigma;
  const long j = static_cast<long>(W - 1) / 2;
  std::vector<double> taps(W * W);
  size_t n = 0;
  for (long v = -j; v <= j; ++v)
    for (long u = -j; u <= j; ++u)
      taps[n++] = std::exp(-(static_cast<double>(u) * u + v * v) / (2.0 * sg * sg)) / (2.0 * kPi * sg * sg);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t npix = w * h;
  StreamAlloc table(s), plane(s);
  if ((rc = table.upload(taps.data(), taps.size() * sizeof(double), "selective blur: table upload"))) return rc;
  if ((rc = plane.alloc(npix * sizeof(double), "selective blur: intensity plane"))) return rc;
  const double *d_taps = table.as<double>();
  double *d_lum = plane.as<double>();
  const unsigned pgrid = static_cast<unsigned>((npix + 255) / 256);
  dim3 grid(static_cast<unsigned>((w + 127) / 128), static_cast<unsigned>(h));
  const int iw = static_cast<int>(w), ih = static_cast<int>(h), iW = static_cast<int>(W);
  return with_channels(channels, "selective blur", [&](auto ch) {
    intensity_plane_kernel<ch()><<<pgrid, 256, 0, s>>>(src, d_lum, npix);
    selective_blur_kernel<ch()><<<grid, 128, 0, s>>>(src, d_lum, dst, iw, ih, iW, d_taps, threshold);
    return launch_status("selective blur launch", 2);
  });
}

namespace {

// one ConvolveMorphology stage with the kernel's cells reflected on the host (morphology.c:2612-2626)
int exact_convolve(const float *src, float *dst, size_t w, size_t h, int channels, const mb200_kernel_info *k, cudaStream_t s) {
  const size_t n = k->width * k->height;
  std::vector<double> cells(n);
  for (size_t i = 0; i < n; ++i) {
    if (k->values[i] != k->values[i]) return fail(MB200_EUNSUPPORTED, "adaptive: kernel with NaN cells");
    cells[i] = k->values[n - 1 - i];
  }
  StreamAlloc table(s);
  const int rc = table.upload(cells.data(), cells.size() * sizeof(double), "adaptive: table upload");
  if (rc) return rc;
  const int iw = static_cast<int>(w), ih = static_cast<int>(h), kw = static_cast<int>(k->width), kh = static_cast<int>(k->height);
  const int ox = kw - static_cast<int>(k->x) - 1, oy = kh - static_cast<int>(k->y) - 1;
  const dim3 grid(static_cast<unsigned>((iw + 127) / 128), static_cast<unsigned>(ih));
  return with_channels(channels, "adaptive", [&](auto ch) {
    exact_convolve_kernel<ch()><<<grid, 128, 0, s>>>(src, dst, iw, ih, table.as<const double>(), kw, kh, ox, oy);
    return launch_status("adaptive: convolution launch");
  });
}

// AutoLevelImage with the default channel mask (enhance.c:266 -> histogram.c:942-953): level.cu's MinMaxStretchImage,
// whose GetImageRange drops a row that starts with NaN as the reference does
int auto_level(float *buf, size_t w, size_t h, int channels, cudaStream_t s) {
  return launch_minmax_stretch(buf, w, h, channels, 0.0, 0.0, 1.0, false, (1u << channels) - 1u, s);
}

}  // namespace

int launch_adaptive(const float *src, float *dst, size_t w, size_t h, int channels, double radius, double sigma, int sharpen,
                    void *stream) {
  int rc = check_image(src, dst, w, h, channels, "adaptive blur / sharpen");
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t n = w * h * static_cast<size_t>(channels);
  if (std::fabs(sigma) < kEps) {                                     // effect.c:171: a plain clone
    const cudaError_t e = cudaMemcpyAsync(dst, src, n * sizeof(float), cudaMemcpyDeviceToDevice, s);
    return e == cudaSuccess ? MB200_OK : cuda_fail(e, "adaptive: copy");
  }
  const size_t width = mb200_optimal_kernel_width_2d(radius, sigma);
  if (width > 255) return fail(MB200_EUNSUPPORTED, "adaptive: window larger than 255");
  // kernel pyramid (effect.c:199-236), libm on the host like the reference
  const double kPi = 3.14159265358979323846264338327950288419716939937510;
  const double sg = std::fabs(sigma) < kEps ? kEps : sigma;
  std::vector<double> kernels;
  std::vector<int> offsets;
  for (size_t jw = 0; jw < width; jw += 2) {
    const long size = static_cast<long>(width - jw), j = (size - 1) / 2;
    const size_t base = kernels.size();
    offsets.push_back(static_cast<int>(base));
    double normalize = 0.0;
    for (long v = -j; v <= j; ++v)
      for (long u = -j; u <= j; ++u) {
        const double g = std::exp(-(static_cast<double>(u) * u + v * v) / (2.0 * sg * sg)) / (2.0 * kPi * sg * sg);
        kernels.push_back(sharpen ? -g : g);
        normalize += kernels.back();
      }
    const size_t centre = base + (kernels.size() - base - 1) / 2;
    if (sharpen) kernels[centre] = (-2.0) * normalize;
    else kernels[centre] += 1.0 - normalize;
    if (sigma < kEps) kernels[centre] = 1.0;
  }
  const KernelList edge_k(mb200_edge_kernel(radius)), blur_k = blur_kernel_pair(radius, sigma);
  if (!edge_k || !blur_k) return fail(MB200_ENOMEM, "adaptive: kernels");

  StreamAlloc edge(s), tmp(s), d_offsets(s), d_kernels(s);
  if ((rc = edge.alloc(n * sizeof(float), "adaptive: temporary")) || (rc = tmp.alloc(n * sizeof(float), "adaptive: temporary")))
    return rc;
  float *d_edge = edge.as<float>(), *d_tmp = tmp.as<float>();
  // EdgeImage -> AutoLevel -> BlurImage (row kernel, then the rotated one: float intermediate) -> AutoLevel
  if ((rc = exact_convolve(src, d_edge, w, h, channels, edge_k.get(), s))) return rc;
  if ((rc = auto_level(d_edge, w, h, channels, s))) return rc;
  if ((rc = exact_convolve(d_edge, d_tmp, w, h, channels, blur_k.get(), s))) return rc;
  if ((rc = exact_convolve(d_tmp, d_edge, w, h, channels, blur_k->next, s))) return rc;
  if ((rc = auto_level(d_edge, w, h, channels, s))) return rc;

  if ((rc = d_kernels.upload(kernels.data(), kernels.size() * sizeof(double), "adaptive: table upload")) ||
      (rc = d_offsets.upload(offsets.data(), offsets.size() * sizeof(int), "adaptive: offsets upload")))
    return rc;
  dim3 grid(static_cast<unsigned>((w + 127) / 128), static_cast<unsigned>(h));
  const int iw = static_cast<int>(w), ih = static_cast<int>(h), iwidth = static_cast<int>(width);
  return with_channels(channels, "adaptive", [&](auto ch) {
    adaptive_kernel<ch()><<<grid, 128, 0, s>>>(src, d_edge, dst, iw, ih, iwidth, d_kernels.as<const double>(),
                                              d_offsets.as<const int>());
    return launch_status("adaptive: launch");
  });
}

}  // namespace mb200
