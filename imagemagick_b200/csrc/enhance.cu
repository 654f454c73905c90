// enhance.cu -- the in-place point operators behind the reference's in-place accelerate hooks (accelerate-private.h:50-60):
//   ContrastImage   MagickCore/enhance.c:1370-1505   HSB brightness pushed along a sine, ClampToQuantum (HDRI: a float cast)
//   ModulateImage   enhance.c:3461-3910              one hue / saturation / brightness leg out and back
//   GrayscaleImage  enhance.c:2474-2650              the PixelIntensityMethod of R, G, B into the gray channel
//   FunctionImage   MagickCore/statistic.c:979-1170  Polynomial / Sinusoid / Arcsin / Arctan on every Update channel
//
// One thread per pixel, in place.  RGBA buffers on a 16-byte boundary move as float4, everything else per channel.  Gray
// images (1 or 2 channels) give the red, green and blue accessors the same gray sample, so the three SetPixel* calls of
// Contrast and Modulate write one slot and the blue result is the one that stays.
//
// Every operation whose result a branch depends on is the reference's own IEEE double operation in its order, unfused
// (the hexcone.cuh legs, Polynomial, the Grayscale means); sin / asin / atan / atan2 / cos come from the CUDA math library
// instead of glibc (<= 1 ULP of the float Quantum), as do the gamma curves and cube roots of colorspace_math.cuh.
#include "mb200_internal.h"
#include "colorspace_math.cuh"
#include "hexcone.cuh"

#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>

namespace mb200 {
namespace {

constexpr double kMagickPI = 3.14159265358979323846264338327950288419716939937510;

template <int CH, bool VEC>
__device__ __forceinline__ void load_px(const float *q, float (&v)[4]) {
  if (VEC) {
    const float4 t = *reinterpret_cast<const float4 *>(q);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  } else {
#pragma unroll
    for (int c = 0; c < CH; ++c) v[c] = q[c];
  }
}
template <int CH, bool VEC>
__device__ __forceinline__ void store_px(float *q, const float (&v)[4]) {
  if (VEC) *reinterpret_cast<float4 *>(q) = make_float4(v[0], v[1], v[2], v[3]);
  else {
#pragma unroll
    for (int c = 0; c < CH; ++c) q[c] = v[c];
  }
}
// GetPixelRed / Green / Blue: the gray sample on gray images
template <int CH>
__device__ __forceinline__ void get_rgb(const float (&v)[4], double &r, double &g, double &b) {
  r = v[0];
  g = CH >= 3 ? v[1] : v[0];
  b = CH >= 3 ? v[2] : v[0];
}
// SetPixelRed / Green / Blue (ClampToQuantum, HDRI: a float cast); on gray images all three write the gray slot, blue last
template <int CH>
__device__ __forceinline__ void set_rgb(float (&v)[4], const Triple &o) {
  if (CH >= 3) { v[0] = static_cast<float>(o.x); v[1] = static_cast<float>(o.y); v[2] = static_cast<float>(o.z); }
  else v[0] = static_cast<float>(o.z);
}

// ------------------------------------------------------------------------------------------------ ContrastImage
template <int CH, bool VEC>
__global__ void __launch_bounds__(256) contrast_kernel(float *buf, size_t npixels, double half_sign) {
  const size_t i = static_cast<size_t>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= npixels) return;
  float *q = buf + i * CH;
  float v[4];
  load_px<CH, VEC>(q, v);
  double r, g, b;
  get_rgb<CH>(v, r, g, b);
  const Triple t = to_hsb(r, g, b);                                                                      // enhance.c:1381
  // brightness += 0.5*sign*(0.5*(sin(MagickPI*(brightness-0.5))+1.0)-brightness)
  double brightness = ad(t.z, ml(half_sign, sb(ml(0.5, ad(sin(ml(kMagickPI, sb(t.z, 0.5))), 1.0)), t.z)));
  if (brightness > 1.0) brightness = 1.0;
  else if (brightness < 0.0) brightness = 0.0;
  set_rgb<CH>(v, from_hsb(t.x, t.y, brightness));
  store_px<CH, VEC>(q, v);
}

// ------------------------------------------------------------------------------------------------ ModulateImage
enum ModulateSpace { kModHCL, kModHCLp, kModHSB, kModHSI, kModHSL, kModHSV, kModHWB, kModLCHab, kModLCHuv };
struct ModulateArgs {
  int space;
  double hue_shift;          // fmod(percent_hue - 100, 200) / 200
  double brightness, saturation;   // 0.01 * percent
  XyzSettings st;            // the LCH spaces' reference white
};

__device__ __forceinline__ void rgb_to_xyz_plain(double R, double G, double B, double &X, double &Y, double &Z) {   // :759
  const double r = QS * decode_pixel_gamma<true>(R), g = QS * decode_pixel_gamma<true>(G), b = QS * decode_pixel_gamma<true>(B);
  X = kk.m[0][0] * r + kk.m[0][1] * g + kk.m[0][2] * b;
  Y = kk.m[1][0] * r + kk.m[1][1] * g + kk.m[1][2] * b;
  Z = kk.m[2][0] * r + kk.m[2][1] * g + kk.m[2][2] * b;
}

// ModulateLCHab / ModulateLCHuv (enhance.c:3594-3630): the chroma is scaled with its +0.5 offset
template <bool UV>
__device__ __noinline__ Triple modulate_lch(double r, double g, double b, const ModulateArgs &a) {
  double X, Y, Z, luma, chroma, hue;
  rgb_to_xyz_plain(r, g, b, X, Y, Z);
  if (UV) {                                                                   // colorspace-private.h:1163-1176
    double u, v;
    xyz_to_luv_unit(a.st, X, Y, Z, luma, u, v);
    const double du = 354.0 * u - 134.0, dv = 262.0 * v - 140.0;
    chroma = hypot(du, dv) / 255.0 + 0.5;
    hue = 180.0 * atan2(dv, du) / kPiD / 360.0;
  } else {                                                                    // :1104-1117
    double la, lb;
    xyz_to_lab_unit(a.st, X, Y, Z, luma, la, lb);
    chroma = hypot(la - 0.5, lb - 0.5) + 0.5;
    hue = 180.0 * atan2(lb - 0.5, la - 0.5) / kPiD / 360.0;
  }
  if (hue < 0.0) hue += 1.0;
  luma *= a.brightness;
  chroma *= a.saturation;
  hue += a.hue_shift;
  const double L = 100.0 * luma, C = 255.0 * (chroma - 0.5), rad = kPiD * (360.0 * hue) / 180.0;   // :572-653
  if (UV) luv_to_xyz_d(a.st, L, C * cos(rad), C * sin(rad), X, Y, Z);
  else lab_to_xyz_d(a.st, L, C * cos(rad), C * sin(rad), X, Y, Z);
  Triple o;
  xyz_to_rgb<true>(X, Y, Z, o.x, o.y, o.z);
  return o;
}

template <int CH, bool VEC>
__global__ void __launch_bounds__(256) modulate_kernel(float *buf, size_t npixels, const ModulateArgs a) {
  const size_t i = static_cast<size_t>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= npixels) return;
  float *q = buf + i * CH;
  float v[4];
  load_px<CH, VEC>(q, v);
  double r, g, b;
  get_rgb<CH>(v, r, g, b);
  Triple t, o;
  switch (a.space) {          // ModulateHCL ... ModulateHWB (enhance.c:3443-3592): hue += shift; the other two scaled
    case kModHCL: case kModHCLp:
      t = to_hcl(r, g, b);
      t.x = ad(t.x, a.hue_shift); t.y = ml(t.y, a.saturation); t.z = ml(t.z, a.brightness);
      o = a.space == kModHCL ? from_hcl<false>(t.x, t.y, t.z) : from_hcl<true>(t.x, t.y, t.z);
      break;
    case kModHSB:
      t = to_hsb(r, g, b);
      t.x = ad(t.x, a.hue_shift); t.y = ml(t.y, a.saturation); t.z = ml(t.z, a.brightness);
      o = from_hsb(t.x, t.y, t.z);
      break;
    case kModHSI:
      t = to_hsi(r, g, b);
      t.x = ad(t.x, a.hue_shift); t.y = ml(t.y, a.saturation); t.z = ml(t.z, a.brightness);
      o = from_hsi(t.x, t.y, t.z);
      break;
    case kModHSV:
      t = to_hsl_hsv<true>(r, g, b);
      t.x = ad(t.x, a.hue_shift); t.y = ml(t.y, a.saturation); t.z = ml(t.z, a.brightness);
      o = from_hsl_hsv<true>(t.x, t.y, t.z);
      break;
    case kModHWB:             // (hue, whiteness, blackness): blackness takes the brightness factor, whiteness the saturation's
      t = to_hwb(r, g, b);
      t.x = ad(t.x, a.hue_shift); t.y = ml(t.y, a.saturation); t.z = ml(t.z, a.brightness);
      o = from_hwb(t.x, t.y, t.z);
      break;
    case kModLCHab: o = modulate_lch<false>(r, g, b, a); break;
    case kModLCHuv: o = modulate_lch<true>(r, g, b, a); break;
    default:
      t = to_hsl_hsv<false>(r, g, b);
      t.x = ad(t.x, a.hue_shift); t.y = ml(t.y, a.saturation); t.z = ml(t.z, a.brightness);
      o = from_hsl_hsv<false>(t.x, t.y, t.z);
      break;
  }
  set_rgb<CH>(v, o);
  store_px<CH, VEC>(q, v);
}

// ------------------------------------------------------------------------------------------------ GrayscaleImage
enum GammaStep { kNoGamma, kEncode, kDecode };

template <int CH, bool VEC>
__global__ void __launch_bounds__(256) grayscale_kernel(float *buf, size_t npixels, int method, int gamma) {
  const size_t i = static_cast<size_t>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= npixels) return;
  float *q = buf + i * CH;
  float v[4];
  load_px<CH, VEC>(q, v);
  double r, g, b;
  get_rgb<CH>(v, r, g, b);
  if (gamma == kEncode) { r = encode_pixel_gamma<true>(r); g = encode_pixel_gamma<true>(g); b = encode_pixel_gamma<true>(b); }
  else if (gamma == kDecode) { r = decode_pixel_gamma<true>(r); g = decode_pixel_gamma<true>(g); b = decode_pixel_gamma<true>(b); }
  const double hi = (r > g ? r : g) > b ? (r > g ? r : g) : b;            // MagickMax(MagickMax(red,green),blue)
  const double lo = (r < g ? r : g) < b ? (r < g ? r : g) : b;
  double intensity;
  switch (method) {                                                       // enhance.c:2547-2633
    case MB200_AveragePixelIntensityMethod: intensity = dv(ad(ad(r, g), b), 3.0); break;
    case MB200_BrightnessPixelIntensityMethod: intensity = hi; break;
    case MB200_LightnessPixelIntensityMethod: intensity = dv(ad(lo, hi), 2.0); break;
    case MB200_MSPixelIntensityMethod: intensity = dv(ad(ad(ml(r, r), ml(g, g)), ml(b, b)), 3.0); break;
    case MB200_Rec601LumaPixelIntensityMethod: case MB200_Rec601LuminancePixelIntensityMethod:
      intensity = ad(ad(ml(0.298839, r), ml(0.586811, g)), ml(0.114350, b));
      break;
    case MB200_RMSPixelIntensityMethod:
      intensity = dv(__dsqrt_rn(ad(ad(ml(r, r), ml(g, g)), ml(b, b))), 1.7320508075688772);   // sqrt(3.0)
      break;
    default:                  // Rec709Luma, Rec709Luminance and Undefined
      intensity = ad(ad(ml(0.212656, r), ml(0.715158, g)), ml(0.072186, b));
      break;
  }
  v[0] = static_cast<float>(intensity);                                   // SetPixelGray: channel 0
  store_px<CH, VEC>(q, v);
}

// ------------------------------------------------------------------------------------------------ FunctionImage
struct FunctionArgs {
  double p[MB200_MAX_FUNCTION_PARAMETERS];
  int n, function;
  unsigned update_mask;
};

__device__ __forceinline__ double arg_or(const FunctionArgs &a, int k, double fallback) { return a.n > k ? a.p[k] : fallback; }

__device__ __forceinline__ float apply_function(float sample, const FunctionArgs &a) {      // statistic.c:962-1055
  const double pixel = sample;
  double result = 0.0;
  switch (a.function) {
    case MB200_PolynomialFunction:
      for (int k = 0; k < a.n; ++k) result = ad(ml(ml(result, QS), pixel), a.p[k]);
      result = ml(result, QR);
      break;
    case MB200_SinusoidFunction: {
      const double frequency = arg_or(a, 0, 1.0), phase = arg_or(a, 1, 0.0), amplitude = arg_or(a, 2, 0.5),
                   bias = arg_or(a, 3, 0.5);
      result = ml(QR, ad(ml(amplitude, sin(ml(2.0 * kMagickPI, ad(ml(ml(frequency, QS), pixel), dv(phase, 360.0))))), bias));
      break;
    }
    case MB200_ArcsinFunction: {
      const double width = arg_or(a, 0, 1.0), center = arg_or(a, 1, 0.5), range = arg_or(a, 2, 1.0), bias = arg_or(a, 3, 0.5);
      result = ml(ml(2.0, reciprocal(width)), sb(ml(QS, pixel), center));
      if (result <= -1.0) result = sb(bias, dv(range, 2.0));
      else if (result >= 1.0) result = ad(bias, dv(range, 2.0));
      else result = ad(ml(dv(range, kMagickPI), asin(result)), bias);
      result = ml(result, QR);
      break;
    }
    case MB200_ArctanFunction: {
      const double slope = arg_or(a, 0, 1.0), center = arg_or(a, 1, 0.5), range = arg_or(a, 2, 1.0), bias = arg_or(a, 3, 0.5);
      result = ml(ml(kMagickPI, slope), sb(ml(QS, pixel), center));
      result = ml(QR, ad(ml(dv(range, kMagickPI), atan(result)), bias));
      break;
    }
    default: break;           // UndefinedFunction writes 0
  }
  return static_cast<float>(result);
}

template <int CH, bool VEC>
__global__ void __launch_bounds__(256) function_kernel(float *buf, size_t npixels, const FunctionArgs a) {
  const size_t i = static_cast<size_t>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= npixels) return;
  float *q = buf + i * CH;
  float v[4];
  load_px<CH, VEC>(q, v);
#pragma unroll
  for (int c = 0; c < CH; ++c)
    if ((a.update_mask >> c) & 1u) v[c] = apply_function(v[c], a);
  store_px<CH, VEC>(q, v);
}

// One launch of KERNEL<CH, VEC> over the image: float4 only for 16-byte aligned RGBA.
template <template <int, bool> class K, typename... Args>
int launch_point(const char *what, float *buf, size_t npixels, int channels, void *stream, Args... args) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const unsigned blocks = static_cast<unsigned>((npixels + 255) / 256);
  const bool vec = channels == 4 && (reinterpret_cast<uintptr_t>(buf) & 15) == 0;
  switch (channels) {
    case 1: K<1, false>::launch(blocks, s, buf, npixels, args...); break;
    case 2: K<2, false>::launch(blocks, s, buf, npixels, args...); break;
    case 3: K<3, false>::launch(blocks, s, buf, npixels, args...); break;
    default:
      if (vec) K<4, true>::launch(blocks, s, buf, npixels, args...);
      else K<4, false>::launch(blocks, s, buf, npixels, args...);
      break;
  }
  count_launch();
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? MB200_OK : cuda_fail(e, what);
}

template <int CH, bool VEC> struct Contrast {
  static void launch(unsigned blocks, cudaStream_t s, float *buf, size_t n, double half_sign) {
    contrast_kernel<CH, VEC><<<blocks, 256, 0, s>>>(buf, n, half_sign);
  }
};
template <int CH, bool VEC> struct Modulate {
  static void launch(unsigned blocks, cudaStream_t s, float *buf, size_t n, ModulateArgs a) {
    modulate_kernel<CH, VEC><<<blocks, 256, 0, s>>>(buf, n, a);
  }
};
template <int CH, bool VEC> struct Grayscale {
  static void launch(unsigned blocks, cudaStream_t s, float *buf, size_t n, int method, int gamma) {
    grayscale_kernel<CH, VEC><<<blocks, 256, 0, s>>>(buf, n, method, gamma);
  }
};
template <int CH, bool VEC> struct Function {
  static void launch(unsigned blocks, cudaStream_t s, float *buf, size_t n, FunctionArgs a) {
    function_kernel<CH, VEC><<<blocks, 256, 0, s>>>(buf, n, a);
  }
};

}  // namespace

int launch_contrast(float *buf, size_t npixels, int channels, bool sharpen, void *stream) {
  const double half_sign = 0.5 * (sharpen ? 1 : -1);
  return launch_point<Contrast>("contrast launch", buf, npixels, channels, stream, half_sign);
}

int launch_modulate(float *buf, size_t npixels, int channels, double percent_brightness, double percent_saturation,
                    double percent_hue, int colorspace, int illuminant, void *stream) {
  ModulateArgs a;
  switch (colorspace) {                                    // enhance.c:3837-3887; anything else (and no artifact) is HSL
    case MB200_HCLColorspace: a.space = kModHCL; break;
    case MB200_HCLpColorspace: a.space = kModHCLp; break;
    case MB200_HSBColorspace: a.space = kModHSB; break;
    case MB200_HSIColorspace: a.space = kModHSI; break;
    case MB200_HSVColorspace: a.space = kModHSV; break;
    case MB200_HWBColorspace: a.space = kModHWB; break;
    case MB200_LCHColorspace: case MB200_LCHabColorspace: a.space = kModLCHab; break;
    case MB200_LCHuvColorspace: a.space = kModLCHuv; break;
    default: a.space = kModHSL; break;
  }
  // The per-pixel constants of the Modulate* helpers, once: the same IEEE values the reference computes per pixel
  a.hue_shift = std::fmod(percent_hue - 100.0, 200.0) / 200.0;
  a.brightness = 0.01 * percent_brightness;
  a.saturation = 0.01 * percent_saturation;
  mb200_colorspace_options o{};
  o.set = MB200_CO_ILLUMINANT;
  o.illuminant = illuminant;
  a.st = xyz_settings(&o);
  return launch_point<Modulate>("modulate launch", buf, npixels, channels, stream, a);
}

int launch_grayscale(float *buf, size_t npixels, int channels, int method, int image_colorspace, void *stream) {
  int gamma = kNoGamma;                                    // enhance.c:2575-2625
  const bool luminance = method == MB200_Rec601LuminancePixelIntensityMethod ||
                         method == MB200_Rec709LuminancePixelIntensityMethod;
  const bool luma = method == MB200_Rec601LumaPixelIntensityMethod || method == MB200_Rec709LumaPixelIntensityMethod ||
                    method == MB200_UndefinedPixelIntensityMethod;
  if (luma && image_colorspace == MB200_RGBColorspace) gamma = kEncode;
  if (luminance && image_colorspace == MB200_sRGBColorspace) gamma = kDecode;
  return launch_point<Grayscale>("grayscale launch", buf, npixels, channels, stream, method, gamma);
}

int launch_function(float *buf, size_t npixels, int channels, int function, size_t n, const double *params,
                    unsigned update_mask, void *stream) {
  FunctionArgs a{};
  for (size_t k = 0; k < n; ++k) a.p[k] = params[k];
  a.n = static_cast<int>(n);
  a.function = function;
  a.update_mask = update_mask;
  return launch_point<Function>("function launch", buf, npixels, channels, stream, a);
}

}  // namespace mb200
