// distort.cu -- DistortImage's sampling loop (MagickCore/distort.c:2474-2890) for the affine and perspective maps,
// through resample.c's elliptical weighted average (ResamplePixelColor :315-670, ClampUpAxes :716-960,
// ScaleResampleFilter :1000-1219) and pixel.c's InterpolatePixelInfo (Average / Bilinear / Integer, :5439-5700).
//
// One thread per output pixel.  This file is compiled with -fmad=false: every double operation is the reference's,
// unfused, in its order.  The map kind and the virtual-pixel family (edge clamp / one constant colour) are template
// parameters; the 1024-entry weight table and every per-call value travel in a __grid_constant__ parameter, so a call
// uploads nothing.  The reference's integer conversions are x86's: (ssize_t) / (int) of NaN or of an out-of-range value
// is the most negative integer, which CUDA's saturating cvt would not give.
#include "mb200_internal.h"
#include "quantum.cuh"

#include <climits>
#include <cmath>

namespace mb200 {
namespace {

constexpr double kEps = 1.0e-12;                  // MagickEpsilon
constexpr double kMaxValue = 1.79769313486231570e+308;   // MagickMaximumValue

struct Ellipse {                 // the part of ResampleFilter that ScaleResampleFilter sets
  double A, B, C, Ulimit, Vlimit, Uwidth, slope;
  int limit_reached;
};

struct Params {
  double lut[MB200_RESAMPLE_LUT];
  double coeff[9];
  double output_scaling, support, image_area;
  long long gx, gy;              // output page
  double sub_x, sub_y;           // the source page when bestfit, else 0
  long long sw, sh, dw, dh;
  int ch;
  Ellipse unit;                  // SetResampleFilter's ScaleResampleFilter(1, 0, 0, 1); the affine map's own below
  Ellipse affine;
  float vcol[4];                 // the constant virtual pixel, in the image's layout
  double invalid[4];             // the matte colour (red, green, blue, alpha)
  int invalid_alpha;             // the matte colour has an alpha trait
};

struct Pix { double r, g, b, a; };

__host__ __device__ inline double perceptible_reciprocal(double x) {
  const double sign = x < 0.0 ? -1.0 : 1.0;
  return (sign * x) >= kEps ? 1.0 / x : sign / kEps;
}

__device__ inline long long x86_ll(double x) {
  return (x >= -9223372036854775808.0 && x < 9223372036854775808.0) ? static_cast<long long>(x) : LLONG_MIN;
}
__device__ inline int x86_int(double x) {
  return (x > -2147483649.0 && x < 2147483648.0) ? static_cast<int>(x) : INT_MIN;
}
__device__ inline long long cast_double_to_long(double x) {     // CastDoubleToLong (image-private.h:67)
  if (isnan(x)) return 0;
  if (x < 0.0) { const double v = ceil(x); return v < -9223372036854775808.0 ? LLONG_MIN : static_cast<long long>(v); }
  const double v = floor(x);
  return v >= 9223372036854775808.0 ? LLONG_MAX : static_cast<long long>(v);
}

// ClampUpAxes + ScaleResampleFilter (resample.c:716-1219).  On a limit the previous ellipse stays, as in the reference.
// For the affine map that previous ellipse is SetResampleFilter's unit one, as it is in the reference.  A perspective
// pixel starts from the unit ellipse too, where the reference keeps whatever its OpenMP thread's previous pixel left
// (a schedule-dependent value): the two can differ only where (4AC - B^2) overflows, at |r| ~ 0 next to the horizon,
// and only under Edge / Undefined virtual pixels, whose miss test reads Ulimit / Vlimit on a limit.
__host__ __device__ inline void scale_filter(Ellipse &e, double support, double image_area, double dux, double duy,
                                             double dvx, double dvy) {
  e.limit_reached = 0;
  const double a = dux, b = duy, c = dvx, d = dvy;
  const double aa = a * a, bb = b * b, cc = c * c, dd = d * d;
  const double n11 = aa + bb, n12 = a * c + b * d, n21 = n12, n22 = cc + dd;
  const double det = a * d - b * c;
  const double twice_det = det + det;
  const double frobenius_squared = n11 + n22;
  const double discriminant = (frobenius_squared + twice_det) * (frobenius_squared - twice_det);
  const double sqrt_discriminant = sqrt(discriminant > 0.0 ? discriminant : 0.0);
  const double s1s1 = 0.5 * (frobenius_squared + sqrt_discriminant);
  const double s2s2 = 0.5 * (frobenius_squared - sqrt_discriminant);
  const double s1s1minusn11 = s1s1 - n11, s1s1minusn22 = s1s1 - n22;
  const double sq11 = s1s1minusn11 * s1s1minusn11, sq22 = s1s1minusn22 * s1s1minusn22;
  const double temp_u11 = sq11 >= sq22 ? n12 : s1s1minusn22;
  const double temp_u21 = sq11 >= sq22 ? s1s1minusn11 : n21;
  const double norm = sqrt(temp_u11 * temp_u11 + temp_u21 * temp_u21);
  const double u11 = norm > 0.0 ? temp_u11 / norm : 1.0;
  const double u21 = norm > 0.0 ? temp_u21 / norm : 0.0;
  const double major_mag = s1s1 <= 1.0 ? 1.0 : sqrt(s1s1);
  const double minor_mag = s2s2 <= 1.0 ? 1.0 : sqrt(s2s2);
  double major_x = u11, major_y = u21, minor_x = -u21, minor_y = u11;
  major_x *= major_mag; major_y *= major_mag;
  minor_x *= minor_mag; minor_y *= minor_mag;
  const double A = major_y * major_y + minor_y * minor_y;
  const double B = -2.0 * (major_x * major_y + minor_x * minor_y);
  const double C = major_x * major_x + minor_x * minor_x;
  double F = major_mag * minor_mag;
  F *= F;
  if ((4 * A * C - B * B) > kMaxValue) { e.limit_reached = 1; return; }
  F *= support;
  F *= support;
  e.Ulimit = sqrt(C * F / (A * C - 0.25 * B * B));
  e.Vlimit = sqrt(A * F / (A * C - 0.25 * B * B));
  e.Uwidth = sqrt(F / A);
  e.slope = -B / (2.0 * A);
  if ((e.Uwidth * e.Vlimit) > (4.0 * image_area)) { e.limit_reached = 1; return; }
  const double scale = static_cast<double>(MB200_RESAMPLE_LUT) * perceptible_reciprocal(F);
  e.A = A * scale;
  e.B = B * scale;
  e.C = C * scale;
}

// The virtual pixel at (x, y) as (red, green, blue, alpha): GetPixelRed/Green/Blue read the one gray slot of a gray
// image, and GetPixelAlpha is QuantumRange without an alpha channel.
template <bool kEdge>
__device__ inline Pix fetch(const Params &p, const float *__restrict__ src, long long x, long long y) {
  float v[4];
  const int ch = p.ch;
  if (x >= 0 && x < p.sw && y >= 0 && y < p.sh) {
    const float *q = src + (static_cast<size_t>(y) * static_cast<size_t>(p.sw) + static_cast<size_t>(x)) * ch;
    for (int c = 0; c < ch; ++c) v[c] = q[c];
  } else if (kEdge) {
    x = x < 0 ? 0 : (x >= p.sw ? p.sw - 1 : x);
    y = y < 0 ? 0 : (y >= p.sh ? p.sh - 1 : y);
    const float *q = src + (static_cast<size_t>(y) * static_cast<size_t>(p.sw) + static_cast<size_t>(x)) * ch;
    for (int c = 0; c < ch; ++c) v[c] = q[c];
  } else {
    for (int c = 0; c < ch; ++c) v[c] = p.vcol[c];
  }
  if (ch <= 2) return {v[0], v[0], v[0], ch == 2 ? static_cast<double>(v[1]) : QR};
  return {v[0], v[1], v[2], ch == 4 ? static_cast<double>(v[3]) : QR};
}

// AlphaBlendPixelInfo (pixel.c:5414)
__device__ inline Pix alpha_blend(const Pix &s, bool has_alpha, double *alpha) {
  if (!has_alpha) { *alpha = 1.0; return s; }
  *alpha = QS * s.a;
  return {*alpha * s.r, *alpha * s.g, *alpha * s.b, s.a};
}

// InterpolatePixelInfo: 0 Integer, 1 Average (4 neighbours), 2 Bilinear
template <bool kEdge>
__device__ Pix interpolate(const Params &p, const float *__restrict__ src, int method, double x, double y) {
  const long long xo = cast_double_to_long(floor(x)), yo = cast_double_to_long(floor(y));
  const bool has_alpha = p.ch == 2 || p.ch == 4;
  if (method == 0) return fetch<kEdge>(p, src, xo, yo);
  if (method == 1) {
    Pix out = {0.0, 0.0, 0.0, 0.0};
    for (int i = 0; i < 4; ++i) {
      double alpha;
      const Pix q = alpha_blend(fetch<kEdge>(p, src, xo + (i & 1), yo + (i >> 1)), has_alpha, &alpha);
      const double gamma = perceptible_reciprocal(alpha);
      out.r += gamma * q.r;
      out.g += gamma * q.g;
      out.b += gamma * q.b;
      out.a += q.a;
    }
    const double gamma = 1.0 / 4;
    out.r *= gamma; out.g *= gamma; out.b *= gamma; out.a *= gamma;
    return out;
  }
  Pix q[4];
  double alpha[4];
  for (int i = 0; i < 4; ++i) q[i] = alpha_blend(fetch<kEdge>(p, src, xo + (i & 1), yo + (i >> 1)), has_alpha, &alpha[i]);
  const double dx = x - xo, dy = y - yo, ex = 1.0 - dx, ey = 1.0 - dy;
  double gamma = ey * (ex * alpha[0] + dx * alpha[1]) + dy * (ex * alpha[2] + dx * alpha[3]);
  gamma = perceptible_reciprocal(gamma);
  Pix out;
  out.r = gamma * (ey * (ex * q[0].r + dx * q[1].r) + dy * (ex * q[2].r + dx * q[3].r));
  out.g = gamma * (ey * (ex * q[0].g + dx * q[1].g) + dy * (ex * q[2].g + dx * q[3].g));
  out.b = gamma * (ey * (ex * q[0].b + dx * q[1].b) + dy * (ex * q[2].b + dx * q[3].b));
  gamma = ey * (ex + dx) + dy * (ex + dx);
  gamma = perceptible_reciprocal(gamma);
  out.a = gamma * (ey * (ex * q[0].a + dx * q[1].a) + dy * (ex * q[2].a + dx * q[3].a));
  return out;
}

// ResamplePixelColor (resample.c:315-670).  Returns false where the reference's scan-line fetch fails.
template <bool kEdge>
__device__ bool resample(const Params &p, const double *lut, const float *__restrict__ src, const Ellipse &e, double u0,
                         double v0, Pix &pixel) {
  const double cols1 = static_cast<double>(p.sw) - 1.0, rows1 = static_cast<double>(p.sh) - 1.0;
  bool hit;
  if (!kEdge)
    hit = e.limit_reached || u0 + e.Ulimit < 0.0 || u0 - e.Ulimit > cols1 || v0 + e.Vlimit < 0.0 ||
          v0 - e.Vlimit > rows1;
  else
    hit = (u0 + e.Ulimit < 0.0 && v0 + e.Vlimit < 0.0) || (u0 + e.Ulimit < 0.0 && v0 - e.Vlimit > rows1) ||
          (u0 - e.Ulimit > cols1 && v0 + e.Vlimit < 0.0) || (u0 - e.Ulimit > cols1 && v0 - e.Vlimit > rows1);
  if (hit) { pixel = interpolate<kEdge>(p, src, 0, u0, v0); return true; }
  if (e.limit_reached) { pixel = interpolate<kEdge>(p, src, 1, u0, v0); return true; }   // Edge only
  const bool has_alpha = p.ch == 2 || p.ch == 4;
  long long hits = 0;
  double divisor_c = 0.0, divisor_m = 0.0;
  pixel.r = pixel.g = pixel.b = 0.0;
  if (has_alpha) pixel.a = 0.0;
  const long long v1 = x86_ll(ceil(v0 - e.Vlimit)), v2 = x86_ll(floor(v0 + e.Vlimit));
  double u1 = u0 + (v1 - v0) * e.slope - e.Uwidth;
  const long long uw = x86_ll(2.0 * e.Uwidth) + 1;
  if (uw <= 0 || uw > (1ll << 40)) return false;                 // GetCacheViewVirtualPixels cannot hold the line
  const double DDQ = 2 * e.A;
  for (long long v = v1; v <= v2; v++) {
    const long long u = x86_ll(ceil(u1));
    u1 += e.slope;
    const double U = static_cast<double>(u) - u0;
    const double V = static_cast<double>(v) - v0;
    double Q = (e.A * U + e.B * V) * U + e.C * V * V;
    double DQ = e.A * (2.0 * U + 1) + e.B * V;
    for (long long k = 0; k < uw; k++) {
      const int qi = x86_int(Q);
      if (qi >= 0 && qi < MB200_RESAMPLE_LUT) {
        double weight = lut[qi];
        const Pix s = fetch<kEdge>(p, src, u + k, v);
        pixel.a += weight * s.a;
        divisor_m += weight;
        if (has_alpha) weight *= QS * s.a;
        pixel.r += weight * s.r;
        pixel.g += weight * s.g;
        pixel.b += weight * s.b;
        divisor_c += weight;
        hits++;
      }
      Q += DQ;
      DQ += DDQ;
    }
  }
  if (hits == 0 || divisor_m <= kEps || divisor_c <= kEps) { pixel = interpolate<kEdge>(p, src, 2, u0, v0); return true; }
  divisor_m = 1.0 / divisor_m;
  if (has_alpha) pixel.a = static_cast<float>(divisor_m * pixel.a);
  divisor_c = 1.0 / divisor_c;
  pixel.r = static_cast<float>(divisor_c * pixel.r);
  pixel.g = static_cast<float>(divisor_c * pixel.g);
  pixel.b = static_cast<float>(divisor_c * pixel.b);
  return true;
}

// SetPixelViaPixelInfo: gray takes blue (red, green, then blue are written to the one slot); alpha is the pixel's when
// it has an alpha trait, else opaque.
__device__ inline void store(float *q, int ch, const Pix &v, bool alpha_trait) {
  const float a = alpha_trait ? static_cast<float>(v.a) : static_cast<float>(QR);
  if (ch <= 2) { q[0] = static_cast<float>(v.b); if (ch == 2) q[1] = a; return; }
  q[0] = static_cast<float>(v.r); q[1] = static_cast<float>(v.g); q[2] = static_cast<float>(v.b);
  if (ch == 4) q[3] = a;
}

template <bool kPerspective, bool kEdge>
__device__ void distort_pixel(const Params &p, const double *lut, const float *__restrict__ src,
                              float *__restrict__ dst, long long i, long long j) {
  const bool has_alpha = p.ch == 2 || p.ch == 4;
  const double *c = p.coeff;
  const double os = p.output_scaling;
  const double dx = static_cast<double>(p.gx + i + 0.5) * os;
  const double dy = static_cast<double>(p.gy + j + 0.5) * os;
  double sx, sy, validity = 1.0;
  Ellipse e = kPerspective ? p.unit : p.affine;
  if (!kPerspective) {
    sx = c[0] * dx + c[1] * dy + c[2];
    sy = c[3] * dx + c[4] * dy + c[5];
  } else {
    const double pp = c[0] * dx + c[1] * dy + c[2];
    const double n = c[3] * dx + c[4] * dy + c[5];
    const double r = c[6] * dx + c[7] * dy + 1.0;
    validity = (r * c[8] < 0.0) ? 0.0 : 1.0;
    const double abs_r = fabs(r) * 2, abs_c6 = fabs(c[6]), abs_c7 = fabs(c[7]);
    if (abs_c6 > abs_c7) {
      if (abs_r < abs_c6 * os) validity = 0.5 - c[8] * r / (c[6] * os);
    } else if (abs_r < abs_c7 * os) {
      validity = 0.5 - c[8] * r / (c[7] * os);
    }
    sx = dx;
    sy = dy;
    if (validity > 0.0) {
      double scale = 1.0 / r;
      sx = pp * scale;
      sy = n * scale;
      scale *= scale;
      scale_filter(e, p.support, p.image_area, os * ((r * c[0] - pp * c[6]) * scale), os * ((r * c[1] - pp * c[7]) * scale),
                   os * ((r * c[3] - n * c[6]) * scale), os * ((r * c[4] - n * c[7]) * scale));
    }
  }
  sx -= p.sub_x;
  sy -= p.sub_y;
  sx -= 0.5;
  sy -= 0.5;
  float *q = dst + (static_cast<size_t>(j) * static_cast<size_t>(p.dw) + static_cast<size_t>(i)) * p.ch;
  const Pix invalid = {p.invalid[0], p.invalid[1], p.invalid[2], p.invalid[3]};
  if (validity <= 0.0) { store(q, p.ch, invalid, p.invalid_alpha); return; }
  Pix pixel = {0.0, 0.0, 0.0, QR};
  if (!resample<kEdge>(p, lut, src, e, sx, sy, pixel)) { store(q, p.ch, invalid, p.invalid_alpha); return; }
  if (validity < 1.0) {          // CompositePixelInfoBlend (composite-private.h:180) -> CompositePixelInfoPlus
    const double Sa = QS * (validity * pixel.a), Da = QS * ((1.0 - validity) * invalid.a);
    double gamma = Sa + Da;
    gamma = gamma < 0.0 ? 0.0 : (gamma > 1.0 ? 1.0 : gamma);
    pixel.a = QR * (gamma < 0.0 ? 0.0 : (gamma > 1.0 ? 1.0 : gamma));
    gamma = perceptible_reciprocal(gamma);
    pixel.r = gamma * (Sa * pixel.r + Da * invalid.r);
    pixel.g = gamma * (Sa * pixel.g + Da * invalid.g);
    pixel.b = gamma * (Sa * pixel.b + Da * invalid.b);
  }
  store(q, p.ch, pixel, has_alpha);
}

// The weight table is indexed per lane by a data-dependent Q; from shared memory, divergent indices cost bank
// conflicts at worst instead of serialising on the constant bank.  Rows are a grid-stride loop, so any height runs.
template <bool kPerspective, bool kEdge>
__global__ void __launch_bounds__(128) distort_kernel(const __grid_constant__ Params p, const float *__restrict__ src,
                                                      float *__restrict__ dst) {
  __shared__ double lut[MB200_RESAMPLE_LUT];
  for (int k = threadIdx.x; k < MB200_RESAMPLE_LUT; k += blockDim.x) lut[k] = p.lut[k];
  __syncthreads();
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= p.dw) return;
  for (long long j = blockIdx.y; j < p.dh; j += gridDim.y) distort_pixel<kPerspective, kEdge>(p, lut, src, dst, i, j);
}

}  // namespace

int distort_check(size_t width, size_t height, int channels, const mb200_distort_params *plan,
                  const mb200_resample_options *o) {
  if (!plan || !o || width == 0 || height == 0 || channels < 1 || channels > 4 || plan->columns == 0 || plan->rows == 0 ||
      (plan->map != MB200_DistortAffineMap && plan->map != MB200_DistortPerspectiveMap))
    return fail(MB200_EINVAL, "distort: bad arguments");
  if (plan->columns > (1u << 30))
    return fail(MB200_EUNSUPPORTED, "distort: outputs wider than 2^30 columns are not supported");
  if (o->filter == MB200_PointFilter)
    return fail(MB200_EUNSUPPORTED, "distort: the Point filter interpolates every pixel");
  if (o->interpolate != 0 && o->interpolate != 5)
    return fail(MB200_EUNSUPPORTED, "distort: interpolate method %d is not implemented", o->interpolate);
  switch (o->virtual_pixel) {
    case 0: case 1: case 3: case 7: case 9: case 10: case 11: break;
    default: return fail(MB200_EUNSUPPORTED, "distort: virtual-pixel method %d is not implemented", o->virtual_pixel);
  }
  if (plan->map == MB200_DistortPerspectiveMap && (channels == 1 || channels == 3)) {
    // the horizon blend band |2 r| < |c6| or |c7| times output_scaling, against r over the output's corners
    const double *c = plan->coeff;
    const double os = plan->output_scaling;
    const double t = (std::fabs(c[6]) > std::fabs(c[7]) ? std::fabs(c[6]) : std::fabs(c[7])) * os;
    double lo = INFINITY, hi = -INFINITY;
    for (int k = 0; k < 4; ++k) {
      const double x = (static_cast<double>(plan->page_x) + ((k & 1) ? static_cast<double>(plan->columns) : 0.0)) * os;
      const double y = (static_cast<double>(plan->page_y) + ((k & 2) ? static_cast<double>(plan->rows) : 0.0)) * os;
      const double r = 2.0 * (c[6] * x + c[7] * y + 1.0);
      lo = r < lo ? r : lo;
      hi = r > hi ? r : hi;
    }
    if (!(hi <= -t || lo >= t))
      return fail(MB200_EUNSUPPORTED, "distort: the horizon blend of an image without alpha is not implemented");
  }
  return MB200_OK;
}

int launch_distort(const float *src, size_t width, size_t height, int channels, float *dst,
                   const mb200_distort_params *plan, const mb200_resample_options *o, void *stream) {
  Params p;
  int rc = mb200_resample_filter_lut(o->filter, o->filter_options, p.lut, &p.support);
  if (rc) return rc;
  for (int k = 0; k < 9; ++k) p.coeff[k] = plan->coeff[k];
  p.output_scaling = plan->output_scaling;
  p.image_area = static_cast<double>(static_cast<long long>(width * height));
  p.gx = plan->page_x;
  p.gy = plan->page_y;
  p.sub_x = plan->bestfit ? static_cast<double>(plan->src_page_x) : 0.0;
  p.sub_y = plan->bestfit ? static_cast<double>(plan->src_page_y) : 0.0;
  p.sw = static_cast<long long>(width);
  p.sh = static_cast<long long>(height);
  p.dw = static_cast<long long>(plan->columns);
  p.dh = static_cast<long long>(plan->rows);
  p.ch = channels;
  p.unit = {};
  scale_filter(p.unit, p.support, p.image_area, 1.0, 0.0, 0.0, 1.0);
  p.affine = p.unit;
  if (plan->map == MB200_DistortAffineMap)
    scale_filter(p.affine, p.support, p.image_area, p.output_scaling * p.coeff[0], p.output_scaling * p.coeff[1],
                 p.output_scaling * p.coeff[3], p.output_scaling * p.coeff[4]);
  // cache.c:2851-2890: the constant virtual pixel; SetPixelRed / Green / Blue all land in a gray image's one slot
  double rgba[4] = {0.0, 0.0, 0.0, QR};
  switch (o->virtual_pixel) {
    case 1: for (int k = 0; k < 4; ++k) rgba[k] = o->background[k]; break;
    case 7: rgba[3] = 0.0; break;
    case 10: rgba[0] = rgba[1] = rgba[2] = static_cast<double>(static_cast<float>(QR / 2)); break;
    case 11: rgba[0] = rgba[1] = rgba[2] = QR; break;
    default: break;
  }
  if (channels <= 2) { p.vcol[0] = static_cast<float>(rgba[2]); p.vcol[1] = static_cast<float>(rgba[3]); }
  else for (int k = 0; k < 4; ++k) p.vcol[k] = static_cast<float>(rgba[k]);
  for (int k = 0; k < 4; ++k) p.invalid[k] = o->matte[k];
  p.invalid_alpha = o->matte_alpha ? 1 : 0;
  const bool edge = o->virtual_pixel == 0 || o->virtual_pixel == 3;
  const bool persp = plan->map == MB200_DistortPerspectiveMap;
  const dim3 block(128), grid(static_cast<unsigned>((plan->columns + 127) / 128),
                                static_cast<unsigned>(plan->rows < 65535u ? plan->rows : 65535u));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (persp && edge) distort_kernel<true, true><<<grid, block, 0, s>>>(p, src, dst);
  else if (persp) distort_kernel<true, false><<<grid, block, 0, s>>>(p, src, dst);
  else if (edge) distort_kernel<false, true><<<grid, block, 0, s>>>(p, src, dst);
  else distort_kernel<false, false><<<grid, block, 0, s>>>(p, src, dst);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "distort launch");
  count_family(kDistort);
  return MB200_OK;
}

}  // namespace mb200
