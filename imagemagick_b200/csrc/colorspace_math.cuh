// colorspace_math.cuh -- the plain (untabled) device forms of the reference's colour helpers, shared by
// TransformImageColorspace (colorspace.cu) and the enhance operators (enhance.cu): DecodePixelGamma / EncodePixelGamma
// (pixel.c:318, :445), ConvertXYZToRGB (colorspace-private.h:72), XYZ <-> Lab / Luv for a given reference white
// (:531-557, :600-625, :1066-1089, :1138-1161) and PerceptibleReciprocal (pixel-accessor.h:242).
// The __constant__ tables here are initialised statically: every translation unit that includes this has its own copy.
#pragma once

#include "mb200_internal.h"
#include "quantum.cuh"

#include <cuda_runtime.h>

namespace mb200 {
namespace {

// Double constants of the sRGB -> XYZ -> Lab path as a __constant__ block: a literal double costs two MOV-immediates
// every time the compiler rematerialises it (ncu r02: 147 of the kernel's 576 SASS instructions were moves and the
// kernel issued 331 instructions per pixel at 87 % issue utilisation); a constant-bank operand costs nothing.
struct LabConstants {
  double third, qs, qr, toe_limit, inv_12_92, c055, inv_1055, four, three;
  double m[3][3];
  double inv_ill_x, inv_ill_z, cie_eps, c116, c16, inv100, c500, c200, inv255, half;
  // folded forms of the sRGB -> Lab leg (see rgb_to_lab_unit): decode to [0, 1], white point inside the matrix rows,
  // QuantumRange inside the L / a / b scale factors
  double toe_unit, slope_unit, offset_unit, two_thirds;
  double mw[3][3];
  double l_scale, a_scale, b_scale, half_qr;
};
__constant__ LabConstants kk = {
    1.0 / 3.0, 1.0 / 65535.0, 65535.0, 0.0404482362771076 * 65535.0, 1.0 / 12.92, 0.055, 1.0 / 1.055, 4.0, 3.0,
    {{0.4123955889674142161, 0.3575834307637148171, 0.1804926473817015735},
     {0.2125862307855955516, 0.7151703037034108499, 0.07220049864333622685},
     {0.01929721549174694484, 0.1191838645808485318, 0.9504971251315797660}},
    1.0 / 0.95047, 1.0 / 1.08883, 216.0 / 24389.0, 116.0, 16.0, 1.0 / 100.0, 500.0, 200.0, 1.0 / 255.0, 0.5,
    (1.0 / 65535.0) / 12.92, (1.0 / 65535.0) / 1.055, 0.055 / 1.055, 2.0 / 3.0,
    {{0.4123955889674142161 / 0.95047, 0.3575834307637148171 / 0.95047, 0.1804926473817015735 / 0.95047},
     {0.2125862307855955516, 0.7151703037034108499, 0.07220049864333622685},
     {0.01929721549174694484 / 1.08883, 0.1191838645808485318 / 1.08883, 0.9504971251315797660 / 1.08883}},
    65535.0 / 100.0, 65535.0 * 500.0 / 255.0, 65535.0 * 200.0 / 255.0, 0.5 * 65535.0};

__constant__ double kDecodeCf[9] = {1.7917488588043277509, 0.82045614371976854984, 0.027694100686325412819,
                                    -0.00094244335181762134018, 0.000064355540911469709545,
                                    -5.7224404636060757485e-06, 5.8767669437311184313e-07,
                                    -6.6139920053589721168e-08, 7.9323242696227458163e-09};
__constant__ double kDecodeP2[5] = {1.0, 2.6390158215457883983, 6.9644045063689921093, 1.8379173679952558018e+01,
                                    4.8502930128332728543e+01};
__constant__ double kEncodeCf[9] = {1.1758200232996901923, 0.16665763094889061230, -0.0083154894939042125035,
                                    0.00075187976780420279038, -0.000083240178519391795367,
                                    0.000010229209410070008679, -1.3400466409860246e-06,
                                    1.8333422241635376682e-07, -2.5878596761348859722e-08};
__constant__ double kEncodeP2[12] = {1.0, 1.3348398541700343678, 1.7817974362806785482, 2.3784142300054420538,
                                     3.1748021039363991669, 4.2378523774371812394, 5.6568542494923805819,
                                     7.5509945014535482244, 1.0079368399158985525e1, 1.3454342644059433809e1,
                                     1.7959392772949968275e1, 2.3972913230026907883e1};

// The reference evaluates its degree-8 Chebyshev series term by term (term[i] = 2*t1*term[i-1] - term[i-2];
// p = sum cf[i]*term[i], pixel.c:299-309): 16 FP64 operations.  The same polynomial in the monomial basis (the
// coefficients below are the exact rational conversion of kDecodeCf / kEncodeCf rounded to double) needs 8 FMAs
// in Horner form and agrees with the term-by-term value to 8.7e-16 relative over the whole argument range
// [-1, 1] -- eight orders of magnitude below the float ULP the result is rounded to.
__constant__ double kDecodeMono[9] = {1.7641185339145438, 0.8232553245523438, 0.05488368139148116,
                                      -0.0036590284335213646, 0.000487905017844988, -8.415137637169515e-05,
                                      1.6774979206916156e-05, -4.232954883429742e-06, 1.0153375065117114e-06};
__constant__ double kEncodeMono[9] = {1.1840535867831192, 0.16445185435297144, -0.015988350284094677,
                                      0.002813201599470727, -0.000605739764869621, 0.00014313391765048851,
                                      -3.6256571740647474e-05, 1.173339023464664e-05, -3.3124603854526542e-06};

__device__ __forceinline__ double cheb9(const double *mono, double t1) {
  double p = mono[8];
#pragma unroll
  for (int i = 7; i >= 0; --i) p = fma(p, t1, mono[i]);
  return p;
}

// frexp / ldexp for positive normal doubles (the only arguments the gamma curves see above their
// linear toe): pure exponent-field arithmetic on the high word.
__device__ __forceinline__ double frexp_normal(double x, int *e) {
  const int hi = __double2hiint(x);
  *e = ((hi >> 20) & 0x7ff) - 1022;
  return __hiloint2double((hi & 0x800fffff) | 0x3fe00000, __double2loint(x));
}
__device__ __forceinline__ double ldexp_normal(double x, int n) {
  return __hiloint2double(__double2hiint(x) + (n << 20), __double2loint(x));
}
__device__ __forceinline__ void floor_divmod(int v, int d, int *quot, int *rem) {   // C div() + the reference's fix-up
  int q = v / d, r = v - q * d;
  if (r < 0) { q -= 1; r += d; }
  *quot = q; *rem = r;
}

__device__ __forceinline__ double decode_gamma(double x) {            // pixel.c:260-316
  int e, quot, rem;
  const double mant = frexp_normal(x, &e);
  const double p = cheb9(kDecodeMono, fma(kk.four, mant, -kk.three));
  floor_divmod(e - 1, 5, &quot, &rem);
  return x * ldexp_normal(kDecodeP2[rem] * p, 7 * quot);
}

__device__ __forceinline__ double encode_gamma(double x) {            // pixel.c:380-443
  int e, quot, rem;
  const double mant = frexp_normal(x, &e);
  const double p = cheb9(kEncodeMono, 4.0 * mant - 3.0);
  floor_divmod(e - 1, 12, &quot, &rem);
  return ldexp_normal(kEncodeP2[rem] * p, 5 * quot);
}

// NONFINITE: settle NaN and +inf the way the reference does (its frexp / Chebyshev chain turns both into NaN); the
// exponent-field frexp above assumes a finite argument.  -inf takes the linear toe in both.
template <bool NONFINITE = false>
__device__ __forceinline__ double decode_pixel_gamma(double pixel) {   // pixel.c:318
  if (pixel <= kk.toe_limit) return pixel * kk.inv_12_92;
  if (NONFINITE && !(pixel <= 1.7976931348623157e308)) return __longlong_as_double(0x7ff8000000000000LL);
  return kk.qr * decode_gamma(fma(kk.qs, pixel, kk.c055) * kk.inv_1055);
}

template <bool NONFINITE = false>
__device__ __forceinline__ double encode_pixel_gamma(double pixel) {   // pixel.c:445
  if (pixel <= (0.0031306684425005883 * QR)) return 12.92 * pixel;
  if (NONFINITE && !(pixel <= 1.7976931348623157e308)) return __longlong_as_double(0x7ff8000000000000LL);
  return QR * (1.055 * encode_gamma(QS * pixel) - 0.055);
}

constexpr double kIllX = 0.95047, kIllY = 1.00000, kIllZ = 1.08883;   // D65
constexpr double kCieEps = 216.0 / 24389.0, kCieK = 24389.0 / 27.0;

// t^(1/3) for t in (216/24389, 2) (~1.3 for in-range samples): z0 = 2^(-log2(t)/3) in fp32 (MUFU, ~2^-21), then one
// Newton step on z = t^(-1/3) folded into the result: t*z1^2 with z1 = z0*(1 + e/3) is w*(1 + 2e/3) + O(e^2), w = t*z0^2,
// e = 1 - w*z0 (|e| < 2^-20, so the dropped e^2/9 term is below 2^-43) -- five FP64 operations.
// (lg2 / ex2 as the bare MUFU instructions: t is in (0.0088, 2), so neither needs the range handling of log2f / exp2f,
// which costs two divergent-branch regions per call.  Other t: cube_root below.)
__device__ __forceinline__ double cube_root5(double t) {
  const float tf = static_cast<float>(t);
  float l, zf;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(l) : "f"(tf));
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(zf) : "f"(l * (-1.0f / 3.0f)));
  const double z0 = static_cast<double>(zf);
  const double w = t * (z0 * z0);
  const double e = fma(-w, z0, 1.0);
  return fma(w * e, kk.two_thirds, w);
}

// pow(t, 1/3) for every t above the CIE epsilon: cube_root5 below 2, the range of every sample up to ~1.35 QuantumRange;
// above, cbrt (1 double ULP), which differs from the reference's pow(t, 0.333...) by a relative 1.9e-17 * ln(t) < 1.4e-14.
// (The seed's error grows with |log2 t|: one Newton step leaves ~3e-11 relative at t = 2^73 and, from t ~ 2^128 -- HDRI
// samples from ~7e20 up -- (float) t overflows and the seed is 0.  Lab's a / b of a near-gray pixel is a difference of
// two cube roots, which brings such an error up to float precision.)
constexpr double kCubeRootSeedMax = 2.0;
__device__ __forceinline__ double cube_root(double t) { return t < kCubeRootSeedMax ? cube_root5(t) : cbrt(t); }

template <bool NONFINITE = false>
__device__ __forceinline__ void xyz_to_rgb(double X, double Y, double Z, double &R, double &G, double &B) {
  double r = (3.240969941904521 * X) + (-1.537383177570093 * Y) + (-0.498610760293 * Z);
  double g = (-0.96924363628087 * X) + (1.87596750150772 * Y) + (0.041555057407175 * Z);
  double b = (0.055630079696993 * X) + (-0.20397695888897 * Y) + (1.056971514242878 * Z);
  const double gb = g < b ? g : b;
  const double m = r < gb ? r : gb;
  if (m < 0.0) { r -= m; g -= m; b -= m; }
  R = encode_pixel_gamma<NONFINITE>(QR * r);
  G = encode_pixel_gamma<NONFINITE>(QR * g);
  B = encode_pixel_gamma<NONFINITE>(QR * b);
}

__device__ __forceinline__ double perceptible_reciprocal_d(double x) {       // pixel-accessor.h:242
  const double sign = x < 0.0 ? -1.0 : 1.0;
  return (sign * x) >= 1.0e-12 ? 1.0 / x : sign / 1.0e-12;
}
// Per-call settings of the XYZ-derived legs: the reference white (illuminant_tristimulus[], colorspace-private.h:32-46,
// selected by the "color:illuminant" artifact, colorspace.c:761-773; D65 by default) with the Luv white point derived
// from it (:608-624, :1150-1159), and Jzazbz's white luminance ("white-luminance" property, colorspace.c:996).
struct XyzSettings {
  double ill[3];
  double un, vn;
  double white_luminance;
};

// Lab in unit range (colorspace-private.h:1066-1089) and back (:531-557), for the polar LCHab space
__device__ __forceinline__ double lab_f(double t) { return t > kCieEps ? cube_root(t) : (kCieK * t + 16.0) / 116.0; }
__device__ __forceinline__ void xyz_to_lab_unit(const XyzSettings &st, double X, double Y, double Z, double &L, double &a, double &b) {
  const double x = lab_f(X / st.ill[0]), y = lab_f(Y / st.ill[1]), z = lab_f(Z / st.ill[2]);
  L = __dsub_rn(__dmul_rn(116.0, y), 16.0) / 100.0;
  a = (500.0 * (x - y)) / 255.0 + 0.5;
  b = (200.0 * (y - z)) / 255.0 + 0.5;
}
__device__ __forceinline__ void lab_to_xyz_d(const XyzSettings &st, double L, double a, double b, double &X, double &Y, double &Z) {
  double y = (L + 16.0) / 116.0;
  double x = y + a / 500.0, z = y - b / 200.0;
  x = (x * x * x) > kCieEps ? x * x * x : __dsub_rn(__dmul_rn(116.0, x), 16.0) / kCieK;
  y = L > (kCieK * kCieEps) ? y * y * y : L / kCieK;
  z = (z * z * z) > kCieEps ? z * z * z : __dsub_rn(__dmul_rn(116.0, z), 16.0) / kCieK;
  X = st.ill[0] * x; Y = st.ill[1] * y; Z = st.ill[2] * z;
}
__device__ __forceinline__ void xyz_to_luv_unit(const XyzSettings &st, double X, double Y, double Z, double &L, double &u, double &v) {
  double l = Y > kCieEps ? __dsub_rn(__dmul_rn(116.0, cube_root(Y)), 16.0) : kCieK * Y;
  const double alpha = perceptible_reciprocal_d(X + 15.0 * Y + 3.0 * Z);
  const double uu = 13.0 * l * (4.0 * alpha * X - st.un), vv = 13.0 * l * (9.0 * alpha * Y - st.vn);
  L = l / 100.0; u = (uu + 134.0) / 354.0; v = (vv + 140.0) / 262.0;
}
__device__ __forceinline__ void luv_to_xyz_d(const XyzSettings &st, double L, double u, double v, double &X, double &Y, double &Z) {
  if (L > (kCieK * kCieEps)) { const double t = (L + 16.0) / 116.0; Y = t * t * t; } else Y = L / kCieK;
  const double pu = ((52.0 * L * perceptible_reciprocal_d(u + 13.0 * L * st.un)) - 1.0) / 3.0;
  const double gamma = perceptible_reciprocal_d(pu - (-1.0 / 3.0));
  X = gamma * ((Y * ((39.0 * L * perceptible_reciprocal_d(v + 13.0 * L * st.vn)) - 5.0)) + 5.0 * Y);
  Z = (X * pu) - 5.0 * Y;
}
constexpr double kPiD = 3.14159265358979323846264338327950288419716939937510;

// Host side: the reference white of a call ("color:illuminant", D65 by default) and the Luv white point derived from it.
constexpr int kD65 = 5;          // IlluminantType (MagickCore/color.h:40-54); also what an unparsable artifact selects
inline int illuminant_of(const mb200_colorspace_options *o) {
  return (o && (o->set & MB200_CO_ILLUMINANT) && o->illuminant >= 0 && o->illuminant <= 10) ? o->illuminant : kD65;
}
inline XyzSettings xyz_settings(const mb200_colorspace_options *o) {
  static const double table[11][3] = {                            // colorspace-private.h:32-46
      {1.09850, 1.00000, 0.35585}, {0.99072, 1.00000, 0.85223}, {0.98074, 1.00000, 1.18232}, {0.96422, 1.00000, 0.82521},
      {0.95682, 1.00000, 0.92149}, {0.95047, 1.00000, 1.08883}, {0.94972, 1.00000, 1.22638}, {1.00000, 1.00000, 1.00000},
      {0.99186, 1.00000, 0.67393}, {0.95041, 1.00000, 1.08747}, {1.00962, 1.00000, 0.64350}};
  XyzSettings st;
  const double *t = table[illuminant_of(o)];
  st.ill[0] = t[0]; st.ill[1] = t[1]; st.ill[2] = t[2];
  const double den = t[0] + 15.0 * t[1] + 3.0 * t[2];
  st.un = 4.0 * t[0] / den;
  st.vn = 9.0 * t[1] / den;
  st.white_luminance = (o && (o->set & MB200_CO_WHITE_LUMINANCE)) ? o->white_luminance : 10000.0;
  return st;
}

}  // namespace
}  // namespace mb200
