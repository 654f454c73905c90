// colorspace.cu -- in-place per-pixel colourspace transforms.
//
// Semantics: TransformImageColorspace (MagickCore/colorspace.c:1751-1783):
//   forward  sRGBTransformImage generic branch :958-1054 (Lab, XYZ) and linear-RGB
//            branch :1164-1225;   inverse TransformsRGBImage generic :2296-2390 and
//            linear-RGB :2494-2550.
//   helpers  ConvertRGBToXYZ colorspace-private.h:759, ConvertXYZToLab :1066,
//            ConvertLabToXYZ :531, ConvertXYZToRGB :72 (D65, :32-46),
//            DecodePixelGamma / EncodePixelGamma pixel.c:318 / :445 whose x^2.4 and
//            x^(1/2.4) are 9-term Chebyshev series on the frexp mantissa (pixel.c:260, :380).
// All arithmetic is FP64 following the reference's formulae.  Two rewrites keep the result within
// ~1e-15 relative of the reference's double value (a float ULP is 6e-8), but cut the FP64
// instruction count by more than half: divisions by constants (12.92, 1.055, the illuminant, 116,
// 100, 255 ...) become multiplications by the rounded reciprocal, and the reference's only libm
// call, pow(t,1/3), is a fp32 MUFU seed refined by one Newton step on t^(-1/3) in FP64.
// Alpha is untouched.  One thread per pixel, float4 access for RGBA; FP64-pipe bound.
#include "launch.cuh"
#include "colorspace_math.cuh"

#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <vector>

namespace mb200 {
namespace {

// kDecodeScale[e + 64] = kDecodeP2[(e-1) mod 5] * 2^(7 * floor((e-1)/5)) for the binary exponents e in [-64, 64): the
// reference's power table and ldexp folded into one exact factor (a power of two times a table entry), filled on the
// host once per device and copied to shared memory by every CTA -- the lanes of a warp index it with different
// exponents, which a constant-bank read would serialise, and the integer floor-division by 5 plus the exponent
// arithmetic (15 instructions per channel) disappears from a kernel that ncu shows to be issue-bound.
__constant__ double kDecodeScale[128];

// +inf settles like the reference's frexp / Chebyshev chain: NaN (decode_gamma's exponent-field frexp assumes a finite
// argument; a NaN argument stays NaN through its final product)
__device__ __noinline__ double decode_gamma_far(double x) {
  if (!(x <= 1.7976931348623157e308)) return __longlong_as_double(0x7ff8000000000000LL);
  return decode_gamma(x);
}

__device__ __forceinline__ double decode_gamma_tab(double x, const double *s_scale) {
  const int hi = __double2hiint(x);
  const int idx = ((hi >> 20) & 0x7ff) - (1022 - 64);
  if (static_cast<unsigned>(idx) >= 128u) return decode_gamma_far(x);  // HDRI values far outside 0..QuantumRange
  const double mant = __hiloint2double((hi & 0x800fffff) | 0x3fe00000, __double2loint(x));
  const double p = cheb9(kDecodeMono, fma(kk.four, mant, -kk.three));
  return x * (s_scale[idx] * p);
}

__device__ __forceinline__ double decode_pixel_gamma_tab(double pixel, const double *s_scale) {   // pixel.c:318
  if (pixel <= kk.toe_limit) return pixel * kk.inv_12_92;
  return kk.qr * decode_gamma_tab(fma(kk.qs, pixel, kk.c055) * kk.inv_1055, s_scale);
}

__device__ __forceinline__ void rgb_to_xyz(double R, double G, double B, double &X, double &Y, double &Z, const double *s_scale) {
  const double r = kk.qs * decode_pixel_gamma_tab(R, s_scale), g = kk.qs * decode_pixel_gamma_tab(G, s_scale),
               b = kk.qs * decode_pixel_gamma_tab(B, s_scale);
  X = fma(kk.m[0][2], b, fma(kk.m[0][1], g, kk.m[0][0] * r));
  Y = fma(kk.m[1][2], b, fma(kk.m[1][1], g, kk.m[1][0] * r));
  Z = fma(kk.m[2][2], b, fma(kk.m[2][1], g, kk.m[2][0] * r));
}

// sRGB -> Lab with the constant factors folded (the reference's chain, colorspace-private.h:1075-1107 on top of
// ConvertRGBToXYZ :1551, multiplies by QuantumScale, 1/white, 1/100, 1/255 and QuantumRange one at a time; each folded
// product differs from the chain by a relative 1e-16, nine orders of magnitude below the float ULP of the result):
// 58 instead of 82 FP64 operations per pixel.  Exact zeros survive: black decodes to 0, (0 + 16)/116 is the reference's
// own toe expression (colorspace-private.h:1075-1086 with IEEE divisions), and 116*f - 16 stays unfused -- L = 116*f(Y) - 16
// cancels there, and a black pixel must give exactly 0, not -1e-13 (a huge ULP distance for a very common value).
// The fast path is straight-line code (no divergent region per channel: the three Horner chains interleave and the
// BSSY / BSYNC / BRA scaffolding of six conditionals disappears): the toe is a select, and the two rare cases -- an
// HDRI sample whose gamma argument leaves the tabled exponents (or is +inf / NaN), a Lab argument below the CIE epsilon
// or at or above 2 (cube_root5's range) -- are collected into one flag each and handled per pixel by out-of-line code.
// (toe test in float: for a float sample p, (double)p <= 0.0404482362771076*QuantumRange  <=>  p <= 2650.775146484375f,
// the largest float below that limit; the Lab test on the high words: positive doubles order like their bit patterns,
// and anything at or below the word of the CIE epsilon -- or negative -- or with the top exponent bit set (2 and above,
// +inf, NaN) takes the exact out-of-line code.)
constexpr float kToeLimitF = 2650.775146484375f;
constexpr int kCieEpsHi = 0x3f822354;          // high word of 216/24389 = 0x3f822354d28f7cd6
constexpr int kTwoAndAboveBit = 0x40000000;    // the top exponent bit of a high word (kCubeRootSeedMax = 2)
__device__ __forceinline__ double decode_unit(float sample, const double *s_scale, bool &far) {   // QuantumScale * DecodePixelGamma
  const double pixel = static_cast<double>(sample);
  const double x = fma(pixel, kk.slope_unit, kk.offset_unit);
  const int hi = __double2hiint(x);
  const int idx = ((hi >> 20) & 0x7ff) - (1022 - 64);
  const bool toe = sample <= kToeLimitF;
  far = far || (!toe && static_cast<unsigned>(idx) >= 128u);
  const double mant = __hiloint2double((hi & 0x800fffff) | 0x3fe00000, __double2loint(x));
  const double p = cheb9(kDecodeMono, fma(kk.four, mant, -kk.three));
  const double curve = x * (s_scale[idx & 127] * p);
  return toe ? pixel * kk.toe_unit : curve;
}
__device__ __noinline__ double decode_unit_far(double pixel) {
  if (pixel <= kk.toe_limit) return pixel * kk.toe_unit;
  if (!(pixel <= 1.7976931348623157e308)) return __longlong_as_double(0x7ff8000000000000LL);   // as decode_gamma_far
  return decode_gamma(fma(pixel, kk.slope_unit, kk.offset_unit));
}
__device__ __noinline__ double lab_f_toe(double t) {
  if (t > kk.cie_eps) return cube_root(t);
  return (kCieK * t + 16.0) / 116.0;
}
__device__ __forceinline__ void rgb_to_lab_unit(float R, float G, float B, double &o0, double &o1, double &o2,
                                                const double *s_scale) {
  bool far = false;
  double r = decode_unit(R, s_scale, far), g = decode_unit(G, s_scale, far), b = decode_unit(B, s_scale, far);
  if (far) { r = decode_unit_far(R); g = decode_unit_far(G); b = decode_unit_far(B); }
  const double tx = fma(kk.mw[0][2], b, fma(kk.mw[0][1], g, kk.mw[0][0] * r));
  const double ty = fma(kk.mw[1][2], b, fma(kk.mw[1][1], g, kk.mw[1][0] * r));
  const double tz = fma(kk.mw[2][2], b, fma(kk.mw[2][1], g, kk.mw[2][0] * r));
  double x, y, z;
  // every ratio in (216/24389, 2): each high word above the epsilon's (signed: a negative ratio's word is below it), and the
  // top exponent bit -- set for 2 and above, +inf and NaN -- clear in all three
  const int hx = __double2hiint(tx), hy = __double2hiint(ty), hz = __double2hiint(tz);
  if (min(hx, min(hy, hz)) > kCieEpsHi && ((hx | hy | hz) & kTwoAndAboveBit) == 0) {
    x = cube_root5(tx); y = cube_root5(ty); z = cube_root5(tz);
  } else { x = lab_f_toe(tx); y = lab_f_toe(ty); z = lab_f_toe(tz); }
  o0 = __dsub_rn(__dmul_rn(kk.c116, y), kk.c16) * kk.l_scale;     // unfused: 116*(16/116) - 16 must be exactly 0 (black)
  o1 = fma(x - y, kk.a_scale, kk.half_qr);
  o2 = fma(y - z, kk.b_scale, kk.half_qr);
}

enum Mode { kToLab, kToXyz, kToLinear, kFromLab, kFromXyz, kFromLinear };
constexpr int kPixels = 4;

template <int CH, int MODE>
__global__ void __launch_bounds__(256) colorspace_kernel(float *buf, size_t npixels) {
  __shared__ double s_scale[128];
  if (MODE == kToLinear || MODE == kToLab || MODE == kToXyz) {
    if (threadIdx.x < 128) s_scale[threadIdx.x] = kDecodeScale[threadIdx.x];
    __syncthreads();
  }
  // kPixels pixels per thread, 256 apart (coalesced): the constant-bank loads, the table fill and the address set-up
  // are paid once per thread instead of once per pixel (the kernel is issue bound, see LabConstants)
  // The next pixel is loaded before the current one is evaluated (ncu r02: with the load at the top of the iteration
  // long_scoreboard was the largest stall, 6.8 cycles per instruction, at 69 % issue utilisation).
  size_t i = static_cast<size_t>(blockIdx.x) * (256 * kPixels) + threadIdx.x;
  if (i >= npixels) return;
  float4 nxt = make_float4(0.f, 0.f, 0.f, 0.f);
  {
    const float *q0 = buf + i * CH;
    if (CH == 4) nxt = *reinterpret_cast<const float4 *>(q0);
    else { nxt.x = q0[0]; nxt.y = q0[1]; nxt.z = q0[2]; }
  }
#pragma unroll 1
  for (int k = 0; k < kPixels; ++k, i += 256) {
  if (i >= npixels) return;
  float *q = buf + i * CH;
  const float in0 = nxt.x, in1 = nxt.y, in2 = nxt.z, in3 = nxt.w;
  if (k + 1 < kPixels && i + 256 < npixels) {
    const float *q1 = q + 256 * CH;
    if (CH == 4) nxt = *reinterpret_cast<const float4 *>(q1);
    else { nxt.x = q1[0]; nxt.y = q1[1]; nxt.z = q1[2]; }
  }
  double o0, o1, o2;
  if (MODE == kToLinear) {
    o0 = decode_pixel_gamma_tab(in0, s_scale); o1 = decode_pixel_gamma_tab(in1, s_scale); o2 = decode_pixel_gamma_tab(in2, s_scale);
  } else if (MODE == kFromLinear) {
    o0 = encode_pixel_gamma<true>(in0); o1 = encode_pixel_gamma<true>(in1); o2 = encode_pixel_gamma<true>(in2);
  } else if (MODE == kToLab) {
    rgb_to_lab_unit(in0, in1, in2, o0, o1, o2, s_scale);
  } else if (MODE == kToXyz) {
    double X, Y, Z;
    rgb_to_xyz(in0, in1, in2, X, Y, Z, s_scale);
    o0 = kk.qr * X; o1 = kk.qr * Y; o2 = kk.qr * Z;
  } else {
    double X = QS * in0, Y = QS * in1, Z = QS * in2;
    if (MODE == kFromLab) {                                  // colorspace-private.h:559-570, :531-557
      const double L = 100.0 * X, a = 255.0 * (Y - 0.5), b = 255.0 * (Z - 0.5);
      // the toe branches cancel (116*x - 16 with x = (L+16)/116): IEEE division and unfused product there, so that
      // L = 0, a = b = 0 (black) gives exactly 0 like the reference (colorspace-private.h:531-557)
      double y = (L + 16.0) / 116.0;
      double x = __dadd_rn(y, a * (1.0 / 500.0));
      double z = __dsub_rn(y, b * (1.0 / 200.0));
      if ((x * x * x) > kCieEps) x = (x * x * x); else x = __dsub_rn(__dmul_rn(116.0, x), 16.0) * (1.0 / kCieK);
      if (L > (kCieK * kCieEps)) y = (y * y * y); else y = L * (1.0 / kCieK);
      if ((z * z * z) > kCieEps) z = (z * z * z); else z = __dsub_rn(__dmul_rn(116.0, z), 16.0) * (1.0 / kCieK);
      X = kIllX * x; Y = kIllY * y; Z = kIllZ * z;
    }
    xyz_to_rgb<true>(X, Y, Z, o0, o1, o2);
  }
  if (CH == 4) *reinterpret_cast<float4 *>(q) = make_float4(static_cast<float>(o0), static_cast<float>(o1), static_cast<float>(o2), in3);
  else { q[0] = static_cast<float>(o0); q[1] = static_cast<float>(o1); q[2] = static_cast<float>(o2); }
  }
}

// kDecodeScale is per-device constant memory: filled once per device, before the first launch that reads it.
int ensure_decode_scale() {
  static std::mutex m;
  static bool done[16] = {false};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 16) return fail(MB200_ENODEVICE, "colorspace: no device");
  std::lock_guard<std::mutex> lock(m);
  if (done[dev]) return MB200_OK;
  static const double p2[5] = {1.0, 2.6390158215457883983, 6.9644045063689921093, 1.8379173679952558018e+01,
                               4.8502930128332728543e+01};            // kDecodeP2 (pixel.c:266-270)
  double host[128];
  for (int e = -64; e < 64; ++e) {
    int q = (e - 1) / 5, r = (e - 1) - q * 5;                          // C div() + the reference's fix-up (pixel.c:310-315)
    if (r < 0) { q -= 1; r += 5; }
    host[e + 64] = std::ldexp(p2[r], 7 * q);
  }
  const cudaError_t err = cudaMemcpyToSymbol(kDecodeScale, host, sizeof(host));
  if (err != cudaSuccess) return cuda_fail(err, "colorspace: table upload");
  done[dev] = true;
  return MB200_OK;
}

template <int MODE>
int launch_mode(float *buf, size_t npixels, int channels, cudaStream_t s) {
  if (MODE == kToLinear || MODE == kToLab || MODE == kToXyz) {
    const int rc = ensure_decode_scale();
    if (rc) return rc;
  }
  const unsigned blocks = static_cast<unsigned>((npixels + 256 * kPixels - 1) / (256 * kPixels));
  if (channels == 4) colorspace_kernel<4, MODE><<<blocks, 256, 0, s>>>(buf, npixels);
  else colorspace_kernel<3, MODE><<<blocks, 256, 0, s>>>(buf, npixels);
  return launch_status("colorspace launch");
}

// ---- XYZ-derived spaces of the generic branch: Adobe98, DisplayP3, ProPhoto (an RGB matrix and the sRGB transfer curve on
// either side of XYZ, colorspace-private.h:53-70, :675-737, :938-980, :1197-1211), LMS / CAT02LMS (:108-117, :655-661,
// :751-757, :1225-1231; the CAT02 legs apply both matrices, colorspace.c:135-143, :424-433), xyY (:1258-1272, :1676-1690)
// and Luv (:600-625, :1138-1161).  Smooth functions of the sample: <= 1 ULP like the Lab / XYZ legs they are built from.
struct XyzFamilyConstants {
  double to_rgb[3][3][3];     // XYZ -> Adobe98, DisplayP3, ProPhoto
  double to_xyz[3][3][3];     // ... and back
  double xyz_to_lms[3][3], lms_to_xyz[3][3];
};
__constant__ XyzFamilyConstants kx = {
    {{{2.041587903810746500, -0.56500697427885960, -0.34473135077832956},
      {-0.969243636280879500, 1.87596750150772020, 0.04155505740717557},
      {0.013444280632031142, -0.11836239223101838, 1.01517499439120540}},
     {{2.49349691194142500, -0.93138361791912390, -0.402710784450716840},
      {-0.82948896956157470, 1.76266406031834630, 0.023624685841943577},
      {0.03584583024378447, -0.07617238926804182, 0.956884524007687200}},
     {{1.3457989731028281, -0.25558010007997534, -0.05110628506753401},
      {-0.5446224939028347, 1.50823274131327810, 0.02053603239147973},
      {0.0, 0.0, 1.21196754563894540}}},
    {{{0.57666904291013050, 0.18555823790654630, 0.18822864623499470},
      {0.29734497525053605, 0.62736356625546610, 0.07529145849399788},
      {0.02703136138641234, 0.07068885253582723, 0.99133753683763880}},
     {{0.4865709486482162, 0.26566769316909306, 0.1982172852343625},
      {0.2289745640697488, 0.69173852183650640, 0.0792869140937450},
      {0.0, 0.04511338185890264, 1.0439443689009760}},
     {{0.7977604896723027, 0.13518583717574031, 0.03134934958152480000},
      {0.2880711282292934, 0.71184321781010140, 0.00008565396060525902},
      {0.0, 0.0, 0.82510460251046010000}}},
    {{0.7328, 0.4296, -0.1624}, {-0.7036, 1.6975, 0.0061}, {0.0030, 0.0136, 0.9834}},
    {{1.096123820835514, -0.278869000218287, 0.182745179382773},
     {0.454369041975359, 0.473533154307412, 0.072097803717229},
     {-0.009627608738429, -0.005698031216113, 1.015325639954543}}};

__device__ __forceinline__ void mul3(const double (&m)[3][3], double x, double y, double z, double &a, double &b, double &c) {
  a = m[0][0] * x + m[0][1] * y + m[0][2] * z;
  b = m[1][0] * x + m[1][1] * y + m[1][2] * z;
  c = m[2][0] * x + m[2][1] * y + m[2][2] * z;
}

// Jzazbz (colorspace-private.h:1274-1478; white luminance 10000 unless the image says otherwise, colorspace.c:995): a perceptual
// quantiser (two pow() per LMS component) around an LMS matrix.  NaN results (negative bases) become 0 / 0.5 / 0.5.
constexpr double kJzB = 1.15, kJzG = 0.66, kJzC1 = 3424.0 / 4096.0, kJzC2 = 2413.0 / 128.0, kJzC3 = 2392.0 / 128.0,
                 kJzN = 2610.0 / 16384.0, kJzP = 1.7 * 2523.0 / 32.0, kJzD = -0.56, kJzD0 = 1.6295499532821566e-11;
__device__ __forceinline__ void xyz_to_jzazbz(double white, double X, double Y, double Z, double &Jz, double &az, double &bz) {
  const double wlr = perceptible_reciprocal_d(white);
  const double Xp = Z + kJzB * (X - Z), Yp = X + kJzG * (Y - X);
  const double L = 0.0146480 * Z + 0.41478972 * Xp + 0.579999 * Yp;
  const double M = 0.0531008 * Z + (-0.2015100) * Xp + 1.120649 * Yp;
  const double S = 0.6684799 * Z + (-0.0166008) * Xp + 0.264800 * Yp;
  auto pq = [](double v) { const double g = pow(v, kJzN); return pow((kJzC1 + kJzC2 * g) / (1.0 + kJzC3 * g), kJzP); };
  const double Lp = pq(L * wlr), Mp = pq(M * wlr), Sp = pq(S * wlr);
  const double Iz = (Lp + Mp) * 0.5, JdI = kJzD * Iz;
  const double J = (JdI + Iz) / (JdI + 1.0) - kJzD0;
  const double a = 0.5 + 3.52400 * Lp + (-4.066708) * Mp + 0.542708 * Sp;
  const double b = 0.5 + 0.199076 * Lp + 1.096799 * Mp + (-1.295875) * Sp;
  Jz = J != J ? 0.0 : J; az = a != a ? 0.5 : a; bz = b != b ? 0.5 : b;
}
__device__ __forceinline__ void jzazbz_to_xyz(double white, double Jz, double az, double bz, double &X, double &Y, double &Z) {
  const double g = Jz + kJzD0, azz = az - 0.5, bzz = bz - 0.5;
  const double C = 0.138605043271539 * azz + 0.0580473161561189 * bzz;
  double Sp = g / (1.0 + kJzD * (1.0 - g));
  const double Lp = Sp + C, Mp = Sp - C;
  Sp += (-0.0960192420263189) * azz;
  Sp += (-0.811891896056039) * bzz;
  auto inv = [white](double v) { const double gg = pow(v, 1.0 / kJzP); return pow((gg - kJzC1) / (kJzC2 + (-2392.0 / 128.0) * gg), 1.0 / kJzN) * white; };
  const double L = inv(Lp), M = inv(Mp), S = inv(Sp);
  double Zp = (-0.0909828109828476) * L + (-0.312728290523074) * M + 1.52276656130526 * S;
  double Xp = 1.92422643578761 * L + (-1.00479231259537) * M + 0.037651404030618 * S;
  double Yp = 0.350316762094999 * L + 0.726481193931655 * M + (-0.065384422948085) * S;
  Zp = Zp != Zp ? 0.0 : Zp;
  Xp = Zp + (Xp - Zp) / kJzB;
  Xp = Xp != Xp ? 0.0 : Xp;
  Yp = Xp + (Yp - Xp) / kJzG;
  Yp = Yp != Yp ? 0.0 : Yp;
  X = Xp; Y = Yp; Z = Zp;
}

template <int CH>
__global__ void __launch_bounds__(256) xyz_family_kernel(float *buf, size_t npixels, int space, int forward, const XyzSettings st) {
  __shared__ double s_scale[128];
  if (threadIdx.x < 128) s_scale[threadIdx.x] = kDecodeScale[threadIdx.x];
  __syncthreads();
  const size_t i = static_cast<size_t>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= npixels) return;
  float *q = buf + i * CH;
  float in0, in1, in2, in3 = 0.f;
  if (CH == 4) { const float4 t = *reinterpret_cast<const float4 *>(q); in0 = t.x; in1 = t.y; in2 = t.z; in3 = t.w; }
  else { in0 = q[0]; in1 = q[1]; in2 = q[2]; }
  const int rgb = space == MB200_Adobe98Colorspace ? 0 : space == MB200_DisplayP3Colorspace ? 1 : space == MB200_ProPhotoColorspace ? 2 : -1;
  double o0, o1, o2;
  if (space == MB200_JzazbzColorspace) {          // the reference swaps green and blue on the way in and out (:1373, :1476)
    double X, Y, Z;
    if (forward) {
      double J, a, b;
      rgb_to_xyz(in0, in2, in1, X, Y, Z, s_scale);
      xyz_to_jzazbz(st.white_luminance, X, Y, Z, J, a, b);
      o0 = QR * J; o1 = QR * a; o2 = QR * b;
    } else {
      jzazbz_to_xyz(st.white_luminance, QS * static_cast<double>(in0), QS * static_cast<double>(in1), QS * static_cast<double>(in2), X, Y, Z);
      xyz_to_rgb<true>(X, Y, Z, o0, o2, o1);
    }
  } else if (space == MB200_OklabColorspace || space == MB200_OklchColorspace) {      // colorspace-private.h:1480-1549
    if (forward) {
      const double R = QS * decode_pixel_gamma_tab(in0, s_scale), G = QS * decode_pixel_gamma_tab(in1, s_scale),
                   B = QS * decode_pixel_gamma_tab(in2, s_scale);
      const double l = cbrt(0.4122214708 * R + 0.5363325363 * G + 0.0514459929 * B);
      const double m = cbrt(0.2119034982 * R + 0.6806995451 * G + 0.1073969566 * B);
      const double t = cbrt(0.0883024619 * R + 0.2817188376 * G + 0.6299787005 * B);
      const double L = 0.2104542553 * l + 0.7936177850 * m - 0.0040720468 * t;
      double a = 1.9779984951 * l - 2.4285922050 * m + 0.4505937099 * t + 0.5;
      double b = 0.0259040371 * l + 0.7827717662 * m - 0.8086757660 * t + 0.5;
      if (space == MB200_OklchColorspace) {
        const double C = sqrt(a * a + b * b), h = 0.5 + 0.5 * atan2(-b, -a) / kPiD;
        a = C; b = h;
      }
      o0 = QR * L; o1 = QR * a; o2 = QR * b;
    } else {
      const double L = QS * static_cast<double>(in0);
      double a = QS * static_cast<double>(in1), b = QS * static_cast<double>(in2);
      if (space == MB200_OklchColorspace) {
        const double C = a, h = b;
        a = C * cos(2.0 * kPiD * h); b = C * sin(2.0 * kPiD * h);
      }
      double l = L + 0.3963377774 * (a - 0.5) + 0.2158037573 * (b - 0.5);
      double m = L - 0.1055613458 * (a - 0.5) - 0.0638541728 * (b - 0.5);
      double t = L - 0.0894841775 * (a - 0.5) - 1.2914855480 * (b - 0.5);
      l *= l * l; m *= m * m; t *= t * t;
      o0 = encode_pixel_gamma<true>(QR * (4.0767416621 * l - 3.3077115913 * m + 0.2309699292 * t));
      o1 = encode_pixel_gamma<true>(QR * (-1.2684380046 * l + 2.6097574011 * m - 0.3413193965 * t));
      o2 = encode_pixel_gamma<true>(QR * (-0.0041960863 * l - 0.7034186147 * m + 1.7076147010 * t));
    }
  } else if (forward) {
    double X, Y, Z, a, b, c;
    rgb_to_xyz(in0, in1, in2, X, Y, Z, s_scale);
    if (space == MB200_LCHColorspace || space == MB200_LCHabColorspace) {       // :1104-1117
      double la, lb;
      xyz_to_lab_unit(st, X, Y, Z, a, la, lb);
      b = hypot(la - 0.5, lb - 0.5) + 0.5;
      c = 180.0 * atan2(lb - 0.5, la - 0.5) / kPiD / 360.0;
      if (c < 0.0) c += 1.0;
    } else if (space == MB200_LCHuvColorspace) {                               // :1163-1176
      double u, v;
      xyz_to_luv_unit(st, X, Y, Z, a, u, v);
      const double du = 354.0 * u - 134.0, dv = 262.0 * v - 140.0;
      b = hypot(du, dv) / 255.0 + 0.5;
      c = 180.0 * atan2(dv, du) / kPiD / 360.0;
      if (c < 0.0) c += 1.0;
    } else if (space == MB200_LabColorspace) {                                 // a reference white other than D65
      xyz_to_lab_unit(st, X, Y, Z, a, b, c);
    } else if (rgb >= 0) {
      mul3(kx.to_rgb[rgb], X, Y, Z, a, b, c);
      a = QS * encode_pixel_gamma<true>(QR * a); b = QS * encode_pixel_gamma<true>(QR * b); c = QS * encode_pixel_gamma<true>(QR * c);
    } else if (space == MB200_LMSColorspace) {
      mul3(kx.xyz_to_lms, X, Y, Z, a, b, c);
    } else if (space == MB200_CAT02LMSColorspace) {
      double L, M, S;
      mul3(kx.xyz_to_lms, X, Y, Z, L, M, S);
      mul3(kx.lms_to_xyz, L, M, S, a, b, c);
    } else if (space == MB200_xyYColorspace) {
      const double gamma = perceptible_reciprocal_d(X + Y + Z);
      a = gamma * X; b = gamma * Y; c = Y;
    } else {                                                       // Luv
      xyz_to_luv_unit(st, X, Y, Z, a, b, c);
    }
    o0 = QR * a; o1 = QR * b; o2 = QR * c;
  } else {
    const double a = QS * static_cast<double>(in0), b = QS * static_cast<double>(in1), c = QS * static_cast<double>(in2);
    double X, Y, Z;
    if (space == MB200_LCHColorspace || space == MB200_LCHabColorspace || space == MB200_LCHuvColorspace) {   // :572-653
      const double luma = 100.0 * a, chroma = 255.0 * (b - 0.5), rad = kPiD * (360.0 * c) / 180.0;
      const double p = chroma * cos(rad), q2 = chroma * sin(rad);
      if (space == MB200_LCHuvColorspace) luv_to_xyz_d(st, luma, p, q2, X, Y, Z);
      else lab_to_xyz_d(st, luma, p, q2, X, Y, Z);
    } else if (space == MB200_LabColorspace) {                                 // colorspace-private.h:559-570
      lab_to_xyz_d(st, 100.0 * a, 255.0 * (b - 0.5), 255.0 * (c - 0.5), X, Y, Z);
    } else if (rgb >= 0) {
      const double r = QS * decode_pixel_gamma_tab(QR * a, s_scale), g = QS * decode_pixel_gamma_tab(QR * b, s_scale),
                   bl = QS * decode_pixel_gamma_tab(QR * c, s_scale);
      mul3(kx.to_xyz[rgb], r, g, bl, X, Y, Z);
    } else if (space == MB200_LMSColorspace) {
      mul3(kx.lms_to_xyz, a, b, c, X, Y, Z);
    } else if (space == MB200_CAT02LMSColorspace) {
      double L, M, S;
      mul3(kx.xyz_to_lms, a, b, c, L, M, S);
      mul3(kx.lms_to_xyz, L, M, S, X, Y, Z);
    } else if (space == MB200_xyYColorspace) {
      const double gamma = perceptible_reciprocal_d(b);
      X = gamma * c * a; Y = c; Z = gamma * c * (1.0 - a - b);
    } else {                                                       // Luv
      luv_to_xyz_d(st, 100.0 * a, 354.0 * b - 134.0, 262.0 * c - 140.0, X, Y, Z);
    }
    xyz_to_rgb<true>(X, Y, Z, o0, o1, o2);
  }
  if (CH == 4) *reinterpret_cast<float4 *>(q) = make_float4(static_cast<float>(o0), static_cast<float>(o1), static_cast<float>(o2), in3);
  else { q[0] = static_cast<float>(o0); q[1] = static_cast<float>(o1); q[2] = static_cast<float>(o2); }
}

bool is_xyz_family(int cs) {
  if (cs == MB200_LCHColorspace || cs == MB200_LCHabColorspace || cs == MB200_LCHuvColorspace || cs == MB200_OklabColorspace ||
      cs == MB200_OklchColorspace || cs == MB200_JzazbzColorspace)
    return true;
  return cs == MB200_Adobe98Colorspace || cs == MB200_DisplayP3Colorspace || cs == MB200_ProPhotoColorspace ||
         cs == MB200_LMSColorspace || cs == MB200_CAT02LMSColorspace || cs == MB200_xyYColorspace || cs == MB200_LuvColorspace;
}

int launch_xyz_family_leg(float *buf, size_t npixels, int channels, int space, bool forward, const XyzSettings &st,
                          cudaStream_t s) {
  const int rc = ensure_decode_scale();
  if (rc) return rc;
  const unsigned blocks = static_cast<unsigned>((npixels + 255) / 256);
  if (channels == 4) xyz_family_kernel<4><<<blocks, 256, 0, s>>>(buf, npixels, space, forward ? 1 : 0, st);
  else xyz_family_kernel<3><<<blocks, 256, 0, s>>>(buf, npixels, space, forward ? 1 : 0, st);
  return launch_status("colorspace launch");
}

// ---- matrix colourspaces: CMY, YCbCr (= YPbPr), YDbDr, YIQ, YPbPr, YUV through the generic branch
// (colorspace.c:958-1054 / :2296-2390, colorspace-private.h:793, :141, :1551-1593, :1637-1701) and the
// LUT branch for OHTA, Rec601YCbCr, Rec709YCbCr (colorspace.c:1229-1494 / :2560-2830): samples quantised to a
// 16-bit map index (ScaleQuantumToMap), three double table entries summed left to right, ScaleMapToQuantum.
// The tables are linear in the index, so they are evaluated instead of stored: c*i (forward),
// c*i and K*(2i - MaxMap) (inverse) -- each a single rounded product like the table entry itself.
// All sums unfused in the reference's order => bit exact.
struct MatrixLeg {
  double m[3][3];     // generic: row coefficients; lut forward: c; lut inverse: column 0 = x, 1 = y (already *0.5), 2 = z
  int kind;           // 0 generic forward, 1 generic inverse, 2 lut forward, 3 lut inverse, 4 cmy forward, 5 cmy inverse
};

__device__ __forceinline__ double quantum_to_map(float q) {       // quantum-private.h:504-514 (HDRI)
  if (q >= 65535.0f) return 65535.0;
  if (q != q || q <= 0.0f) return 0.0;
  return static_cast<double>(static_cast<unsigned int>(__fadd_rn(q, 0.5f)));
}
__device__ __forceinline__ float map_to_quantum(double v) {
  if (v <= 0.0) return 0.0f;
  if (v >= 65535.0) return 65535.0f;
  return static_cast<float>(v);
}

template <int CH>
__global__ void __launch_bounds__(256) matrix_leg_kernel(float *buf, size_t npixels, const MatrixLeg a) {
  const size_t i = static_cast<size_t>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= npixels) return;
  float *q = buf + i * CH;
  float in[3], in3 = 0.f;
  if (CH == 4) { const float4 t = *reinterpret_cast<const float4 *>(q); in[0] = t.x; in[1] = t.y; in[2] = t.z; in3 = t.w; }
  else { in[0] = q[0]; in[1] = q[1]; in[2] = q[2]; }
  float o[3];
  if (a.kind == 2 || a.kind == 3) {
    const double r = quantum_to_map(in[0]), g = quantum_to_map(in[1]), b = quantum_to_map(in[2]);
    const double g2 = __dsub_rn(__dmul_rn(2.0, g), 65535.0), b2 = __dsub_rn(__dmul_rn(2.0, b), 65535.0);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      double v;
      if (a.kind == 2) {
        v = __dadd_rn(__dadd_rn(__dmul_rn(a.m[k][0], r), __dmul_rn(a.m[k][1], g)), __dmul_rn(a.m[k][2], b));
        v = __dadd_rn(v, k == 0 ? 0.0 : 32768.0);
      } else {
        v = __dadd_rn(__dadd_rn(__dmul_rn(a.m[k][0], r), __dmul_rn(a.m[k][1], g2)), __dmul_rn(a.m[k][2], b2));
      }
      o[k] = map_to_quantum(v);
    }
  } else if (a.kind == 4 || a.kind == 5) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double p = static_cast<double>(in[k]);
      o[k] = a.kind == 4 ? static_cast<float>(__dmul_rn(QR, __dmul_rn(QS, __dsub_rn(QR, p))))
                         : static_cast<float>(__dmul_rn(QR, __dsub_rn(1.0, __dmul_rn(QS, p))));
    }
  } else if (a.kind == 0) {
    const double R = in[0], G = in[1], B = in[2];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      double X = __dmul_rn(QS, __dadd_rn(__dadd_rn(__dmul_rn(a.m[k][0], R), __dmul_rn(a.m[k][1], G)), __dmul_rn(a.m[k][2], B)));
      if (k) X = __dadd_rn(X, 0.5);
      o[k] = static_cast<float>(__dmul_rn(QR, X));
    }
  } else {
    const double Y = __dmul_rn(QS, static_cast<double>(in[0]));
    const double U = __dsub_rn(__dmul_rn(QS, static_cast<double>(in[1])), 0.5);
    const double V = __dsub_rn(__dmul_rn(QS, static_cast<double>(in[2])), 0.5);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double t = __dmul_rn(a.m[k][0], Y);        // * 1.0 is exact where the reference writes plain Y
      o[k] = static_cast<float>(__dmul_rn(QR, __dadd_rn(__dadd_rn(t, __dmul_rn(a.m[k][1], U)), __dmul_rn(a.m[k][2], V))));
    }
  }
  if (CH == 4) *reinterpret_cast<float4 *>(q) = make_float4(o[0], o[1], o[2], in3);
  else { q[0] = o[0]; q[1] = o[1]; q[2] = o[2]; }
}

bool matrix_leg(int cs, bool forward, MatrixLeg &leg) {
  auto set = [&](int kind, const double (&m)[3][3]) {
    leg.kind = kind;
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) leg.m[r][c] = m[r][c];
    return true;
  };
  static const double zero[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
  // forward generic (colorspace-private.h:1551-1593)
  static const double f_ydbdr[3][3] = {{0.298839, 0.586811, 0.114350}, {-0.450, -0.883, 1.333}, {-1.333, 1.116, 0.217}};
  static const double f_yiq[3][3] = {{0.298839, 0.586811, 0.114350}, {0.595716, -0.274453, -0.321263}, {0.211456, -0.522591, 0.311135}};
  static const double f_ypbpr[3][3] = {{0.298839, 0.586811, 0.114350}, {-0.1687367, -0.331264, 0.5}, {0.5, -0.418688, -0.081312}};
  static const double f_yuv[3][3] = {{0.298839, 0.586811, 0.114350}, {-0.147, -0.289, 0.436}, {0.615, -0.515, -0.100}};
  // inverse generic (colorspace-private.h:1637-1701)
  static const double i_ydbdr[3][3] = {{1.0, 9.2303716147657e-05, -0.52591263066186533}, {1.0, -0.12913289889050927, 0.26789932820759876},
                                       {1.0, 0.66467905997895482, -7.9202543533108e-05}};
  static const double i_yiq[3][3] = {{1.0, 0.9562957197589482261, 0.6210244164652610754}, {1.0, -0.2721220993185104464, -0.6473805968256950427},
                                     {1.0, -1.1069890167364901945, 1.7046149983646481374}};
  static const double i_ypbpr[3][3] = {{0.99999999999914679361, -1.2188941887145875e-06, 1.4019995886561440468},
                                       {0.99999975910502514331, -0.34413567816504303521, -0.71413649331646789076},
                                       {1.00000124040004623180, 1.77200006607230409200, 2.1453384174593273e-06}};
  static const double i_yuv[3][3] = {{1.0, -3.945707070708279e-05, 1.1398279671717170825}, {1.0, -0.3946101641414141437, -0.5805003156565656797},
                                     {1.0, 2.0319996843434342537, -4.813762626262513e-04}};
  // LUT forward (colorspace.c:1254-1345)
  static const double l_ohta[3][3] = {{0.33333, 0.33334, 0.33333}, {0.50000, 0.00000, -0.50000}, {-0.25000, 0.50000, -0.25000}};
  static const double l_601[3][3] = {{0.298839, 0.586811, 0.114350}, {-0.1687367, -0.331264, 0.500000}, {0.500000, -0.418688, -0.081312}};
  static const double l_709[3][3] = {{0.212656, 0.715158, 0.072186}, {-0.114572, -0.385428, 0.500000}, {0.500000, -0.454153, -0.045847}};
  // LUT inverse (colorspace.c:2591-2678): rows = R, G, B; columns = x (on i_r), 0.5*y (on 2 i_g - MaxMap), 0.5*z
  static const double li_ohta[3][3] = {{1.0, 0.5 * 1.00000, -0.5 * 0.66668}, {1.0, 0.5 * 0.00000, 0.5 * 1.33333}, {1.0, -0.5 * 1.00000, -0.5 * 0.66668}};
  static const double li_601[3][3] = {{0.99999999999914679361, 0.5 * (-1.2188941887145875e-06), 0.5 * 1.4019995886561440468},
                                      {0.99999975910502514331, 0.5 * (-0.34413567816504303521), 0.5 * (-0.71413649331646789076)},
                                      {1.00000124040004623180, 0.5 * 1.77200006607230409200, 0.5 * 2.1453384174593273e-06}};
  static const double li_709[3][3] = {{1.0, 0.5 * 0.000000, 0.5 * 1.574800}, {1.0, 0.5 * (-0.187324), 0.5 * (-0.468124)},
                                      {1.0, 0.5 * 1.855600, 0.5 * 0.000000}};
  switch (cs) {
    case MB200_CMYColorspace: return set(forward ? 4 : 5, zero);
    case MB200_YDbDrColorspace: return set(forward ? 0 : 1, forward ? f_ydbdr : i_ydbdr);
    case MB200_YIQColorspace: return set(forward ? 0 : 1, forward ? f_yiq : i_yiq);
    case MB200_YCbCrColorspace: case MB200_YPbPrColorspace: return set(forward ? 0 : 1, forward ? f_ypbpr : i_ypbpr);
    case MB200_YUVColorspace: return set(forward ? 0 : 1, forward ? f_yuv : i_yuv);
    case MB200_OHTAColorspace: return set(forward ? 2 : 3, forward ? l_ohta : li_ohta);
    case MB200_Rec601YCbCrColorspace: return set(forward ? 2 : 3, forward ? l_601 : li_601);
    case MB200_Rec709YCbCrColorspace: return set(forward ? 2 : 3, forward ? l_709 : li_709);
    default: return false;
  }
}

int launch_matrix_leg(float *buf, size_t npixels, int channels, const MatrixLeg &leg, cudaStream_t s) {
  const unsigned blocks = static_cast<unsigned>((npixels + 255) / 256);
  if (channels == 4) matrix_leg_kernel<4><<<blocks, 256, 0, s>>>(buf, npixels, leg);
  else matrix_leg_kernel<3><<<blocks, 256, 0, s>>>(buf, npixels, leg);
  return launch_status("colorspace launch");
}

// ---- Log (colorspace.c:1055-1163 forward, :2391-2500 inverse): a 65536-entry Quantum table indexed by ScaleQuantumToMap
// of the linearised (forward) or the stored (inverse) sample.  The table is built on the host with the C library's
// log10 / pow exactly as the reference builds it (one table per call: 256 KB against an image of many MB), the pixel
// pass is a gather.  The forward index is taken of the decoded sample rounded to float, as ClampToQuantum does (HDRI).
// DisplayGamma = 1/1.7 is both density and gamma: the reference's "gamma" property lookup (:1081) cannot succeed,
// SetImageProperty diverts that key to image->gamma (property.c:4583).
double host_perceptible_reciprocal(double x) {
  const double sign = x < 0.0 ? -1.0 : 1.0;
  return (sign * x) >= 1.0e-12 ? 1.0 / x : sign / 1.0e-12;
}
float host_map_to_quantum(double v) { return v <= 0.0 ? 0.0f : v >= 65535.0 ? 65535.0f : static_cast<float>(v); }

void build_log_table(bool forward, const mb200_colorspace_options *o, float *logmap) {
  const double film_gamma = (o && (o->set & MB200_CO_FILM_GAMMA)) ? o->film_gamma : 0.6;
  const double reference_black = (o && (o->set & MB200_CO_REFERENCE_BLACK)) ? o->reference_black : 95.0;
  const double reference_white = (o && (o->set & MB200_CO_REFERENCE_WHITE)) ? o->reference_white : 685.0;
  const double density = 1.0 / 1.7, gamma = 1.0 / 1.7;
  const double black = std::pow(10.0, (reference_black - reference_white) * (gamma / density) * 0.002 *
                                          host_perceptible_reciprocal(film_gamma));
  long i = 0;
  if (forward) {
    for (; i <= 65535; ++i)
      logmap[i] = host_map_to_quantum((65535.0 * (reference_white + std::log10(black + (1.0 * static_cast<double>(i) / 65535.0) *
                                        (1.0 - black)) / ((gamma / density) * 0.002 * host_perceptible_reciprocal(film_gamma))) / 1024.0));
    return;
  }
  for (; i <= 65535 && i <= static_cast<long>(reference_black * 65535.0 / 1024.0); ++i) logmap[i] = 0.0f;
  for (; i <= 65535 && i < static_cast<long>(reference_white * 65535.0 / 1024.0); ++i)
    logmap[i] = static_cast<float>(QR / (1.0 - black) * (std::pow(10.0, (1024.0 * static_cast<double>(i) / 65535.0 - reference_white) *
                                   (gamma / density) * 0.002 * host_perceptible_reciprocal(film_gamma)) - black));
  for (; i <= 65535; ++i) logmap[i] = static_cast<float>(QR);
}

__device__ __forceinline__ unsigned quantum_to_index(float q) {      // quantum-private.h:504-514 (HDRI)
  if (q >= 65535.0f) return 65535u;
  if (q != q || q <= 0.0f) return 0u;
  return static_cast<unsigned>(__fadd_rn(q, 0.5f));
}

template <int CH>
__global__ void __launch_bounds__(256) log_leg_kernel(float *buf, size_t npixels, const float *__restrict__ logmap, int forward) {
  __shared__ double s_scale[128];
  if (threadIdx.x < 128) s_scale[threadIdx.x] = kDecodeScale[threadIdx.x];
  __syncthreads();
  const size_t i = static_cast<size_t>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= npixels) return;
  float *q = buf + i * CH;
  float in[3], in3 = 0.f, o[3];
  if (CH == 4) { const float4 t = *reinterpret_cast<const float4 *>(q); in[0] = t.x; in[1] = t.y; in[2] = t.z; in3 = t.w; }
  else { in[0] = q[0]; in[1] = q[1]; in[2] = q[2]; }
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    if (forward) {
      const float linear = static_cast<float>(decode_pixel_gamma_tab(static_cast<double>(in[k]), s_scale));
      o[k] = __ldg(logmap + quantum_to_index(linear));
    } else {
      o[k] = static_cast<float>(encode_pixel_gamma(static_cast<double>(__ldg(logmap + quantum_to_index(in[k])))));
    }
  }
  if (CH == 4) *reinterpret_cast<float4 *>(q) = make_float4(o[0], o[1], o[2], in3);
  else { q[0] = o[0]; q[1] = o[1]; q[2] = o[2]; }
}

// ---- YCC (PhotoYCC) in the LUT branch (colorspace.c:1347-1389 forward, :2681-2711 + :2788-2796 inverse).  Forward: the
// three tables are piecewise in the map index -- a linear toe up to (ssize_t) (0.018 * MaxMap) = 1179, then
// c * (1.099 * i - 0.099) -- and are evaluated instead of stored, with the same single roundings as the table entries;
// the C1 / C2 zeros are 156 and 137 on the 8-bit scale (x 257).  Inverse: a linear combination of the indices, scaled
// to 0..1388 and looked up in the reference's 1389-entry float table, which is the sequence "%.6f" of (float) i / 1388
// (regenerated on the host by that rule; tests/test_oracle_vs_ref.py pins the rule to the compiled reference).
// Unfused double operations in the reference's order: bit exact.
constexpr int kYccEntries = 1389;
void build_ycc_table(float *table) {
  char text[32];
  for (int i = 0; i < kYccEntries; ++i) {
    std::snprintf(text, sizeof(text), "%.6f", static_cast<double>(static_cast<float>(i) / 1388.0f));
    table[i] = std::strtof(text, nullptr);
  }
}

template <int CH>
__global__ void __launch_bounds__(256) ycc_leg_kernel(float *buf, size_t npixels, const float *__restrict__ ycc, int forward) {
  const size_t i = static_cast<size_t>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= npixels) return;
  float *q = buf + i * CH;
  float in[3], in3 = 0.f, o[3];
  if (CH == 4) { const float4 t = *reinterpret_cast<const float4 *>(q); in[0] = t.x; in[1] = t.y; in[2] = t.z; in3 = t.w; }
  else { in[0] = q[0]; in[1] = q[1]; in[2] = q[2]; }
  const double idx[3] = {quantum_to_map(in[0]), quantum_to_map(in[1]), quantum_to_map(in[2])};
  constexpr double kC1Zero = 40092.0, kC2Zero = 35209.0;
  if (forward) {
    constexpr double toe[3][3] = {{0.005382, -0.003296, 0.009410}, {0.010566, -0.006471, -0.007880}, {0.002052, 0.009768, -0.001530}};
    constexpr double curve[3][3] = {{0.298839, -0.298839, 0.70100}, {0.586811, -0.586811, -0.586811}, {0.114350, 0.88600, -0.114350}};
    double t[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) t[c] = __dsub_rn(__dmul_rn(1.099, idx[c]), 0.099);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      double e[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) e[c] = idx[c] <= 1179.0 ? __dmul_rn(toe[c][k], idx[c]) : __dmul_rn(curve[c][k], t[c]);
      const double v = __dadd_rn(__dadd_rn(__dadd_rn(e[0], e[1]), e[2]), k == 0 ? 0.0 : k == 1 ? kC1Zero : kC2Zero);
      o[k] = map_to_quantum(v);
    }
  } else {
    const double y = __dmul_rn(1.3584000, idx[0]), c1 = __dsub_rn(idx[1], kC1Zero), c2 = __dsub_rn(idx[2], kC2Zero);
    double v[3];
    v[0] = __dadd_rn(y, __dmul_rn(1.8215000, c2));
    v[1] = __dadd_rn(__dadd_rn(y, __dmul_rn(-0.4302726, c1)), __dmul_rn(-0.9271435, c2));
    v[2] = __dadd_rn(y, __dmul_rn(2.2179000, c1));
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double t = __ddiv_rn(__dmul_rn(1024.0, v[k]), 65535.0);
      const int at = t <= 0.0 ? 0 : t >= 1388.0 ? 1388 : static_cast<int>(__dadd_rn(t, 0.5));        // RoundToYCC :1814
      o[k] = static_cast<float>(__dmul_rn(QR, static_cast<double>(__ldg(ycc + at))));
    }
  }
  if (CH == 4) *reinterpret_cast<float4 *>(q) = make_float4(o[0], o[1], o[2], in3);
  else { q[0] = o[0]; q[1] = o[1]; q[2] = o[2]; }
}

int launch_log_leg(float *buf, size_t npixels, int channels, bool forward, const mb200_colorspace_options *o, cudaStream_t s) {
  int rc = ensure_decode_scale();
  if (rc) return rc;
  std::vector<float> table(65536);
  build_log_table(forward, o, table.data());
  StreamAlloc d(s);
  if ((rc = d.upload(table.data(), table.size() * sizeof(float), "colorspace: table upload"))) return rc;
  const unsigned blocks = static_cast<unsigned>((npixels + 255) / 256);
  if (channels == 4) log_leg_kernel<4><<<blocks, 256, 0, s>>>(buf, npixels, d.as<float>(), forward ? 1 : 0);
  else log_leg_kernel<3><<<blocks, 256, 0, s>>>(buf, npixels, d.as<float>(), forward ? 1 : 0);
  return launch_status("colorspace launch");
}

int launch_ycc_leg(float *buf, size_t npixels, int channels, bool forward, cudaStream_t s) {
  float table[kYccEntries];
  build_ycc_table(table);
  StreamAlloc d(s);
  const int rc = d.upload(table, sizeof(table), "colorspace: table upload");
  if (rc) return rc;
  const unsigned blocks = static_cast<unsigned>((npixels + 255) / 256);
  if (channels == 4) ycc_leg_kernel<4><<<blocks, 256, 0, s>>>(buf, npixels, d.as<float>(), forward ? 1 : 0);
  else ycc_leg_kernel<3><<<blocks, 256, 0, s>>>(buf, npixels, d.as<float>(), forward ? 1 : 0);
  return launch_status("colorspace launch");
}

}  // namespace

bool colorspace_served(int cs) {
  MatrixLeg leg{};
  return cs == MB200_sRGBColorspace || cs == MB200_RGBColorspace || cs == MB200_XYZColorspace || cs == MB200_LabColorspace ||
         cs == MB200_LogColorspace || cs == MB200_YCCColorspace || is_hexcone_colorspace(cs) || is_xyz_family(cs) ||
         matrix_leg(cs, true, leg);
}

int launch_colorspace(float *buf, size_t npixels, int channels, int from, int to, const mb200_colorspace_options *options,
                      void *stream) {
  if (channels != 3 && channels != 4) return fail(MB200_EUNSUPPORTED, "colorspace: %d channels", channels);
  if (npixels == 0) return MB200_OK;
  if (npixels > 0xffffffffull * 256) return fail(MB200_EINVAL, "colorspace: image too large");
  if (channels == 4 && !aligned16(buf)) return fail(MB200_EINVAL, "colorspace: RGBA buffers must be 16-byte aligned");
  if (options && (options->set & MB200_CO_ILLUMINANT) && (options->illuminant < 0 || options->illuminant > 10))
    return fail(MB200_EINVAL, "colorspace: illuminant %d", options->illuminant);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const XyzSettings st = xyz_settings(options);
  const bool d65 = illuminant_of(options) == kD65;
  enum Route { kNone, kCore, kLabGeneric, kHex, kXyz, kMatrix, kLog, kYcc };
  MatrixLeg from_leg{}, to_leg{};
  auto route = [&](int cs, bool forward, MatrixLeg &leg) {
    if (cs == MB200_LabColorspace) return d65 ? kCore : kLabGeneric;      // the specialised Lab kernels fold the D65 white
    if (cs == MB200_sRGBColorspace || cs == MB200_XYZColorspace || cs == MB200_RGBColorspace) return kCore;
    if (cs == MB200_LogColorspace) return kLog;
    if (cs == MB200_YCCColorspace) return kYcc;
    if (is_hexcone_colorspace(cs)) return kHex;
    if (is_xyz_family(cs)) return kXyz;
    return matrix_leg(cs, forward, leg) ? kMatrix : kNone;
  };
  const Route rf = route(from, false, from_leg), rt = route(to, true, to_leg);
  if (rf == kNone || rt == kNone) return fail(MB200_EUNSUPPORTED, "colorspace %d -> %d not implemented", from, to);
  if (from == to) return MB200_OK;
  auto leg = [&](Route r, int cs, bool forward, const MatrixLeg &m) -> int {
    switch (r) {
      case kHex: return launch_hexcone_leg(buf, npixels, channels, cs, forward, s);
      case kXyz: case kLabGeneric: return launch_xyz_family_leg(buf, npixels, channels, cs, forward, st, s);
      case kMatrix: return launch_matrix_leg(buf, npixels, channels, m, s);
      case kLog: return launch_log_leg(buf, npixels, channels, forward, options, s);
      case kYcc: return launch_ycc_leg(buf, npixels, channels, forward, s);
      default: break;
    }
    if (cs == MB200_LabColorspace) return forward ? launch_mode<kToLab>(buf, npixels, channels, s) : launch_mode<kFromLab>(buf, npixels, channels, s);
    if (cs == MB200_XYZColorspace) return forward ? launch_mode<kToXyz>(buf, npixels, channels, s) : launch_mode<kFromXyz>(buf, npixels, channels, s);
    return forward ? launch_mode<kToLinear>(buf, npixels, channels, s) : launch_mode<kFromLinear>(buf, npixels, channels, s);
  };
  int rc = MB200_OK;
  if (from != MB200_sRGBColorspace) rc = leg(rf, from, false, from_leg);          // colorspace.c:1773-1774: back to sRGB first
  if (rc == MB200_OK && to != MB200_sRGBColorspace) rc = leg(rt, to, true, to_leg);
  return rc;
}

}  // namespace mb200

// Host-side table builders, exported so that the tables can be pinned without a GPU (tests/test_host_logic.py).
extern "C" {

int mb200_log_colorspace_table(int forward, const mb200_colorspace_options *options, float *table) {
  if (!table) return mb200::fail(MB200_EINVAL, "log table: null buffer");
  mb200::build_log_table(forward != 0, options, table);
  return MB200_OK;
}

int mb200_ycc_table(float *table) {
  if (!table) return mb200::fail(MB200_EINVAL, "ycc table: null buffer");
  mb200::build_ycc_table(table);
  return MB200_OK;
}

}  // extern "C"
