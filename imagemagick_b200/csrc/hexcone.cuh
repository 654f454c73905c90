// hexcone.cuh -- the per-pixel legs of the hue / saturation colourspaces HCL, HCLp, HSB, HSI, HSL, HSV, HWB
// (ConvertRGBTo* / Convert*ToRGB of colorspace-private.h:149-529, :801-1064 and colorspace.c:307, :597), shared by
// TransformImageColorspace (hexcone.cu) and ModulateImage / ContrastImage (enhance.cu).
//
// to_*: raw Quantum samples -> the space's unit components; from_*: unit components -> Quantum-range doubles.  Every
// operation is the reference's own IEEE double operation, in its order, unfused (see hexcone.cu).  The from_* legs
// also accept what ModulateImage feeds them: hues shifted into (-1, 2) and the HWB "undefined" hue -1 moved off -1.
#pragma once

#include "mb200_internal.h"
#include "quantum.cuh"

#include <cuda_runtime.h>

namespace mb200 {
namespace {

constexpr double kEps = 1.0e-12;

enum Space { kHCL = MB200_HCLColorspace, kHCLp = MB200_HCLpColorspace, kHSB = MB200_HSBColorspace, kHSI = MB200_HSIColorspace,
             kHSL = MB200_HSLColorspace, kHSV = MB200_HSVColorspace, kHWB = MB200_HWBColorspace };

__device__ __forceinline__ double ad(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double sb(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double ml(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dv(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ double hi3(double a, double b, double c) { const double m = b > c ? b : c; return a > m ? a : m; }
__device__ __forceinline__ double lo3(double a, double b, double c) { const double m = b < c ? b : c; return a < m ? a : m; }
__device__ __forceinline__ bool tiny(double x) { return fabs(x) < kEps; }
__device__ __forceinline__ double reciprocal(double x) {              // PerceptibleReciprocal, pixel-accessor.h:242
  const double sign = x < 0.0 ? -1.0 : 1.0;
  return ml(sign, x) >= kEps ? dv(1.0, x) : dv(sign, kEps);
}
__device__ __forceinline__ double luma601(double r, double g, double b) {      // 0.298839 r + 0.586811 g + 0.114350 b
  return ad(ad(ml(0.298839, r), ml(0.586811, g)), ml(0.114350, b));
}

struct Triple { double x, y, z; };

// Which of the three sector values lands in R, G, B: sector s puts value kSector[s][c] (0 = dominant, 1 = secondary,
// 2 = remaining) into channel c.  The same fan-out serves HCL (c, x, 0), HSL / HSV (min+c, min+x, min) and HWB (v, n, w).
__constant__ int kSector[6][3] = {{0, 1, 2}, {1, 0, 2}, {2, 0, 1}, {2, 1, 0}, {1, 2, 0}, {0, 2, 1}};

__device__ __forceinline__ Triple fan_out(int sector, double dominant, double secondary, double remaining) {
  const double v[3] = {dominant, secondary, remaining};
  Triple t;
  t.x = v[kSector[sector][0]];
  t.y = v[kSector[sector][1]];
  t.z = v[kSector[sector][2]];
  return t;
}

// ------------------------------------------------------------------------------------------------ sRGB -> space
__device__ Triple to_hcl(double r, double g, double b) {                        // :801 (HCL) == :834 (HCLp)
  const double top = hi3(r, g, b), span = sb(top, lo3(r, g, b));
  double h = 0.0;
  if (!tiny(span)) {
    if (tiny(sb(r, top))) h = fmod(ad(dv(sb(g, b), span), 6.0), 6.0);
    else if (tiny(sb(g, top))) h = ad(dv(sb(b, r), span), 2.0);
    else if (tiny(sb(b, top))) h = ad(dv(sb(r, g), span), 4.0);
  }
  return {dv(h, 6.0), ml(QS, span), ml(QS, luma601(r, g, b))};
}

// ConvertRGBToHSB takes its extremes as max(max(red, green), blue), the other legs as max(red, max(green, blue)); the two
// differ only where a sample is NaN, so the order is kept.
__device__ Triple to_hsb(double r, double g, double b) {                        // :867
  const double top = hi3(b, r, g);
  if (tiny(top)) return {0.0, 0.0, 0.0};
  const double span = sb(top, lo3(b, r, g));
  Triple t{0.0, dv(span, top), ml(QS, top)};
  if (tiny(span)) return t;
  double h;
  if (tiny(sb(r, top))) h = dv(sb(g, b), span);
  else if (tiny(sb(g, top))) h = ad(2.0, dv(sb(b, r), span));
  else h = ad(4.0, dv(sb(r, g), span));
  h = dv(h, 6.0);
  t.x = h < 0.0 ? ad(h, 1.0) : h;
  return t;
}

__device__ Triple to_hsi(double r, double g, double b) {                        // :909
  const double rs = ml(QS, r), gs = ml(QS, g), bs = ml(QS, b);
  const double intensity = dv(ad(ad(rs, gs), bs), 3.0);
  if (intensity <= 0.0) return {0.0, 0.0, intensity};
  const double saturation = sb(1.0, dv(lo3(rs, gs, bs), intensity));
  const double alpha = ml(0.5, sb(sb(ml(ml(2.0, QS), r), gs), bs));
  const double beta = ml(0.8660254037844385, sb(gs, bs));
  double h = dv(ml(atan2(beta, alpha), 180.0 / 3.14159265358979323846264338327950288419716939937510), 360.0);
  if (h < 0.0) h = ad(h, 1.0);
  return {h, saturation, intensity};
}

template <bool VALUE>      // HSL (colorspace.c:597) / HSV (:994): same hue, different third component and saturation
__device__ Triple to_hsl_hsv(double r, double g, double b) {
  const double rs = ml(QS, r), gs = ml(QS, g), bs = ml(QS, b);
  const double top = hi3(rs, gs, bs), bottom = lo3(rs, gs, bs), span = sb(top, bottom);
  const double third = VALUE ? top : dv(ad(top, bottom), 2.0);
  if (span <= 0.0) return {0.0, 0.0, third};
  double h;
  if (tiny(sb(top, rs))) {
    h = dv(sb(gs, bs), span);
    if (gs < bs) h = ad(h, 6.0);
  } else if (tiny(sb(top, gs))) h = ad(2.0, dv(sb(bs, rs), span));
  else h = ad(4.0, dv(sb(rs, gs), span));
  h = ml(h, 60.0 / 360.0);
  double s;
  if (VALUE) s = ml(span, reciprocal(top));
  else if (third <= 0.5) s = ml(span, reciprocal(ml(2.0, third)));
  else s = ml(span, reciprocal(sb(2.0, ml(2.0, third))));
  return {h, s, third};
}

__device__ Triple to_hwb(double r, double g, double b) {                        // :1035
  const double w = lo3(r, g, b), v = hi3(r, g, b);
  Triple t{-1.0, ml(QS, w), sb(1.0, ml(QS, v))};
  if (tiny(sb(v, w))) return t;
  double f, p;
  if (tiny(sb(r, w))) { f = sb(g, b); p = 3.0; }
  else if (tiny(sb(g, w))) { f = sb(b, r); p = 5.0; }
  else { f = sb(r, g); p = 1.0; }
  t.x = dv(sb(p, dv(f, sb(v, ml(1.0, w)))), 6.0);
  return t;
}

// ------------------------------------------------------------------------------------------------ space -> sRGB
template <bool CLIP>       // HCL (:149) / HCLp (:214)
__device__ Triple from_hcl(double hue, double chroma, double luma) {
  const double h = ml(6.0, hue);
  const double x = ml(chroma, sb(1.0, fabs(sb(fmod(h, 2.0), 1.0))));
  Triple t{0.0, 0.0, 0.0};
  if (h >= 0.0 && h < 6.0) t = fan_out(static_cast<int>(h), chroma, x, 0.0);      // the six range tests of the reference
  double m = sb(luma, luma601(t.x, t.y, t.z));
  if (!CLIP) return {ml(QR, ad(t.x, m)), ml(QR, ad(t.y, m)), ml(QR, ad(t.z, m))};
  double z = 1.0;
  if (m < 0.0) {
    z = dv(luma, sb(luma, m));
    m = 0.0;
  } else if (ad(m, chroma) > 1.0) {
    z = dv(sb(1.0, luma), sb(ad(m, chroma), luma));
    m = sb(1.0, ml(z, chroma));
  }
  return {ml(QR, ad(ml(z, t.x), m)), ml(QR, ad(ml(z, t.y), m)), ml(QR, ad(ml(z, t.z), m))};
}

__device__ Triple from_hsb(double hue, double saturation, double brightness) {   // :292
  if (tiny(saturation)) { const double v = ml(QR, brightness); return {v, v, v}; }
  const double h = ml(6.0, sb(hue, floor(hue)));
  const double f = sb(h, floor(h));
  const double p = ml(brightness, sb(1.0, saturation));
  const double q = ml(brightness, sb(1.0, ml(saturation, f)));
  const double t = ml(brightness, sb(1.0, ml(saturation, sb(1.0, f))));
  int sector = static_cast<int>(h);
  if (sector < 0 || sector > 5) sector = 0;
  // dominant = brightness; even sectors rise through t, odd sectors fall through q; p is the floor
  const Triple o = fan_out(sector, brightness, (sector & 1) ? q : t, p);
  return {ml(QR, o.x), ml(QR, o.y), ml(QR, o.z)};
}

__device__ Triple from_hsi(double hue, double saturation, double intensity) {    // :368
  constexpr double kRad = 3.14159265358979323846264338327950288419716939937510 / 180.0;
  double h = ml(360.0, hue);
  h = sb(h, ml(360.0, floor(dv(h, 360.0))));
  int third = 0;
  if (!(h < 120.0)) {
    if (h < 240.0) { h = sb(h, 120.0); third = 1; }
    else { h = sb(h, 240.0); third = 2; }
  }
  const double low = ml(intensity, sb(1.0, saturation));
  const double lead = ml(intensity, ad(1.0, dv(ml(saturation, cos(ml(h, kRad))), cos(ml(sb(60.0, h), kRad)))));
  // third 0: (r, g, b) = (lead, rest, low); 1: (low, lead, rest); 2: (rest, low, lead)
  double r, g, b;
  if (third == 0) { b = low; r = lead; g = sb(sb(ml(3.0, intensity), r), b); }
  else if (third == 1) { r = low; g = lead; b = sb(sb(ml(3.0, intensity), r), g); }
  else { g = low; b = lead; r = sb(sb(ml(3.0, intensity), g), b); }
  return {ml(QR, r), ml(QR, g), ml(QR, b)};
}

template <bool VALUE>      // HSL (colorspace.c:307) / HSV (:414)
__device__ Triple from_hsl_hsv(double hue, double saturation, double third) {
  double c, floor_level;
  if (VALUE) { c = ml(third, saturation); floor_level = sb(third, c); }
  else {
    c = third <= 0.5 ? ml(ml(2.0, third), saturation) : ml(sb(2.0, ml(2.0, third)), saturation);
    floor_level = sb(third, ml(0.5, c));
  }
  double h = ml(hue, 360.0);
  h = sb(h, ml(360.0, floor(dv(h, 360.0))));
  h = dv(h, 60.0);
  const double x = ml(c, sb(1.0, fabs(sb(sb(h, ml(2.0, floor(dv(h, 2.0)))), 1.0))));
  int sector = static_cast<int>(floor(h));
  if (sector < 0 || sector > 5) sector = 0;
  const Triple o = fan_out(sector, ad(floor_level, c), ad(floor_level, x), floor_level);
  return {ml(QR, o.x), ml(QR, o.y), ml(QR, o.z)};
}

__device__ Triple from_hwb(double hue, double whiteness, double blackness) {     // :483
  const double v = sb(1.0, blackness);
  if (tiny(sb(hue, -1.0))) { const double g = ml(QR, v); return {g, g, g}; }
  const long long i = static_cast<long long>(floor(ml(6.0, hue)));                // CastDoubleToLong: NaN -> 0, saturating
  double f = sb(ml(6.0, hue), static_cast<double>(i));
  if ((i & 1) != 0) f = sb(1.0, f);
  const double n = ad(whiteness, ml(f, sb(v, whiteness)));
  const int sector = (i >= 0 && i <= 5) ? static_cast<int>(i) : 0;
  const Triple o = fan_out(sector, v, n, whiteness);
  return {ml(QR, o.x), ml(QR, o.y), ml(QR, o.z)};
}

}  // namespace
}  // namespace mb200
