// fuzzy.cuh -- IsFuzzyEquivalencePixelInfo (MagickCore/pixel.c:6028-6106) for two pixels of one image.
//
// A restatement in double, in the reference's operation order and with its early returns; compile with -fmad=false
// so no product is contracted into the sum after it.  Both pixels come from the same image, so they share the fuzz, the
// alpha trait and the colourspace.  Every comparison is `distance > fuzz`, which is false for a NaN: a NaN sample
// compares as equal, as in the reference.
#pragma once

namespace mb200 {

// The colourspace classes the comparison distinguishes: CMYK adds the black term, a hue-compatible space (HCL, HCLp,
// HSB, HSI, HSL, HSV) measures the first channel as an arc.
enum FuzzyClass { kFuzzyPlain = 0, kFuzzyHue = 1, kFuzzyCMYK = 2 };

// The PixelInfo fields the comparison reads (GetPixelInfoPixel, pixel-accessor.h:427): a gray image gives red, green
// and blue the gray sample; alpha is OpaqueAlpha without an alpha channel; black is read for CMYK only.
struct FuzzyPixel {
  double red, green, blue, black, alpha;
};

// fuzz_sq: MagickMax(fuzz, MagickSQ1_2) squared (:6037-6039), the same for every pair of one image.
__host__ __device__ inline double fuzzy_fuzz_sq(double fuzz) {
  double f = fuzz > 0.70710678118654752440084436210484903928483593768847 ? fuzz
                                                                        : 0.70710678118654752440084436210484903928483593768847;
  f *= f;
  return f;
}

__host__ __device__ inline bool fuzzy_equivalent(const FuzzyPixel &p, const FuzzyPixel &q, double fuzz_sq, bool alpha,
                                                 int cls) {
  constexpr double kQuantumRange = 65535.0;
  constexpr double kQuantumScale = 1.0 / 65535.0;
  double fuzz = fuzz_sq, scale = 1.0, distance = 0.0, pixel;
  if (alpha) {                                                          // :6042-6064
    pixel = p.alpha - q.alpha;
    distance = pixel * pixel;
    if (distance > fuzz) return false;
    scale = kQuantumScale * p.alpha;
    scale *= kQuantumScale * q.alpha;
    if (scale <= 1.0e-12) return true;                                  // MagickEpsilon
  }
  if (cls == kFuzzyCMYK) {                                              // :6068-6076
    pixel = p.black - q.black;
    distance += pixel * pixel * scale;
    if (distance > fuzz) return false;
    scale *= kQuantumScale * (kQuantumRange - p.black);
    scale *= kQuantumScale * (kQuantumRange - q.black);
  }
  distance *= 3.0;                                                      // :6080-6105
  fuzz *= 3.0;
  pixel = p.red - q.red;
  if (cls == kFuzzyHue) {
    if (fabs(pixel) > kQuantumRange / 2.0) pixel -= kQuantumRange;
    pixel *= 2.0;
  }
  distance += pixel * pixel * scale;
  if (distance > fuzz) return false;
  pixel = p.green - q.green;
  distance += pixel * pixel * scale;
  if (distance > fuzz) return false;
  pixel = p.blue - q.blue;
  distance += pixel * pixel * scale;
  if (distance > fuzz) return false;
  return true;
}

}  // namespace mb200
