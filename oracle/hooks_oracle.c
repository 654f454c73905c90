/*
  oracle/hooks_oracle.c -- TEST INFRASTRUCTURE ONLY.  Never linked into, imported by or executed from the product.

  The plain-C oracle of the last three image-returning accelerate hooks (accelerate-private.h:36-48): DespeckleImage,
  LocalContrastImage and WaveletDenoiseImage of ImageMagick 7.1.1-45 Q16-HDRI, restated in the reference's operation
  order.  Built by oracle/hooks.mk into oracle/libhooks_oracle.so, next to the main oracle (oracle.c) and with the same
  flags (no contraction, standard excess precision); pinned bit for bit against the reference compiled from source by
  tests/test_oracle_hooks_vs_ref.py.  Buffers as in oracle.h: tightly packed, channel-interleaved float32 Quantum,
  channels 1 Gray, 2 Gray+Alpha, 3 RGB, 4 RGBA.

    int orc_despeckle(const float *src, float *dst, size_t w, size_t h, int ch);
    int orc_local_contrast(const float *src, float *dst, size_t w, size_t h, int ch, double radius, double strength);
        -1 where width > w - 1: the reference reads padding it never wrote
    int orc_wavelet_denoise(const float *src, float *dst, size_t w, size_t h, int ch, double threshold, double softness);
        -1 below 32 columns or rows: HatTransform leaves the line
*/
#include <math.h>
#include <stdlib.h>
#include <string.h>

static long clampl(long v, long lo, long hi) { return v < lo ? lo : (v > hi ? hi : v); }

/* ------------------------------------------------------------------------------------------
   effect.c:1308 DespeckleImage with :1211 Hull.  Every channel (alpha included: only Copy-trait channels are skipped,
   :1412) is copied into a zero-bordered (w+2)x(h+2) plane and goes through 16 Hulls; each Hull is two data-parallel
   sweeps (f -> g, then g -> f) that compare in double against v +/- ScaleCharToQuantum(2) and step by
   ScaleCharToQuantum(1) (HDRI: 257.0*value).  The border stays 0 throughout.
   ------------------------------------------------------------------------------------------ */
static void despeckle_hull(long xo, long yo, size_t w, size_t h, int polarity, float *f, float *g)
{
  const long stride = (long) w + 2, off = yo * stride + xo;
  float *p = f + stride, *q = g + stride;
  long y;
#pragma omp parallel for schedule(static)
  for (y = 0; y < (long) h; y++) {
    long i = (2 * y + 1) + y * (long) w, x;
    for (x = 0; x < (long) w; x++, i++) {
      double v = (double) p[i];
      if (polarity > 0) { if ((double) p[i + off] >= v + 514.0) v += 257.0; }
      else if ((double) p[i + off] <= v - 514.0) v -= 257.0;
      q[i] = (float) v;
    }
  }
#pragma omp parallel for schedule(static)
  for (y = 0; y < (long) h; y++) {
    long i = (2 * y + 1) + y * (long) w, x;
    for (x = 0; x < (long) w; x++, i++) {
      double v = (double) q[i];
      if (polarity > 0) { if ((double) q[i - off] >= v + 514.0 && (double) q[i + off] > v) v += 257.0; }
      else if ((double) q[i - off] <= v - 514.0 && (double) q[i + off] < v) v -= 257.0;
      p[i] = (float) v;
    }
  }
}

int orc_despeckle(const float *src, float *dst, size_t w, size_t h, int ch)
{
  static const long X[4] = {0, 1, 1, -1}, Y[4] = {1, 0, 1, 1};
  const size_t length = (w + 2) * (h + 2);
  float *f = (float *) malloc(length * sizeof(float)), *g = (float *) malloc(length * sizeof(float));
  int c, k;
  if (!f || !g) { free(f); free(g); return -1; }
  for (c = 0; c < ch; c++) {
    size_t x, y;
    memset(f, 0, length * sizeof(float));
    memset(g, 0, length * sizeof(float));
    for (y = 0; y < h; y++)
      for (x = 0; x < w; x++) f[(y + 1) * (w + 2) + x + 1] = src[(y * w + x) * ch + c];
    for (k = 0; k < 4; k++) {
      despeckle_hull(X[k], Y[k], w, h, 1, f, g);
      despeckle_hull(-X[k], -Y[k], w, h, 1, f, g);
      despeckle_hull(-X[k], -Y[k], w, h, -1, f, g);
      despeckle_hull(X[k], Y[k], w, h, -1, f, g);
    }
    for (y = 0; y < h; y++)
      for (x = 0; x < w; x++) dst[(y * w + x) * ch + c] = f[(y + 1) * (w + 2) + x + 1];
  }
  free(f); free(g);
  return 0;
}

/* ------------------------------------------------------------------------------------------
   effect.c:2013 LocalContrastImage.  width = (ssize_t) (max(w,h) * 0.002 * |radius|); both passes apply the
   reference's asymmetric triangle of 2*width-1 taps (weights 1..width, then width+1 down to 3: the second loop starts at
   i = width+1 without advancing past the centre) to the float luma (0.212656 R + 0.715158 G + 0.072186 B, gray: the
   one sample), summing in double in tap order.  The vertical pass reads edge-clamped rows and stores sum/totalWeight
   as float into a row-padded intermediate whose padding it fills by mirroring (:2166-2170); the horizontal pass keeps
   the quotient in double and scales R, G, B by mult = (src + (src - blur) * strength/100) / src (:2246-2260; alpha
   untouched, ClampToQuantum is a bare cast in HDRI, so a black pixel gives NaN).  The mirror fills only width <=
   w - 1 columns on the left; beyond that the reference reads padding it never wrote: returns -1 then.
   ------------------------------------------------------------------------------------------ */
static double luma_of(const float *p, int ch)
{
  const double r = (double) p[0], g = ch >= 3 ? (double) p[1] : r, b = ch >= 3 ? (double) p[2] : r;
  return 0.212656 * r + 0.715158 * g + 0.072186 * b;
}

int orc_local_contrast(const float *src, float *dst, size_t w, size_t h, int ch, double radius, double strength)
{
  const long width = (long) ((double) (long) (w > h ? w : h) * 0.002 * fabs(radius));
  const long pw = (long) w + 2 * width;                       /* padded row length */
  const double total = (float) ((width + 1) * (width + 1));
  float *lum, *inter;
  long x, y;
  if (width > (long) w - 1 && width > 0) return -1;
  lum = (float *) malloc(w * h * sizeof(float));
  inter = (float *) malloc((size_t) pw * h * sizeof(float));
  if (!lum || !inter) { free(lum); free(inter); return -1; }
  for (y = 0; y < (long) (w * h); y++) lum[y] = (float) luma_of(src + (size_t) y * ch, ch);
#pragma omp parallel for schedule(static) private(y)
  for (x = 0; x < (long) w; x++) {
    float *out = inter + x + width;
    for (y = 0; y < (long) h; y++) {
      double sum = 0, weight = 1.0;
      long i, k = 0;
      for (i = 0; i < width; i++, k++) { sum += weight * (double) lum[clampl(y + k - width, 0, (long) h - 1) * (long) w + x]; weight += 1.0; }
      for (i = width + 1; i < 2 * width; i++, k++) { sum += weight * (double) lum[clampl(y + k - width, 0, (long) h - 1) * (long) w + x]; weight -= 1.0; }
      *out = (float) (sum / total);
      if (x <= width && x != 0) *(out - x * 2) = *out;
      if (x > (long) w - width - 2 && x != (long) w - 1) *(out + ((long) w - x - 1) * 2) = *out;
      out += pw;
    }
  }
#pragma omp parallel for schedule(static) private(x)
  for (y = 0; y < (long) h; y++) {
    const float *row = inter + (size_t) y * pw;
    for (x = 0; x < (long) w; x++) {
      const float *p = src + ((size_t) y * w + (size_t) x) * ch;
      float *q = dst + ((size_t) y * w + (size_t) x) * ch;
      const float *pix = row + x;
      double sum = 0, weight = 1.0, mult, srcval;
      long i;
      int c;
      for (i = 0; i < width; i++) { sum += weight * (double) *pix++; weight += 1.0; }
      for (i = width + 1; i < 2 * width; i++) { sum += weight * (double) *pix++; weight -= 1.0; }
      srcval = (float) luma_of(p, ch);
      mult = (srcval - sum / total) * (strength / 100.0);
      mult = (srcval + mult) / srcval;
      for (c = 0; c < ch; c++) q[c] = p[c];
      q[0] = (float) ((double) p[0] * mult);
      if (ch >= 3) { q[1] = (float) ((double) p[1] * mult); q[2] = (float) ((double) p[2] * mult); }
    }
  }
  free(lum); free(inter);
  return 0;
}

/* ------------------------------------------------------------------------------------------
   visual-effects.c:3515 WaveletDenoiseImage with :3478 HatTransform, on the Red / Green / Blue (gray) channels; alpha
   is untouched.  Five levels over three float planes: the row hat (step 2^level) reads the high-pass plane and writes
   the low-pass plane (plane 1 on even levels, 2 on odd ones), the column hat filters the low-pass plane in place, then
   the detail (high - low) is thresholded against +/- threshold * noise_levels[level] and added to plane 0 (at level 0
   plane 0 IS the detail plane).  Output: (double) plane 0 + (double) last low-pass plane, cast to float.  All float
   arithmetic evaluated as written.  HatTransform reads outside the line below 2 * 2^4 = 32 samples: returns -1 then.
   ------------------------------------------------------------------------------------------ */
static void hat_transform(const float *pixels, size_t stride, size_t extent, size_t scale, float *kernel)
{
  const float *p = pixels, *q = pixels + scale * stride, *r = pixels + scale * stride;
  long i;
  for (i = 0; i < (long) scale; i++) {
    kernel[i] = 0.25f * (*p + (*p) + (*q) + (*r));
    p += stride; q -= stride; r += stride;
  }
  for (; i < (long) (extent - scale); i++) {
    kernel[i] = 0.25f * (2.0f * (*p) + *(p - scale * stride) + *(p + scale * stride));
    p += stride;
  }
  q = p - scale * stride;
  r = pixels + stride * (extent - 2);
  for (; i < (long) extent; i++) {
    kernel[i] = 0.25f * (*p + (*p) + (*q) + (*r));
    p += stride; q += stride; r -= stride;
  }
}

int orc_wavelet_denoise(const float *src, float *dst, size_t w, size_t h, int ch, double threshold, double softness)
{
  static const float noise_levels[] = { 0.8002f, 0.2735f, 0.1202f, 0.0585f, 0.0291f };
  const size_t n = w * h;
  const int colours = ch >= 3 ? 3 : 1;
  float *pixels;
  int c;
  if (w < 32 || h < 32) return -1;
  pixels = (float *) malloc(3 * n * sizeof(float));
  if (!pixels) return -1;
  memcpy(dst, src, n * (size_t) ch * sizeof(float));
  for (c = 0; c < colours; c++) {
    size_t i, high_pass = 0, low_pass = 0;
    int level;
    for (i = 0; i < n; i++) pixels[i] = src[i * ch + c];
    for (level = 0; level < 5; level++) {
      const size_t scale = (size_t) 1 << level;
      double magnitude;
      long y, x;
      low_pass = n * (size_t) ((level & 1) + 1);
#pragma omp parallel for schedule(static)
      for (y = 0; y < (long) h; y++) {
        float *k = (float *) malloc(w * sizeof(float));
        hat_transform(pixels + high_pass + (size_t) y * w, 1, w, scale, k);
        memcpy(pixels + low_pass + (size_t) y * w, k, w * sizeof(float));
        free(k);
      }
#pragma omp parallel for schedule(static)
      for (x = 0; x < (long) w; x++) {
        float *k = (float *) malloc(h * sizeof(float));
        size_t r;
        hat_transform(pixels + low_pass + x, w, h, scale, k);
        for (r = 0; r < h; r++) pixels[low_pass + x + r * w] = k[r];
        free(k);
      }
      magnitude = threshold * (double) noise_levels[level];
      for (i = 0; i < n; i++) {
        pixels[high_pass + i] -= pixels[low_pass + i];
        if ((double) pixels[high_pass + i] < -magnitude)
          pixels[high_pass + i] += (float) (magnitude - softness * magnitude);
        else if ((double) pixels[high_pass + i] > magnitude)
          pixels[high_pass + i] -= (float) (magnitude - softness * magnitude);
        else
          pixels[high_pass + i] *= (float) softness;
        if (high_pass != 0) pixels[i] += pixels[high_pass + i];
      }
      high_pass = low_pass;
    }
    for (i = 0; i < n; i++) dst[i * ch + c] = (float) ((double) pixels[i] + (double) pixels[low_pass + i]);
  }
  free(pixels);
  return 0;
}
