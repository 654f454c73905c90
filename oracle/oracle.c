/*
  oracle/oracle.c -- TEST INFRASTRUCTURE ONLY (see oracle.h).

  CPU restatement of ImageMagick 7.1.1-45's per-pixel hot path on raw float
  buffers.  Arithmetic is kept in the reference's evaluation order (double
  accumulate, mul then add, no FMA contraction: build with -ffp-contract=off)
  so that results are bit-identical to the compiled reference; this is checked
  by tests/test_oracle_vs_ref.py and by the golden vectors in tests/golden/.
*/
#include "oracle.h"
#include <limits.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define EPS   ORC_MAGICK_EPSILON
#define QR    ORC_QUANTUM_RANGE
#define QS    ORC_QUANTUM_SCALE
/* image-private.h:44-51 */
#define PI_     3.1415926535897932384626433832795028841971693993751058209749445923078164062
#define PI2_    1.57079632679489661923132169163975144209858469968755
#define TWOPI_  6.28318530717958647692528676655900576839433879875020
#define SQ2PI_  2.50662827463100024161235523934010416269302368164062

void orc_set_threads(int n)
{
#ifdef _OPENMP
  omp_set_num_threads(n > 0 ? n : 1);
#else
  (void) n;
#endif
}

/* pixel-accessor.h:242-254 PerceptibleReciprocal */
static double precip(double x)
{
  double s = x < 0.0 ? -1.0 : 1.0;
  if (s * x >= EPS) return 1.0 / x;
  return s / EPS;
}

static long clampl(long v, long lo, long hi) { return v < lo ? lo : (v > hi ? hi : v); }

/* ------------------------------------------------------------------ kernels */

/* gem.c:262-300 GetOptimalKernelWidth1D */
size_t orc_optimal_kernel_width_1d(double radius, double sigma)
{
  double g, a, b;
  size_t width;
  if (radius > EPS) return (size_t) (2.0 * ceil(radius) + 1.0);
  g = fabs(sigma);
  if (g <= EPS) return 3;
  a = precip(2.0 * g * g);
  b = precip(SQ2PI_ * g);
  for (width = 5;; width += 2) {
    long j = (long) (width - 1) / 2, i;
    double norm = 0.0, value;
    for (i = -j; i <= j; i++) norm += exp(-((double) (i * i)) * a) * b;
    value = exp(-((double) (j * j)) * a) * b / norm;
    if (value < QS || value < EPS) break;
  }
  return width - 2;
}

/* gem.c:302-342 GetOptimalKernelWidth2D */
size_t orc_optimal_kernel_width_2d(double radius, double sigma)
{
  double g, a, b;
  size_t width;
  if (radius > EPS) return (size_t) (2.0 * ceil(radius) + 1.0);
  g = fabs(sigma);
  if (g <= EPS) return 3;
  a = precip(2.0 * g * g);
  b = precip(TWOPI_ * g * g);
  for (width = 5;; width += 2) {
    long j = (long) (width - 1) / 2, u, v;
    double norm = 0.0, value;
    for (v = -j; v <= j; v++)
      for (u = -j; u <= j; u++) norm += exp(-((double) (u * u + v * v)) * a) * b;
    value = exp(-((double) (j * j)) * a) * b / norm;
    if (value < QS || value < EPS) break;
  }
  return width - 2;
}

/* morphology.c:2485-2504 CalcKernelMetaData */
static void kernel_meta(orc_kernel *k)
{
  size_t i, n = k->width * k->height;
  k->minimum = k->maximum = 0.0;
  k->negative_range = k->positive_range = 0.0;
  for (i = 0; i < n; i++) {
    if (fabs(k->values[i]) < EPS) k->values[i] = 0.0;
    if (k->values[i] < 0) k->negative_range += k->values[i];
    else k->positive_range += k->values[i];
    if (k->values[i] < k->minimum) k->minimum = k->values[i];
    if (k->values[i] > k->maximum) k->maximum = k->values[i];
  }
}

/* morphology.c:4571-4632 ScaleKernelInfo(kernel, factor, CorrelateNormalizeValue) */
static void kernel_scale_correlate_normalize(orc_kernel *k, double factor)
{
  size_t i, n = k->width * k->height;
  double pos = fabs(k->positive_range) >= EPS ? k->positive_range : 1.0;
  double neg = fabs(k->negative_range) >= EPS ? -k->negative_range : 1.0;
  pos = factor / pos;
  neg = factor / neg;
  for (i = 0; i < n; i++)
    if (!isnan(k->values[i])) k->values[i] *= (k->values[i] >= 0) ? pos : neg;
  k->positive_range *= pos;
  k->negative_range *= neg;
  k->maximum *= (k->maximum >= 0.0) ? pos : neg;
  k->minimum *= (k->minimum >= 0.0) ? pos : neg;
}

static int kernel_alloc(orc_kernel *k, size_t w, size_t h)
{
  k->width = w; k->height = h;
  k->values = (double *) calloc((w * h) != 0 ? w * h : 1, sizeof(double));
  return k->values ? 0 : -1;
}

void orc_kernel_free(orc_kernel *k)
{
  if (k && k->values) { free(k->values); k->values = NULL; }
}

int orc_kernel_user(size_t w, size_t h, long x, long y, const double *values, orc_kernel *k)
{
  size_t i;
  memset(k, 0, sizeof(*k));
  if (kernel_alloc(k, w, h)) return -1;
  k->x = x; k->y = y; k->type = ORC_K_USER;
  /* morphology.c:318-339 ParseKernelArray range bookkeeping */
  k->minimum = 1.79769313486231570e308; k->maximum = -k->minimum;
  for (i = 0; i < w * h; i++) {
    k->values[i] = values[i];
    if (isnan(values[i])) continue;
    if (values[i] < 0) k->negative_range += values[i]; else k->positive_range += values[i];
    if (values[i] < k->minimum) k->minimum = values[i];
    if (values[i] > k->maximum) k->maximum = values[i];
  }
  return 0;
}

/* morphology.c:950-1650 AcquireKernelBuiltIn */
int orc_kernel_builtin(int type, double rho, double sigma_arg, double xi, double psi, orc_kernel *k)
{
  long u, v;
  size_t i;
  const double nan_ = sqrt(-1.0);
  memset(k, 0, sizeof(*k));
  k->type = type;
  switch (type) {
  case ORC_K_GAUSSIAN: {           /* :1045-1139 (Gaussian only) */
    double sigma = fabs(sigma_arg), A, B;
    size_t w = rho >= 1.0 ? (size_t) rho * 2 + 1 : orc_optimal_kernel_width_2d(rho, sigma);
    if (kernel_alloc(k, w, w)) return -1;
    k->x = k->y = (long) (w - 1) / 2;
    if (sigma > EPS) {
      A = 1.0 / (2.0 * sigma * sigma);
      B = (double) (1.0 / (TWOPI_ * sigma * sigma));
      for (i = 0, v = -k->y; v <= k->y; v++)
        for (u = -k->x; u <= k->x; u++, i++)
          k->values[i] = exp(-((double) (u * u + v * v)) * A) * B;
    } else
      k->values[k->x + k->y * (long) w] = 1.0;
    kernel_meta(k);
    kernel_scale_correlate_normalize(k, 1.0);
    return 0;
  }
  case ORC_K_BLUR: {               /* :1140-1227; xi = rotation angle */
    double sigma = fabs(sigma_arg), alpha, beta, angle;
    size_t w = rho >= 1.0 ? (size_t) rho * 2 + 1 : orc_optimal_kernel_width_1d(rho, sigma);
    if (kernel_alloc(k, w, 1)) return -1;
    k->x = (long) (w - 1) / 2; k->y = 0;
    v = (long) (w * 3 - 1) / 2;                 /* KernelRank 3 */
    if (sigma > EPS) {
      sigma *= 3;
      alpha = 1.0 / (2.0 * sigma * sigma);
      beta = (double) (1.0 / (SQ2PI_ * sigma));
      for (u = -v; u <= v; u++)
        k->values[(u + v) / 3] += exp(-((double) (u * u)) * alpha) * beta;
    } else
      k->values[k->x] = 1.0;
    kernel_meta(k);
    kernel_scale_correlate_normalize(k, 1.0);
    /* :4258-4364 RotateKernelInfo for a BlurKernel: only +-90 transposes */
    angle = fmod(xi, 360.0);
    if (angle < 0) angle += 360.0;
    if (337.5 < angle || angle <= 22.5) return 0;
    if (135.0 < angle && angle <= 225.0) return 0;
    if (225.0 < angle && angle <= 315.0) angle -= 180;
    if (45.0 < fmod(angle, 180.0) && fmod(angle, 180.0) <= 135.0) {
      size_t t = k->width; long tt = k->x;
      k->width = k->height; k->height = t;
      k->x = k->y; k->y = tt;
    }
    return 0;
  }
  case ORC_K_DISK: {               /* :1625-1650; sigma_arg = scale (default 1) */
    long limit = (long) (rho * rho);
    size_t w;
    if (rho < 0.4) { w = 9; limit = 18; } else w = (size_t) fabs(rho) * 2 + 1;
    if (kernel_alloc(k, w, w)) return -1;
    k->x = k->y = (long) (w - 1) / 2;
    for (i = 0, v = -k->y; v <= k->y; v++)
      for (u = -k->x; u <= k->x; u++, i++)
        if (u * u + v * v <= limit) k->positive_range += k->values[i] = sigma_arg;
        else k->values[i] = nan_;
    k->minimum = k->maximum = sigma_arg;
    return 0;
  }
  case ORC_K_DIAMOND:              /* :1537-1559 */
  case ORC_K_OCTAGON:              /* :1601-1624 */
  case ORC_K_PLUS:                 /* :1651-1672 */
  case ORC_K_CROSS: {              /* :1673-1694 */
    size_t w;
    if (rho < 1.0) w = (type == ORC_K_DIAMOND) ? 3 : 5; else w = ((size_t) rho) * 2 + 1;
    if (kernel_alloc(k, w, w)) return -1;
    k->x = k->y = (long) (w - 1) / 2;
    for (i = 0, v = -k->y; v <= k->y; v++)
      for (u = -k->x; u <= k->x; u++, i++) {
        int in;
        if (type == ORC_K_DIAMOND) in = labs(u) + labs(v) <= k->x;
        else if (type == ORC_K_OCTAGON) in = labs(u) + labs(v) <= k->x + k->x / 2;
        else if (type == ORC_K_PLUS) in = (u == 0 || v == 0);
        else in = (u == v || u == -v);
        if (in) { k->values[i] = sigma_arg; if (type == ORC_K_DIAMOND || type == ORC_K_OCTAGON) k->positive_range += sigma_arg; }
        else k->values[i] = nan_;
      }
    k->minimum = k->maximum = sigma_arg;
    if (type == ORC_K_PLUS || type == ORC_K_CROSS)
      k->positive_range = sigma_arg * (k->width * 2.0 - 1.0);
    return 0;
  }
  case ORC_K_SQUARE:               /* :1560-1599 */
  case ORC_K_RECTANGLE: {
    double scale;
    size_t w, h, n;
    if (type == ORC_K_SQUARE) {
      w = h = rho < 1.0 ? 3 : (size_t) (2 * rho + 1);
      k->x = k->y = (long) (w - 1) / 2;
      scale = sigma_arg;
    } else {
      if (rho < 1.0 || sigma_arg < 1.0) return -1;
      w = (size_t) rho; h = (size_t) sigma_arg;
      if (xi < 0.0 || xi > (double) w || psi < 0.0 || psi > (double) h) return -1;
      k->x = (long) xi; k->y = (long) psi;
      scale = 1.0;
    }
    if (kernel_alloc(k, w, h)) return -1;
    n = w * h;
    for (i = 0; i < n; i++) k->values[i] = scale;
    k->minimum = k->maximum = scale;
    k->positive_range = scale * (long) n;
    return 0;
  }
  default:
    return -1;
  }
}

/* morphology.c:4370-4398: 180 degree rotation == reversal + reflected origin */
static int kernel_reflect(const orc_kernel *in, orc_kernel *out)
{
  size_t n = in->width * in->height, i;
  *out = *in;
  out->values = (double *) malloc(n * sizeof(double));
  if (!out->values) return -1;
  /* RotateKernelInfo(...,180) is a no-op for these built-in types (:4281-4305) */
  if (in->type == ORC_K_GAUSSIAN || in->type == ORC_K_DISK || in->type == ORC_K_SQUARE ||
      in->type == ORC_K_DIAMOND || in->type == ORC_K_PLUS || in->type == ORC_K_CROSS ||
      in->type == ORC_K_BLUR) {
    memcpy(out->values, in->values, n * sizeof(double));
    return 0;
  }
  for (i = 0; i < n; i++) out->values[i] = in->values[n - 1 - i];
  out->x = (long) in->width - in->x - 1;
  out->y = (long) in->height - in->y - 1;
  return 0;
}

/* --------------------------------------------------------- MorphologyPrimitive */

static double pixel_intensity(const float *q, int ch);      /* pixel.c:2356, below (threshold operators) */

static int is_blend_channel(int ch, int i) { return (ch == 2 || ch == 4) && i != ch - 1; }
static int update_channels(int ch) { return ch; }   /* image-private.h:147 all carry Update */

/* morphology.c:2566-3227 */
long orc_morphology_primitive(const float *src, float *dst, size_t w, size_t h, int ch,
                              int method, const orc_kernel *k, double bias)
{
  const long W = (long) w, H = (long) h, kw = (long) k->width, kh = (long) k->height;
  const int alpha_i = ch - 1;
  long ox, oy, changed = 0;
  if (method == ORC_CONVOLVE || method == ORC_DILATE || method == ORC_DILATE_INTENSITY ||
      method == ORC_ITERATIVE_DISTANCE) {                   /* reflected (:2612-2626) */
    ox = kw - k->x - 1; oy = kh - k->y - 1;
  } else if (method == ORC_ERODE || method == ORC_ERODE_INTENSITY || method == ORC_HIT_AND_MISS ||
             method == ORC_THINNING || method == ORC_THICKEN) {
    ox = k->x; oy = k->y;
  } else
    return -1;

  if (method == ORC_CONVOLVE && kw == 1) {
    /* column fast path, :2654-2807 */
    long x;
#pragma omp parallel for schedule(static) reduction(+:changed)
    for (x = 0; x < W; x++) {
      long r;
      for (r = 0; r < H; r++) {
        int i;
        for (i = 0; i < ch; i++) {
          double pixel = bias, gamma = 1.0;
          size_t count = 0;
          long v;
          const double centre = (double) src[((size_t) r * w + x) * ch + i];
          if (!is_blend_channel(ch, i)) {
            for (v = 0; v < kh; v++) {
              double kv = k->values[kh - 1 - v];
              if (!isnan(kv)) {
                long yy = clampl(r - oy + v, 0, H - 1);
                pixel += kv * (double) src[((size_t) yy * w + x) * ch + i];
                count++;
              }
            }
          } else {
            gamma = 0.0;
            for (v = 0; v < kh; v++) {
              double kv = k->values[kh - 1 - v];
              if (!isnan(kv)) {
                long yy = clampl(r - oy + v, 0, H - 1);
                const float *p = src + ((size_t) yy * w + x) * ch;
                double alpha = (double) (QS * (double) p[alpha_i]);
                pixel += alpha * kv * (double) p[i];
                gamma += alpha * kv;
                count++;
              }
            }
          }
          if (fabs(pixel - centre) >= EPS) changed++;
          gamma = precip(gamma);
          if (count != 0) gamma *= (double) kh / count;
          dst[((size_t) r * w + x) * ch + i] = (float) (gamma * pixel);
        }
      }
    }
    return changed / update_channels(ch);
  }

  {
    long y;
#pragma omp parallel for schedule(static) reduction(+:changed)
    for (y = 0; y < H; y++) {
      long x;
      for (x = 0; x < W; x++) {
        int i;
        for (i = 0; i < ch; i++) {
          const double centre = (double) src[((size_t) y * w + x) * ch + i];
          double pixel, gamma = 1.0;
          long u, v;
          const float *selected = NULL;              /* quantum_pixels (:2886): the *Intensity methods copy a whole pixel */
          double minimum = QR, maximum = 0.0;        /* :2887-2888 */
          if (method == ORC_CONVOLVE) pixel = bias;
          else if (method == ORC_DILATE || method == ORC_ERODE_INTENSITY) pixel = 0.0;     /* :2902-2907 */
          else pixel = centre;
          if (method == ORC_CONVOLVE) {
            const int blend = is_blend_channel(ch, i);
            if (blend) gamma = 0.0;
            for (v = 0; v < kh; v++) {
              long yy = clampl(y - oy + v, 0, H - 1);
              for (u = 0; u < kw; u++) {
                double kv = k->values[kw * kh - 1 - (v * kw + u)];
                if (!isnan(kv)) {
                  long xx = clampl(x - ox + u, 0, W - 1);
                  const float *p = src + ((size_t) yy * w + xx) * ch;
                  if (!blend)
                    pixel += kv * (double) p[i];
                  else {
                    double alpha = (double) (QS * (double) p[alpha_i]);
                    pixel += alpha * kv * (double) p[i];
                    gamma += alpha * kv;
                  }
                }
              }
            }
          } else if (method == ORC_ERODE) {          /* :2980-3006, not reflected */
            for (v = 0; v < kh; v++) {
              long yy = clampl(y - oy + v, 0, H - 1);
              for (u = 0; u < kw; u++) {
                double kv = k->values[v * kw + u];
                if (!isnan(kv) && kv >= 0.5) {
                  long xx = clampl(x - ox + u, 0, W - 1);
                  double p = (double) src[((size_t) yy * w + xx) * ch + i];
                  if (p < pixel) pixel = p;
                }
              }
            }
          } else if (method == ORC_DILATE) {         /* :3007-3036, reflected */
            for (v = 0; v < kh; v++) {
              long yy = clampl(y - oy + v, 0, H - 1);
              for (u = 0; u < kw; u++) {
                double kv = k->values[kw * kh - 1 - (v * kw + u)];
                if (!isnan(kv) && kv > 0.5) {
                  long xx = clampl(x - ox + u, 0, W - 1);
                  double p = (double) src[((size_t) yy * w + xx) * ch + i];
                  if (p > pixel) pixel = p;
                }
              }
            }
          } else if (method == ORC_HIT_AND_MISS || method == ORC_THINNING || method == ORC_THICKEN) {
            /* :3037-3083: minimum of the foreground cells (> 0.7) minus maximum of the background cells (< 0.3), never
               negative; not reflected */
            for (v = 0; v < kh; v++) {
              long yy = clampl(y - oy + v, 0, H - 1);
              for (u = 0; u < kw; u++) {
                double kv = k->values[v * kw + u];
                if (!isnan(kv)) {
                  long xx = clampl(x - ox + u, 0, W - 1);
                  double p = (double) src[((size_t) yy * w + xx) * ch + i];
                  if (kv > 0.7) { if (p < minimum) minimum = p; }
                  else if (kv < 0.3) { if (p > maximum) maximum = p; }
                }
              }
            }
            minimum -= maximum;
            if (minimum < 0.0) minimum = 0.0;
            pixel = minimum;
            if (method == ORC_THINNING) pixel = centre - minimum;
            else if (method == ORC_THICKEN) pixel = centre + minimum;
          } else if (method == ORC_ERODE_INTENSITY) {   /* :3084-3110: the pixel of least intensity, not reflected */
            for (v = 0; v < kh; v++) {
              long yy = clampl(y - oy + v, 0, H - 1);
              for (u = 0; u < kw; u++) {
                double kv = k->values[v * kw + u];
                if (!isnan(kv) && kv >= 0.5) {
                  long xx = clampl(x - ox + u, 0, W - 1);
                  const float *p = src + ((size_t) yy * w + xx) * ch;
                  double intensity = pixel_intensity(p, ch);
                  if (intensity < minimum) { selected = p; pixel = (double) p[i]; minimum = intensity; }
                }
              }
            }
          } else if (method == ORC_DILATE_INTENSITY) {  /* :3111-3137: the pixel of greatest intensity, reflected */
            for (v = 0; v < kh; v++) {
              long yy = clampl(y - oy + v, 0, H - 1);
              for (u = 0; u < kw; u++) {
                double kv = k->values[kw * kh - 1 - (v * kw + u)];
                if (!isnan(kv) && kv >= 0.5) {
                  long xx = clampl(x - ox + u, 0, W - 1);
                  const float *p = src + ((size_t) yy * w + xx) * ch;
                  double intensity = pixel_intensity(p, ch);
                  if (intensity > maximum) { pixel = (double) p[i]; selected = p; maximum = intensity; }
                }
              }
            }
          } else {                                   /* IterativeDistance :3138-3181, reflected: min(pixel + k) */
            for (v = 0; v < kh; v++) {
              long yy = clampl(y - oy + v, 0, H - 1);
              for (u = 0; u < kw; u++) {
                double kv = k->values[kw * kh - 1 - (v * kw + u)];
                if (!isnan(kv)) {
                  long xx = clampl(x - ox + u, 0, W - 1);
                  double p = (double) src[((size_t) yy * w + xx) * ch + i];
                  if ((p + kv) < pixel) pixel = p + kv;
                }
              }
            }
          }
          if (selected != NULL) {                    /* :3186-3190: copied verbatim, not counted as a change */
            dst[((size_t) y * w + x) * ch + i] = selected[i];
            continue;
          }
          gamma = precip(gamma);
          dst[((size_t) y * w + x) * ch + i] = (float) (gamma * pixel);
          if (fabs(pixel - centre) >= EPS) changed++;
        }
      }
    }
  }
  return changed / update_channels(ch);
}

/* composite.c:1439 CompositeImage(canvas, source, DifferenceCompositeOp, clip_to_self = MagickTrue, 0, 0)
   for two images of the same size and channel layout, default artifacts (compose:sync and
   compose:clamp true, :1529-1536), every channel with its default traits -- the call MorphologyApply
   makes for the Edge / TopHat / BottomHat methods (morphology.c:3995-4012).  Per pixel (:2377-3562):
     Sa, Da = QuantumScale*alpha (1 for images without alpha)      alpha = RoundToUnity(Sa+Da-Sa*Da)
     colour : Sca = QS*Sa*Sc, Dca = QS*Da*Dc, gamma = PerceptibleReciprocal(alpha)
              pixel = QR*gamma*(Sca+Dca-2*min(Sca*Da,Dca*Sa))                        (:2922-2932)
     alpha  : pixel = QR*|Sa-Da|                                                       (:2635-2639)
     q = ClampPixel(pixel)                                                             (:2708, :3562) */
static double perceptible_reciprocal(double x)
{
  const double sign = x < 0.0 ? -1.0 : 1.0;
  if ((sign * x) >= EPS) return 1.0 / x;
  return sign / EPS;
}

static float clamp_pixel(double pixel)
{
  if (pixel < 0.0) return 0.0f;
  if (pixel >= QR) return (float) QR;
  return (float) pixel;
}

static void composite_difference(float *canvas, const float *source, size_t w, size_t h, int ch)
{
  const long n = (long) (w * h);
  const int has_alpha = (ch == 2 || ch == 4);
  long i;
#pragma omp parallel for schedule(static)
  for (i = 0; i < n; i++) {
    float *q = canvas + (size_t) i * ch;
    const float *p = source + (size_t) i * ch;
    const double Sa = QS * (has_alpha ? (double) p[ch - 1] : 65535.0);
    const double Da = QS * (has_alpha ? (double) q[ch - 1] : 65535.0);
    double alpha = Sa + Da - Sa * Da;
    int c;
    alpha = alpha < 0.0 ? 0.0 : (alpha > 1.0 ? 1.0 : alpha);
    for (c = 0; c < ch; c++) {
      double pixel;
      if (has_alpha && c == ch - 1) pixel = QR * fabs(Sa - Da);
      else {
        const double Sc = (double) p[c], Dc = (double) q[c];
        const double Sca = QS * Sa * Sc, Dca = QS * Da * Dc;
        const double gamma = perceptible_reciprocal(alpha);
        const double a = Sca * Da, b = Dca * Sa;
        pixel = QR * gamma * (Sca + Dca - 2.0 * (a < b ? a : b));
      }
      q[c] = clamp_pixel(pixel);
    }
  }
}

static int morphology_apply_basic(const float *src, float *dst, size_t w, size_t h, int ch,
                                  int method, long iterations, const orc_kernel *kernels, int nk,
                                  double bias);

/* morphology.c:3634-4077 MorphologyApply, compose == None (re-iterate).  The methods that end in
   "difference with the original" (:3813-3893 staging, :3995-4012 composite) are single-kernel only. */
int orc_morphology_apply(const float *src, float *dst, size_t w, size_t h, int ch,
                         int method, long iterations, const orc_kernel *kernels, int nk,
                         double bias)
{
  const size_t n = w * h * (size_t) ch;
  int rc;
  if (method < ORC_EDGE_IN || method > ORC_BOTTOMHAT)
    return morphology_apply_basic(src, dst, w, h, ch, method, iterations, kernels, nk, bias);
  if (nk != 1) return -1;
  if (method == ORC_EDGE) {                /* dilate, keep; erode the ORIGINAL; canvas = eroded, source = dilated */
    float *dil = (float *) malloc(n * sizeof(float));
    if (!dil) return -1;
    rc = morphology_apply_basic(src, dil, w, h, ch, ORC_DILATE, iterations, kernels, 1, bias);
    if (rc == 0) rc = morphology_apply_basic(src, dst, w, h, ch, ORC_ERODE, iterations, kernels, 1, bias);
    if (rc == 0) composite_difference(dst, dil, w, h, ch);
    free(dil);
    return rc;
  }
  rc = morphology_apply_basic(src, dst, w, h, ch,
                              method == ORC_EDGE_IN ? ORC_ERODE : method == ORC_EDGE_OUT ? ORC_DILATE :
                              method == ORC_TOPHAT ? ORC_OPEN : ORC_CLOSE, iterations, kernels, 1, bias);
  if (rc == 0) composite_difference(dst, src, w, h, ch);
  return rc;
}

/* composite.c CompositeImage(canvas, source, LightenCompositeOp, clip_to_self = MagickTrue, 0, 0) as MorphologyApply
   calls it to unite the results of a HitAndMiss kernel list (morphology.c:3722, :4044-4046); same assumptions as
   composite_difference above.  alpha = RoundToUnity(Sa+Da-Sa*Da) (:2427); alpha channel = QR*alpha (:2702-2706);
   colour (:3110-3124): (Sca*Da > Dca*Sa) ? QR*(Sca+Dca*(1-Sa)) : QR*(Dca+Sca*(1-Da));  ClampPixel. */
static void composite_lighten(float *canvas, const float *source, size_t w, size_t h, int ch)
{
  const long n = (long) (w * h);
  const int has_alpha = (ch == 2 || ch == 4);
  long i;
#pragma omp parallel for schedule(static)
  for (i = 0; i < n; i++) {
    float *q = canvas + (size_t) i * ch;
    const float *p = source + (size_t) i * ch;
    const double Sa = QS * (has_alpha ? (double) p[ch - 1] : 65535.0);
    const double Da = QS * (has_alpha ? (double) q[ch - 1] : 65535.0);
    double alpha = Sa + Da - Sa * Da;
    int c;
    alpha = alpha < 0.0 ? 0.0 : (alpha > 1.0 ? 1.0 : alpha);
    for (c = 0; c < ch; c++) {
      double pixel;
      if (has_alpha && c == ch - 1) pixel = QR * alpha;
      else {
        const double Sc = (double) p[c], Dc = (double) q[c];
        const double Sca = QS * Sa * Sc, Dca = QS * Da * Dc;
        if ((Sca * Da) > (Dca * Sa)) pixel = QR * (Sca + Dca * (1.0 - Sa));
        else pixel = QR * (Dca + Sca * (1.0 - Da));
      }
      q[c] = clamp_pixel(pixel);
    }
  }
}

static int morphology_apply_basic(const float *src, float *dst, size_t w, size_t h, int ch,
                         int method, long iterations, const orc_kernel *kernels, int nk,
                         double bias)
{
  const size_t n = w * h * (size_t) ch;
  size_t kernel_limit, method_limit = 1, method_loop = 0, method_changed = 1, stage_limit = 1;
  float *cur, *work, *tmp, *rslt = NULL;
  orc_kernel *refl = NULL;
  int kn, rc = 0, lighten = 0;
  if (iterations == 0) return -1;
  kernel_limit = iterations < 0 ? (w > h ? w : h) : (size_t) iterations;
  switch (method) {                            /* :3711-3738 */
    case ORC_SMOOTH: stage_limit = 4; break;
    case ORC_OPEN: case ORC_CLOSE: case ORC_OPEN_INTENSITY: case ORC_CLOSE_INTENSITY: stage_limit = 2; break;
    case ORC_HIT_AND_MISS: lighten = 1;        /* union of the kernel list's results */
      /* fall through */
    case ORC_THINNING: case ORC_THICKEN:
      method_limit = kernel_limit;             /* iterate the whole method, each kernel once */
      kernel_limit = 1;
      break;
    case ORC_CONVOLVE: case ORC_CORRELATE: case ORC_ERODE: case ORC_DILATE:
    case ORC_ERODE_INTENSITY: case ORC_DILATE_INTENSITY: case ORC_ITERATIVE_DISTANCE: break;
    default: return -1;
  }
  cur = (float *) malloc(n * sizeof(float));
  work = (float *) malloc(n * sizeof(float));
  if (!cur || !work) { free(cur); free(work); return -1; }
  memcpy(cur, src, n * sizeof(float));
  if (method == ORC_CORRELATE || method == ORC_CLOSE || method == ORC_SMOOTH || method == ORC_CLOSE_INTENSITY) {
    refl = (orc_kernel *) calloc((size_t) nk, sizeof(orc_kernel));
    for (kn = 0; kn < nk; kn++) kernel_reflect(&kernels[kn], &refl[kn]);
  }
  while (method_loop < method_limit && method_changed > 0 && rc == 0) {       /* Loop 1 :3787 */
  method_loop++;
  method_changed = 0;
  for (kn = 0; kn < nk && rc == 0; kn++) {
    size_t stage;
    for (stage = 1; stage <= stage_limit && rc == 0; stage++) {
      const orc_kernel *kk = &kernels[kn];
      int prim = method;
      size_t loop = 0;
      long changed = 1;
      switch (method) {                       /* :3813-3893 */
        case ORC_OPEN: prim = stage == 2 ? ORC_DILATE : ORC_ERODE; break;
        case ORC_OPEN_INTENSITY: prim = stage == 2 ? ORC_DILATE_INTENSITY : ORC_ERODE_INTENSITY; break;
        case ORC_CLOSE: kk = &refl[kn]; prim = stage == 2 ? ORC_ERODE : ORC_DILATE; break;
        case ORC_CLOSE_INTENSITY: kk = &refl[kn]; prim = stage == 2 ? ORC_ERODE_INTENSITY : ORC_DILATE_INTENSITY; break;
        case ORC_SMOOTH:
          if (stage == 1) prim = ORC_ERODE;
          else if (stage == 2) prim = ORC_DILATE;
          else if (stage == 3) { kk = &refl[kn]; prim = ORC_DILATE; }
          else { kk = &refl[kn]; prim = ORC_ERODE; }
          break;
        case ORC_CORRELATE: kk = &refl[kn]; prim = ORC_CONVOLVE; break;
        default: break;
      }
      while (loop < kernel_limit && changed > 0) {      /* :3919-3962 */
        loop++;
        changed = orc_morphology_primitive(cur, work, w, h, ch, prim, kk, bias);
        if (changed < 0) { rc = -1; break; }
        method_changed += (size_t) changed;
        tmp = cur; cur = work; work = tmp;
      }
    }
    /* multi-kernel handling (:4016-4052): a single kernel or compose == None re-iterates on the result; HitAndMiss
       keeps the first result and lightens it with every further one, each computed from the ORIGINAL image */
    if (rc == 0 && nk > 1 && lighten) {
      if (rslt == NULL) {
        rslt = (float *) malloc(n * sizeof(float));
        if (!rslt) { rc = -1; break; }
        memcpy(rslt, cur, n * sizeof(float));
      } else
        composite_lighten(rslt, cur, w, h, ch);
      memcpy(cur, src, n * sizeof(float));
    }
  }
  }
  if (rc == 0 && rslt != NULL) memcpy(cur, rslt, n * sizeof(float));
  free(rslt);
  if (rc == 0) memcpy(dst, cur, n * sizeof(float));
  if (refl) { for (kn = 0; kn < nk; kn++) orc_kernel_free(&refl[kn]); free(refl); }
  free(cur); free(work);
  return rc;
}

/* effect.c:765-796: "blur:RxS;blur:RxS+90" -> ConvolveImage */
int orc_blur(const float *src, float *dst, size_t w, size_t h, int ch, double radius, double sigma)
{
  orc_kernel k[2];
  int rc;
  if (orc_kernel_builtin(ORC_K_BLUR, radius, sigma, 0.0, 0.0, &k[0])) return -1;
  if (orc_kernel_builtin(ORC_K_BLUR, radius, sigma, 90.0, 0.0, &k[1])) { orc_kernel_free(&k[0]); return -1; }
  rc = orc_morphology_apply(src, dst, w, h, ch, ORC_CONVOLVE, 1, k, 2, 0.0);
  orc_kernel_free(&k[0]); orc_kernel_free(&k[1]);
  return rc;
}

/* effect.c:1709-1735: "gaussian:RxS" */
int orc_gaussian_blur(const float *src, float *dst, size_t w, size_t h, int ch, double radius, double sigma)
{
  orc_kernel k;
  int rc;
  if (orc_kernel_builtin(ORC_K_GAUSSIAN, radius, sigma, 0.0, 0.0, &k)) return -1;
  rc = orc_morphology_apply(src, dst, w, h, ch, ORC_CONVOLVE, 1, &k, 1, 0.0);
  orc_kernel_free(&k);
  return rc;
}

/* effect.c:4256-4391 */
int orc_unsharp(const float *src, float *dst, size_t w, size_t h, int ch,
                double radius, double sigma, double gain, double threshold)
{
  const size_t n = w * h * (size_t) ch;
  const double qt = (double) QR * threshold;
  long i;
  if (orc_blur(src, dst, w, h, ch, radius, sigma)) return -1;
#pragma omp parallel for schedule(static)
  for (i = 0; i < (long) n; i++) {
    double pixel = (double) src[i] - (double) dst[i];
    if (fabs(2.0 * pixel) < qt) pixel = (double) src[i];
    else pixel = (double) src[i] + gain * pixel;
    dst[i] = (float) pixel;
  }
  return 0;
}

/* ------------------------------------------------------------------ resize */

enum { FN_BOX, FN_TRIANGLE, FN_CUBICBC, FN_HANN, FN_HAMMING, FN_BLACKMAN, FN_GAUSSIAN,
       FN_QUADRATIC, FN_SINC, FN_SINCFAST, FN_WELCH, FN_BOHMAN, FN_LAGRANGE, FN_COSINE,
       FN_CUBICSPLINE, FN_MKS2013, FN_MKS2021, FN_JINC, FN_KAISER, FN_UNSUPPORTED };

typedef struct { int fn; double support, scale, B, C; } fn_entry;

/* resize.c:888-942 `filters[]` (function, support, window scale, B, C) */
static const fn_entry fn_table[ORC_F_SENTINEL] = {
  { FN_BOX, 0.5, 0.5, 0, 0 }, { FN_BOX, 0.0, 0.5, 0, 0 }, { FN_BOX, 0.5, 0.5, 0, 0 },
  { FN_TRIANGLE, 1.0, 1.0, 0, 0 }, { FN_CUBICBC, 1.0, 1.0, 0, 0 }, { FN_HANN, 1.0, 1.0, 0, 0 },
  { FN_HAMMING, 1.0, 1.0, 0, 0 }, { FN_BLACKMAN, 1.0, 1.0, 0, 0 }, { FN_GAUSSIAN, 2.0, 1.5, 0, 0 },
  { FN_QUADRATIC, 1.5, 1.5, 0, 0 }, { FN_CUBICBC, 2.0, 2.0, 1.0, 0.0 }, { FN_CUBICBC, 2.0, 1.0, 0.0, 0.5 },
  { FN_CUBICBC, 2.0, 8.0 / 7.0, 1. / 3., 1. / 3. }, { FN_JINC, 3.0, 1.2196698912665045, 0, 0 },
  { FN_SINC, 4.0, 1.0, 0, 0 }, { FN_SINCFAST, 4.0, 1.0, 0, 0 }, { FN_KAISER, 1.0, 1.0, 0, 0 },
  { FN_WELCH, 1.0, 1.0, 0, 0 }, { FN_CUBICBC, 2.0, 2.0, 1.0, 0.0 }, { FN_BOHMAN, 1.0, 1.0, 0, 0 },
  { FN_TRIANGLE, 1.0, 1.0, 0, 0 }, { FN_LAGRANGE, 2.0, 1.0, 0, 0 }, { FN_SINCFAST, 3.0, 1.0, 0, 0 },
  { FN_SINCFAST, 3.0, 1.0, 0, 0 }, { FN_SINCFAST, 2.0, 1.0, 0, 0 }, { FN_SINCFAST, 2.0, 1.0, 0, 0 },
  { FN_CUBICBC, 2.0, 1.1685777620836932, 0.37821575509399867, 0.31089212245300067 },
  { FN_CUBICBC, 2.0, 1.105822933719019, 0.2620145123990142, 0.3689927438004929 },
  { FN_COSINE, 1.0, 1.0, 0, 0 }, { FN_CUBICBC, 2.0, 2.0, 1.0, 0.0 }, { FN_SINCFAST, 3.0, 1.0, 0, 0 },
  { FN_CUBICSPLINE, 2.0, 0.5, 0, 0 }, { FN_MKS2013, 2.5, 1.0, 0, 0 }, { FN_MKS2021, 4.5, 1.0, 0, 0 },
};

/* resize.c:835-876 `mapping[]`: filter -> (weighting filter, window filter) */
static const int map_filter[ORC_F_SENTINEL] = {
  ORC_F_UNDEFINED, ORC_F_POINT, ORC_F_BOX, ORC_F_TRIANGLE, ORC_F_HERMITE, ORC_F_SINCFAST, ORC_F_SINCFAST,
  ORC_F_SINCFAST, ORC_F_GAUSSIAN, ORC_F_QUADRATIC, ORC_F_CUBIC, ORC_F_CATROM, ORC_F_MITCHELL, ORC_F_JINC,
  ORC_F_SINC, ORC_F_SINCFAST, ORC_F_SINCFAST, ORC_F_LANCZOS, ORC_F_SINCFAST, ORC_F_SINCFAST, ORC_F_SINCFAST,
  ORC_F_LAGRANGE, ORC_F_LANCZOS, ORC_F_LANCZOS_SHARP, ORC_F_LANCZOS2, ORC_F_LANCZOS2_SHARP, ORC_F_ROBIDOUX,
  ORC_F_ROBIDOUX_SHARP, ORC_F_LANCZOS, ORC_F_SPLINE, ORC_F_LANCZOS_RADIUS, ORC_F_CUBIC_SPLINE,
  ORC_F_MKS2013, ORC_F_MKS2021 };
static const int map_window[ORC_F_SENTINEL] = {
  ORC_F_BOX, ORC_F_BOX, ORC_F_BOX, ORC_F_BOX, ORC_F_BOX, ORC_F_HANN, ORC_F_HAMMING,
  ORC_F_BLACKMAN, ORC_F_BOX, ORC_F_BOX, ORC_F_BOX, ORC_F_BOX, ORC_F_BOX, ORC_F_BOX,
  ORC_F_BOX, ORC_F_BOX, ORC_F_KAISER, ORC_F_WELCH, ORC_F_CUBIC, ORC_F_BOHMAN, ORC_F_TRIANGLE,
  ORC_F_BOX, ORC_F_LANCZOS, ORC_F_LANCZOS_SHARP, ORC_F_LANCZOS2, ORC_F_LANCZOS2_SHARP, ORC_F_BOX,
  ORC_F_BOX, ORC_F_COSINE, ORC_F_BOX, ORC_F_LANCZOS, ORC_F_BOX, ORC_F_BOX, ORC_F_BOX };

typedef struct {
  int filter_fn, window_fn;
  double support, window_support, scale, blur, coef[7];
} rfilter;

/* resize.c:1385-1407 I0: zeroth-order modified Bessel function, power series until the term drops below MagickEpsilon */
static double bessel_i0(double x)
{
  double sum = 1.0, y = x * x / 4.0, t = y;
  long i;
  for (i = 2; t > EPS; i++) {
    sum += t;
    t *= y / ((double) i * i);
  }
  return sum;
}

/* resize.c:1410-1453 J1 (|x| < 8: rational approximation in x*x), :1456-1533 P1 / Q1 (asymptotic range, in (8/x)^2) */
static double ratio_xx(const double *pc, const double *qc, int n, double x)
{
  double p = pc[n - 1], q = qc[n - 1];
  int i;
  for (i = n - 2; i >= 0; i--) {
    p = p * x * x + pc[i];
    q = q * x * x + qc[i];
  }
  return p / q;
}
static double ratio_8x(const double *pc, const double *qc, int n, double x)
{
  double p = pc[n - 1], q = qc[n - 1];
  int i;
  for (i = n - 2; i >= 0; i--) {
    p = p * (8.0 / x) * (8.0 / x) + pc[i];
    q = q * (8.0 / x) * (8.0 / x) + qc[i];
  }
  return p / q;
}
/* resize.c:1535-1553 BesselOrderOne */
static double bessel_order_one(double x)
{
  static const double j1p[9] = {
    0.581199354001606143928050809e+21, -0.6672106568924916298020941484e+20, 0.2316433580634002297931815435e+19,
    -0.3588817569910106050743641413e+17, 0.2908795263834775409737601689e+15, -0.1322983480332126453125473247e+13,
    0.3413234182301700539091292655e+10, -0.4695753530642995859767162166e+7, 0.270112271089232341485679099e+4 };
  static const double j1q[9] = {
    0.11623987080032122878585294e+22, 0.1185770712190320999837113348e+20, 0.6092061398917521746105196863e+17,
    0.2081661221307607351240184229e+15, 0.5243710262167649715406728642e+12, 0.1013863514358673989967045588e+10,
    0.1501793594998585505921097578e+7, 0.1606931573481487801970916749e+4, 0.1e+1 };
  static const double p1p[6] = {
    0.352246649133679798341724373e+5, 0.62758845247161281269005675e+5, 0.313539631109159574238669888e+5,
    0.49854832060594338434500455e+4, 0.2111529182853962382105718e+3, 0.12571716929145341558495e+1 };
  static const double p1q[6] = {
    0.352246649133679798068390431e+5, 0.626943469593560511888833731e+5, 0.312404063819041039923015703e+5,
    0.4930396490181088979386097e+4, 0.2030775189134759322293574e+3, 0.1e+1 };
  static const double q1p[6] = {
    0.3511751914303552822533318e+3, 0.7210391804904475039280863e+3, 0.4259873011654442389886993e+3,
    0.831898957673850827325226e+2, 0.45681716295512267064405e+1, 0.3532840052740123642735e-1 };
  static const double q1q[6] = {
    0.74917374171809127714519505e+4, 0.154141773392650970499848051e+5, 0.91522317015169922705904727e+4,
    0.18111867005523513506724158e+4, 0.1038187585462133728776636e+3, 0.1e+1 };
  double p, q;
  if (x == 0.0) return 0.0;
  p = x;
  if (x < 0.0) x = -x;
  if (x < 8.0) return p * ratio_xx(j1p, j1q, 9, x);
  q = sqrt((double) (2.0 / (PI_ * x))) * (ratio_8x(p1p, p1q, 6, x) * (1.0 / sqrt(2.0) * (sin(x) - cos(x))) -
      8.0 / x * ratio_8x(q1p, q1q, 6, x) * (-1.0 / sqrt(2.0) * (sin(x) + cos(x))));
  if (p < 0.0) q = -q;
  return q;
}

/* resize.c:803-1226 AcquireResizeFilter with no "filter:*" artifacts, not cylindrical */
static int rfilter_init_ex(rfilter *rf, int filter, const orc_filter_options *opt)
{
  int ft, wt;
  const unsigned set = opt ? opt->set : 0u;
  double B = 0.0, C = 0.0;
  if (filter <= ORC_F_UNDEFINED || filter >= ORC_F_SENTINEL) return -1;
  ft = map_filter[filter]; wt = map_window[filter];
  if ((set & ORC_FO_WINDOW) && opt->window > ORC_F_UNDEFINED && opt->window < ORC_F_SENTINEL) {   /* :999-1043 */
    if (!opt->keep_filter) ft = ORC_F_SINCFAST;
    wt = opt->window;
  }
  memset(rf, 0, sizeof(*rf));
  rf->blur = 1.0;
  rf->filter_fn = fn_table[ft].fn;
  rf->support = fn_table[ft].support;
  rf->window_fn = fn_table[wt].fn;
  rf->scale = fn_table[wt].scale;
  if (rf->filter_fn == FN_UNSUPPORTED || rf->window_fn == FN_UNSUPPORTED) return -1;
  if (ft == ORC_F_LANCZOS_SHARP) rf->blur *= 0.9812505644269356;       /* :1064-1076 */
  if (ft == ORC_F_LANCZOS2_SHARP) rf->blur *= 0.9549963639785485;
  if (rf->filter_fn == FN_GAUSSIAN || rf->window_fn == FN_GAUSSIAN) {   /* :1083-1097 */
    double value = 0.5;
    if (set & ORC_FO_SIGMA) value = opt->sigma;
    rf->coef[0] = value;
    rf->coef[1] = precip(2.0 * value * value);
    rf->coef[2] = precip(TWOPI_ * value * value);
    if (value > 0.5) rf->support *= 2 * value;                         /* :1097-1098 */
  }
  if (rf->filter_fn == FN_KAISER || rf->window_fn == FN_KAISER) {       /* :1104-1120 */
    double value = 6.5;
    if (set & ORC_FO_KAISER_BETA) value = opt->kaiser_beta;
    rf->coef[0] = value;
    rf->coef[1] = precip(bessel_i0(value));
  }
  if (set & ORC_FO_LOBES) {                                             /* :1123-1133 */
    long lobes = opt->lobes;
    if (lobes < 1) lobes = 1;
    rf->support = (double) lobes;
  }
  if (rf->filter_fn == FN_JINC) {                                       /* :1135-1150: lobes -> first zeros of the Jinc */
    static const double jinc_zeros[16] = {
      1.2196698912665045, 2.2331305943815286, 3.2383154841662362, 4.2410628637960699, 5.2427643768701817,
      6.2439216898644877, 7.2447598687199570, 8.2453949139520427, 9.2458926849494673, 10.246293348754916,
      11.246622794877883, 12.246898461138105, 13.247132522181061, 14.247333735806849, 15.247508563037300,
      16.247661874700962 };
    if (rf->support > 16) rf->support = jinc_zeros[15];
    else rf->support = jinc_zeros[((long) rf->support) - 1];
  }
  if (set & ORC_FO_BLUR) rf->blur *= opt->blur;                         /* :1155-1157 */
  if (rf->blur < EPS) rf->blur = EPS;
  if (set & ORC_FO_SUPPORT) rf->support = fabs(opt->support);           /* :1163-1165 */
  rf->window_support = rf->support;
  if (set & ORC_FO_WIN_SUPPORT) rf->window_support = fabs(opt->win_support);   /* :1170-1173 */
  rf->scale *= precip(rf->window_support);                              /* :1177 */
  if (rf->filter_fn == FN_CUBICBC || rf->window_fn == FN_CUBICBC) {     /* :1181-1226 */
    B = fn_table[ft].B; C = fn_table[ft].C;
    if (fn_table[wt].fn == FN_CUBICBC) { B = fn_table[wt].B; C = fn_table[wt].C; }
    if (set & ORC_FO_B) {                                               /* :1196-1212 */
      B = opt->b;
      C = (1.0 - B) / 2.0;
      if (set & ORC_FO_C) C = opt->c;
    } else if (set & ORC_FO_C) {
      C = opt->c;
      B = 1.0 - 2.0 * C;
    }
    {
      const double twoB = B + B;
      rf->coef[0] = 1.0 - (1.0 / 3.0) * B;
      rf->coef[1] = -3.0 + twoB + C;
      rf->coef[2] = 2.0 - 1.5 * B - C;
      rf->coef[3] = (4.0 / 3.0) * B + 4.0 * C;
      rf->coef[4] = -8.0 * C - twoB;
      rf->coef[5] = B + 5.0 * C;
      rf->coef[6] = (-1.0 / 6.0) * B - C;
    }
  }
  return 0;
}

static int rfilter_init(rfilter *rf, int filter) { return rfilter_init_ex(rf, filter, NULL); }

/* resize.c:493-587 SincFast, Q16 branch (:547-563) */
static double sinc_fast(double x)
{
  static const double c[10] = {
    0.173611107357320220183368594093166520811e-2L, -0.384240921114946632192116762889211361285e-3L,
    0.394201182359318128221229891724947048771e-4L, -0.250963301609117217660068889165550534856e-5L,
    0.111902032818095784414237782071368805120e-6L, -0.372895101408779549368465614321137048875e-8L,
    0.957694196677572570319816780188718518330e-10L, -0.187208577776590710853865174371617338991e-11L,
    0.253524321426864752676094495396308636823e-13L, -0.177084805010701112639035485248501049364e-15L };
  if (x > 4.0) {
    const double alpha = (double) (PI_ * x);
    return sin((double) alpha) / alpha;
  }
  {
    const double xx = x * x;
    const double p = c[0] + xx * (c[1] + xx * (c[2] + xx * (c[3] + xx * (c[4] + xx * (c[5] + xx *
                     (c[6] + xx * (c[7] + xx * (c[8] + xx * c[9]))))))));
    return (xx - 1.0) * (xx - 4.0) * (xx - 9.0) * (xx - 16.0) * p;
  }
}

static double eval_fn(int fn, double x, const rfilter *rf)
{
  switch (fn) {
  case FN_BOX: return 1.0;                                              /* :166-178 */
  case FN_TRIANGLE: return x < 1.0 ? 1.0 - x : 0.0;                     /* :589-602 */
  case FN_CUBICBC:                                                      /* :209-247 */
    if (x < 1.0) return rf->coef[0] + x * (x * (rf->coef[1] + x * rf->coef[2]));
    if (x < 2.0) return rf->coef[3] + x * (rf->coef[4] + x * (rf->coef[5] + x * rf->coef[6]));
    return 0.0;
  case FN_HANN: { const double c = cos((double) (PI_ * x)); return 0.5 + 0.5 * c; }      /* :322-333 */
  case FN_HAMMING: { const double c = cos((double) (PI_ * x)); return 0.54 + 0.46 * c; } /* :335-346 */
  case FN_BLACKMAN: { const double c = cos((double) (PI_ * x)); return 0.34 + c * (0.5 + c * 0.16); } /* :132-145 */
  case FN_GAUSSIAN: return exp((double) (-rf->coef[1] * x * x));        /* :288-320 */
  case FN_QUADRATIC:                                                    /* :460-474 */
    if (x < 0.5) return 0.75 - x * x;
    if (x < 1.5) return 0.5 * (x - 1.5) * (x - 1.5);
    return 0.0;
  case FN_SINC:                                                         /* :476-491 */
    if (x != 0.0) { const double a = (double) (PI_ * x); return sin((double) a) / a; }
    return 1.0;
  case FN_SINCFAST: return sinc_fast(x);
  case FN_WELCH: return x < 1.0 ? 1.0 - x * x : 0.0;                    /* :604-615 */
  case FN_BOHMAN: {                                                     /* :147-164 */
    const double c = cos((double) (PI_ * x));
    const double s = sqrt(1.0 - c * c);
    return (1.0 - x) * c + (1.0 / PI_) * s;
  }
  case FN_COSINE: return cos((double) (PI2_ * x));                      /* :180-190 */
  case FN_LAGRANGE: {                                                   /* :388-420 */
    double value;
    long i, n, order;
    if (x > rf->support) return 0.0;
    order = (long) (2.0 * rf->window_support);
    n = (long) (rf->window_support + x);
    value = 1.0f;
    for (i = 0; i < order; i++)
      if (i != n) value *= (n - i - x) / (n - i);
    return value;
  }
  case FN_CUBICSPLINE:                                                  /* :249-286, 2 lobes */
    if (x < 1.0) return ((x - 9.0 / 5.0) * x - 1.0 / 5.0) * x + 1.0;
    if (x < 2.0) return ((-1.0 / 3.0 * (x - 1.0) + 4.0 / 5.0) * (x - 1.0) - 7.0 / 15.0) * (x - 1.0);
    return 0.0;
  case FN_JINC:                                                         /* :348-364 */
    if (x == 0.0) return 0.5 * PI_;
    return bessel_order_one(PI_ * x) / x;
  case FN_KAISER:                                                       /* :366-382 */
    return rf->coef[1] * bessel_i0(rf->coef[0] * sqrt((double) (1.0 - x * x)));
  case FN_MKS2013:                                                      /* :422-438 */
    if (x < 0.5) return 0.625 + 1.75 * (0.5 - x) * (0.5 + x);
    if (x < 1.5) return (1.0 - x) * (1.75 - x);
    if (x < 2.5) return -0.125 * (2.5 - x) * (2.5 - x);
    return 0.0;
  case FN_MKS2021:                                                      /* :440-458 */
    if (x < 0.5) return 577.0 / 576.0 - 239.0 / 144.0 * x * x;
    if (x < 1.5) return 35.0 / 36.0 * (x - 1.0) * (x - 239.0 / 140.0);
    if (x < 2.5) return 1.0 / 6.0 * (x - 2.0) * (65.0 / 24.0 - x);
    if (x < 3.5) return 1.0 / 36.0 * (x - 3.0) * (x - 3.75);
    if (x < 4.5) return -1.0 / 288.0 * (x - 4.5) * (x - 4.5);
    return 0.0;
  default: return 0.0;
  }
}

/* resize.c:1690-1714 GetResizeFilterWeight */
static double rfilter_weight(const rfilter *rf, double x)
{
  double scale, xb = fabs((double) x) * precip(rf->blur);
  if (rf->window_support < EPS || rf->window_fn == FN_BOX) scale = 1.0;
  else scale = eval_fn(rf->window_fn, xb * rf->scale, rf);
  return scale * eval_fn(rf->filter_fn, xb, rf);
}

double orc_filter_weight(int f, double x)
{
  rfilter rf;
  if (rfilter_init(&rf, f)) return NAN;
  return rfilter_weight(&rf, x);
}

double orc_filter_weight_ex(int f, const orc_filter_options *options, double x)
{
  rfilter rf;
  if (rfilter_init_ex(&rf, f, options)) return NAN;
  return rfilter_weight(&rf, x);
}

double orc_filter_support_ex(int f, const orc_filter_options *options)
{
  rfilter rf;
  if (rfilter_init_ex(&rf, f, options)) return NAN;
  return rf.support * rf.blur;
}

double orc_filter_support(int f)
{
  rfilter rf;
  if (rfilter_init(&rf, f)) return NAN;
  return rf.support * rf.blur;                       /* :1656-1661 */
}

/* One axis of resize.c:3333-3547 (HorizontalFilter) / :3549-3759 (VerticalFilter).
   axis 0: filter along x (src w -> dst ow, rows unchanged); axis 1: along y. */
static int resize_axis(const rfilter *rf, const float *src, size_t w, size_t h, int ch,
                       float *dst, size_t on, double factor, int axis)
{
  const long in_n = axis == 0 ? (long) w : (long) h;
  const size_t ow = axis == 0 ? on : w, oh = axis == 0 ? h : on;
  const long lines = axis == 0 ? (long) h : (long) w;
  const int alpha_i = ch - 1;
  double scale = fmax(1.0 / factor + EPS, 1.0);
  double support = scale * (rf->support * rf->blur);
  long o;
  if (support < 0.5) { support = 0.5; scale = 1.0; }
  scale = precip(scale);
#pragma omp parallel for schedule(static)
  for (o = 0; o < (long) on; o++) {
    double bisect = (double) (o + 0.5) / factor + EPS;
    long start = (long) fmax(bisect - support + 0.5, 0.0);
    long stop = (long) fmin(bisect + support + 0.5, (double) in_n);
    long n = stop - start, j, l;
    double density = 0.0;
    double *wt;
    if (n <= 0) continue;
    wt = (double *) malloc((size_t) n * sizeof(double));
    for (j = 0; j < n; j++) {
      wt[j] = rfilter_weight(rf, scale * ((double) (start + j) - bisect + 0.5));
      density += wt[j];
    }
    if (density != 0.0 && density != 1.0) {
      density = precip(density);
      for (j = 0; j < n; j++) wt[j] *= density;
    }
    for (l = 0; l < lines; l++) {
      int i;
      for (i = 0; i < ch; i++) {
        double pixel = 0.0;
#define SRC(jj) (axis == 0 ? src + ((size_t) l * w + (size_t) (start + (jj))) * ch \
                           : src + ((size_t) (start + (jj)) * w + (size_t) l) * ch)
        float *q = axis == 0 ? dst + ((size_t) l * ow + (size_t) o) * ch
                             : dst + ((size_t) o * ow + (size_t) l) * ch;
        (void) oh;
        if (!is_blend_channel(ch, i)) {
          for (j = 0; j < n; j++) {
            double alpha = wt[j];
            pixel += alpha * (double) SRC(j)[i];
          }
          q[i] = (float) pixel;
        } else {
          double gamma = 0.0;
          for (j = 0; j < n; j++) {
            const float *p = SRC(j);
            double alpha = wt[j] * QS * (double) p[alpha_i];
            pixel += alpha * (double) p[i];
            gamma += alpha;
          }
          gamma = precip(gamma);
          q[i] = (float) (gamma * pixel);
        }
#undef SRC
      }
    }
    free(wt);
  }
  return 0;
}

/* resize.c:3761-3874 ResizeImage */
int orc_resize(const float *src, size_t w, size_t h, int ch,
               float *dst, size_t ow, size_t oh, int filter)
{
  return orc_resize_ex(src, w, h, ch, dst, ow, oh, filter, NULL);
}

int orc_resize_ex(const float *src, size_t w, size_t h, int ch, float *dst, size_t ow, size_t oh, int filter,
                  const orc_filter_options *options)
{
  rfilter rf;
  double xf, yf;
  float *tmp;
  int ft = ORC_F_LANCZOS;
  if (ow == 0 || oh == 0) return -1;
  if (ow == w && oh == h && filter == ORC_F_UNDEFINED) {
    memcpy(dst, src, w * h * (size_t) ch * sizeof(float));
    return 0;
  }
  xf = (double) (ow * precip((double) w));
  yf = (double) (oh * precip((double) h));
  if (filter != ORC_F_UNDEFINED) ft = filter;
  else if (xf == 1.0 && yf == 1.0) ft = ORC_F_POINT;
  else if ((ch == 2 || ch == 4) || (xf * yf) > 1.0) ft = ORC_F_MITCHELL;
  if (rfilter_init_ex(&rf, ft, options)) return -1;
  if (xf > yf) {
    tmp = (float *) malloc(ow * h * (size_t) ch * sizeof(float));
    if (!tmp) return -1;
    resize_axis(&rf, src, w, h, ch, tmp, ow, xf, 0);
    resize_axis(&rf, tmp, ow, h, ch, dst, oh, yf, 1);
  } else {
    tmp = (float *) malloc(w * oh * (size_t) ch * sizeof(float));
    if (!tmp) return -1;
    resize_axis(&rf, src, w, h, ch, tmp, oh, yf, 1);
    resize_axis(&rf, tmp, w, oh, ch, dst, ow, xf, 0);
  }
  free(tmp);
  return 0;
}

/* -------------------------------------------------------------- colorspace */

/* pixel.c:260-316 DecodeGamma: x^2.4 via Chebyshev on the frexp mantissa */
static double decode_gamma(double x)
{
  static const double cf[9] = { 1.7917488588043277509, 0.82045614371976854984, 0.027694100686325412819,
    -0.00094244335181762134018, 0.000064355540911469709545, -5.7224404636060757485e-06,
    5.8767669437311184313e-07, -6.6139920053589721168e-08, 7.9323242696227458163e-09 };
  static const double p2[5] = { 1.0, 2.6390158215457883983, 6.9644045063689921093,
    1.8379173679952558018e+01, 4.8502930128332728543e+01 };
  double t[9], p;
  int e, quot, rem, i;
  t[0] = 1.0;
  t[1] = 4.0 * frexp(x, &e) - 3.0;
  for (i = 2; i < 9; i++) t[i] = 2.0 * t[1] * t[i - 1] - t[i - 2];
  p = cf[0] * t[0] + cf[1] * t[1] + cf[2] * t[2] + cf[3] * t[3] + cf[4] * t[4] + cf[5] * t[5] +
      cf[6] * t[6] + cf[7] * t[7] + cf[8] * t[8];
  quot = (e - 1) / 5; rem = (e - 1) % 5;
  if (rem < 0) { quot -= 1; rem += 5; }
  return x * ldexp(p2[rem] * p, 7 * quot);
}

/* pixel.c:318-324 */
static double decode_pixel_gamma(double pixel)
{
  if (pixel <= (0.0404482362771076 * (double) QR)) return pixel / 12.92;
  return (double) QR * decode_gamma((double) (QS * pixel + 0.055) / 1.055);
}

/* pixel.c:380-443 EncodeGamma: x^(1/2.4) */
static double encode_gamma(double x)
{
  static const double cf[9] = { 1.1758200232996901923, 0.16665763094889061230, -0.0083154894939042125035,
    0.00075187976780420279038, -0.000083240178519391795367, 0.000010229209410070008679,
    -1.3400466409860246e-06, 1.8333422241635376682e-07, -2.5878596761348859722e-08 };
  static const double p2[12] = { 1.0, 1.3348398541700343678, 1.7817974362806785482, 2.3784142300054420538,
    3.1748021039363991669, 4.2378523774371812394, 5.6568542494923805819, 7.5509945014535482244,
    1.0079368399158985525e1, 1.3454342644059433809e1, 1.7959392772949968275e1, 2.3972913230026907883e1 };
  double t[9], p;
  int e, quot, rem, i;
  t[0] = 1.0;
  t[1] = 4.0 * frexp(x, &e) - 3.0;
  for (i = 2; i < 9; i++) t[i] = 2.0 * t[1] * t[i - 1] - t[i - 2];
  p = cf[0] * t[0] + cf[1] * t[1] + cf[2] * t[2] + cf[3] * t[3] + cf[4] * t[4] + cf[5] * t[5] +
      cf[6] * t[6] + cf[7] * t[7] + cf[8] * t[8];
  quot = (e - 1) / 12; rem = (e - 1) % 12;
  if (rem < 0) { quot -= 1; rem += 12; }
  return ldexp(p2[rem] * p, 5 * quot);
}

/* pixel.c:445-451 */
static double encode_pixel_gamma(double pixel)
{
  if (pixel <= (0.0031306684425005883 * (double) QR)) return 12.92 * pixel;
  return (double) QR * (1.055 * encode_gamma((double) QS * pixel) - 0.055);
}

/* illuminant_tristimulus[] (colorspace-private.h:32-46), indexed by IlluminantType (color.h:40-54); D65 unless the
   "color:illuminant" artifact names another (colorspace.c:761-773) */
static const double illuminant_table[11][3] = {
  {1.09850, 1.00000, 0.35585}, {0.99072, 1.00000, 0.85223}, {0.98074, 1.00000, 1.18232}, {0.96422, 1.00000, 0.82521},
  {0.95682, 1.00000, 0.92149}, {0.95047, 1.00000, 1.08883}, {0.94972, 1.00000, 1.22638}, {1.00000, 1.00000, 1.00000},
  {0.99186, 1.00000, 0.67393}, {0.95041, 1.00000, 1.08747}, {1.00962, 1.00000, 0.64350}};
static double cs_ill[3] = {0.95047, 1.00000, 1.08883};
static double cs_white_luminance = 10000.0;
#define ILL_X cs_ill[0]
#define ILL_Y cs_ill[1]
#define ILL_Z cs_ill[2]
#define CIE_EPS (216.0 / 24389.0)
#define CIE_K   (24389.0 / 27.0)

/* colorspace-private.h:759-779 */
static void rgb_to_xyz(double red, double green, double blue, double *X, double *Y, double *Z)
{
  double r = QS * decode_pixel_gamma(red), g = QS * decode_pixel_gamma(green), b = QS * decode_pixel_gamma(blue);
  *X = (0.4123955889674142161 * r) + (0.3575834307637148171 * g) + (0.1804926473817015735 * b);
  *Y = (0.2125862307855955516 * r) + (0.7151703037034108499 * g) + (0.07220049864333622685 * b);
  *Z = (0.01929721549174694484 * r) + (0.1191838645808485318 * g) + (0.9504971251315797660 * b);
}

/* colorspace-private.h:72-94 */
static void xyz_to_rgb(double X, double Y, double Z, double *red, double *green, double *blue)
{
  double r = (3.240969941904521 * X) + (-1.537383177570093 * Y) + (-0.498610760293 * Z);
  double g = (-0.96924363628087 * X) + (1.87596750150772 * Y) + (0.041555057407175 * Z);
  double b = (0.055630079696993 * X) + (-0.20397695888897 * Y) + (1.056971514242878 * Z);
  /* MagickMin is a plain (x<y?x:y) macro */
  double m = r < (g < b ? g : b) ? r : (g < b ? g : b);
  if (m < 0.0) { r -= m; g -= m; b -= m; }
  *red = encode_pixel_gamma((double) QR * r);
  *green = encode_pixel_gamma((double) QR * g);
  *blue = encode_pixel_gamma((double) QR * b);
}

/* colorspace-private.h:1066-1089 */
static void xyz_to_lab(double X, double Y, double Z, double *L, double *a, double *b)
{
  double x, y, z;
  if ((X / ILL_X) > CIE_EPS) x = pow(X / ILL_X, 1.0 / 3.0); else x = (CIE_K * X / ILL_X + 16.0) / 116.0;
  if ((Y / ILL_Y) > CIE_EPS) y = pow(Y / ILL_Y, 1.0 / 3.0); else y = (CIE_K * Y / ILL_Y + 16.0) / 116.0;
  if ((Z / ILL_Z) > CIE_EPS) z = pow(Z / ILL_Z, 1.0 / 3.0); else z = (CIE_K * Z / ILL_Z + 16.0) / 116.0;
  *L = ((116.0 * y) - 16.0) / 100.0;
  *a = (500.0 * (x - y)) / 255.0 + 0.5;
  *b = (200.0 * (y - z)) / 255.0 + 0.5;
}

/* colorspace-private.h:531-557 */
static void lab_to_xyz(double L, double a, double b, double *X, double *Y, double *Z)
{
  double x, y, z;
  y = (L + 16.0) / 116.0;
  x = y + a / 500.0;
  z = y - b / 200.0;
  if ((x * x * x) > CIE_EPS) x = (x * x * x); else x = (116.0 * x - 16.0) / CIE_K;
  if (L > (CIE_K * CIE_EPS)) y = (y * y * y); else y = L / CIE_K;
  if ((z * z * z) > CIE_EPS) z = (z * z * z); else z = (116.0 * z - 16.0) / CIE_K;
  *X = ILL_X * x; *Y = ILL_Y * y; *Z = ILL_Z * z;
}

/* colorspace.c:1751-1783; forward generic branch :958-1054, linear :1164-1225;
   inverse generic :2296-2390, linear RGB->sRGB :2494-2550 */
static int colorspace_core(float *buf, size_t w, size_t h, int ch, int from, int to)
{
  const long n = (long) (w * h);
  long i;
  if (ch < 3) return -1;
  if (from == to) return 0;
  if (from != ORC_CS_SRGB) {
    if (from != ORC_CS_LAB && from != ORC_CS_XYZ && from != ORC_CS_RGB) return -1;
#pragma omp parallel for schedule(static)
    for (i = 0; i < n; i++) {
      float *q = buf + (size_t) i * ch;
      double r, g, b;
      if (from == ORC_CS_RGB) {
        r = encode_pixel_gamma((double) q[0]);
        g = encode_pixel_gamma((double) q[1]);
        b = encode_pixel_gamma((double) q[2]);
      } else {
        double X = QS * q[0], Y = QS * q[1], Z = QS * q[2];
        if (from == ORC_CS_LAB) {
          double x2, y2, z2;
          lab_to_xyz(100.0 * X, 255.0 * (Y - 0.5), 255.0 * (Z - 0.5), &x2, &y2, &z2);
          X = x2; Y = y2; Z = z2;
        }
        xyz_to_rgb(X, Y, Z, &r, &g, &b);
      }
      q[0] = (float) r; q[1] = (float) g; q[2] = (float) b;
    }
  }
  if (to == ORC_CS_SRGB) return 0;
  if (to != ORC_CS_LAB && to != ORC_CS_XYZ && to != ORC_CS_RGB) return -1;
#pragma omp parallel for schedule(static)
  for (i = 0; i < n; i++) {
    float *q = buf + (size_t) i * ch;
    if (to == ORC_CS_RGB) {
      double r = decode_pixel_gamma((double) q[0]), g = decode_pixel_gamma((double) q[1]),
             b = decode_pixel_gamma((double) q[2]);
      q[0] = (float) r; q[1] = (float) g; q[2] = (float) b;
    } else {
      double X, Y, Z;
      rgb_to_xyz((double) q[0], (double) q[1], (double) q[2], &X, &Y, &Z);
      if (to == ORC_CS_LAB) {
        double L, a, b;
        xyz_to_lab(X, Y, Z, &L, &a, &b);
        X = L; Y = a; Z = b;
      }
      q[0] = (float) ((double) QR * X); q[1] = (float) ((double) QR * Y); q[2] = (float) ((double) QR * Z);
    }
  }
  return 0;
}



/* ---- matrix colourspaces -------------------------------------------------------------------------
   Generic branch (colorspace.c:958-1054 forward, :2296-2390 inverse) through
   ConvertRGBToGeneric / ConvertGenericToRGB for CMY, YCbCr (= YPbPr), YDbDr, YIQ, YPbPr, YUV
   (colorspace-private.h:793-798, :141-147, :1551-1593, :1637-1701): each component is
   QS*(m0*R+m1*G+m2*B) [+0.5], stored as (float)(QR*X); inverse QR*(a0*Y+a1*(U-.5)+a2*(V-.5)).
   LUT branch (forward :1229-1494, inverse :2560-2830) for OHTA, Rec601YCbCr, Rec709YCbCr: the
   samples are first quantised to a 16-bit map index (ScaleQuantumToMap, quantum-private.h:504-514),
   the tables hold c*i (forward) or c*i / K*(2i-MaxMap) (inverse) in double, three entries are
   summed left to right (+ the primary offset), and ScaleMapToQuantum clamps to 0..QuantumRange. */
typedef struct { double m[3][3]; double off[3]; } cs_matrix;

static const cs_matrix *generic_forward(int cs)
{
  static const cs_matrix ydbdr = {{{0.298839, 0.586811, 0.114350}, {-0.450, -0.883, 1.333}, {-1.333, 1.116, 0.217}}, {0, 0.5, 0.5}};
  static const cs_matrix yiq = {{{0.298839, 0.586811, 0.114350}, {0.595716, -0.274453, -0.321263}, {0.211456, -0.522591, 0.311135}}, {0, 0.5, 0.5}};
  static const cs_matrix ypbpr = {{{0.298839, 0.586811, 0.114350}, {-0.1687367, -0.331264, 0.5}, {0.5, -0.418688, -0.081312}}, {0, 0.5, 0.5}};
  static const cs_matrix yuv = {{{0.298839, 0.586811, 0.114350}, {-0.147, -0.289, 0.436}, {0.615, -0.515, -0.100}}, {0, 0.5, 0.5}};
  switch (cs) {
    case ORC_CS_YDBDR: return &ydbdr;
    case ORC_CS_YIQ: return &yiq;
    case ORC_CS_YCBCR: case ORC_CS_YPBPR: return &ypbpr;
    case ORC_CS_YUV: return &yuv;
    default: return NULL;
  }
}

static const cs_matrix *generic_inverse(int cs)
{
  static const cs_matrix ydbdr = {{{1.0, 9.2303716147657e-05, -0.52591263066186533}, {1.0, -0.12913289889050927, 0.26789932820759876},
                                   {1.0, 0.66467905997895482, -7.9202543533108e-05}}, {0, 0, 0}};
  static const cs_matrix yiq = {{{1.0, 0.9562957197589482261, 0.6210244164652610754}, {1.0, -0.2721220993185104464, -0.6473805968256950427},
                                 {1.0, -1.1069890167364901945, 1.7046149983646481374}}, {0, 0, 0}};
  static const cs_matrix ypbpr = {{{0.99999999999914679361, -1.2188941887145875e-06, 1.4019995886561440468},
                                   {0.99999975910502514331, -0.34413567816504303521, -0.71413649331646789076},
                                   {1.00000124040004623180, 1.77200006607230409200, 2.1453384174593273e-06}}, {0, 0, 0}};
  static const cs_matrix yuv = {{{1.0, -3.945707070708279e-05, 1.1398279671717170825}, {1.0, -0.3946101641414141437, -0.5805003156565656797},
                                 {1.0, 2.0319996843434342537, -4.813762626262513e-04}}, {0, 0, 0}};
  switch (cs) {
    case ORC_CS_YDBDR: return &ydbdr;
    case ORC_CS_YIQ: return &yiq;
    case ORC_CS_YCBCR: case ORC_CS_YPBPR: return &ypbpr;
    case ORC_CS_YUV: return &yuv;
    default: return NULL;
  }
}

static unsigned int scale_quantum_to_map(float q)      /* quantum-private.h:504-514 (HDRI) */
{
  if (q >= (float) 65535.0f) return 65535u;
  if (q != q || q <= 0.0f) return 0u;
  return (unsigned int) (q + 0.5f);
}

static float scale_map_to_quantum(double v)            /* quantum-private.h (HDRI): clamp, no rounding */
{
  if (v <= 0.0) return 0.0f;
  if (v >= 65535.0) return 65535.0f;
  return (float) v;
}

static int lut_forward_coeffs(int cs, double c[3][3])
{
  static const double ohta[3][3] = {{0.33333, 0.33334, 0.33333}, {0.50000, 0.00000, -0.50000}, {-0.25000, 0.50000, -0.25000}};
  static const double r601[3][3] = {{0.298839, 0.586811, 0.114350}, {-0.1687367, -0.331264, 0.500000}, {0.500000, -0.418688, -0.081312}};
  static const double r709[3][3] = {{0.212656, 0.715158, 0.072186}, {-0.114572, -0.385428, 0.500000}, {0.500000, -0.454153, -0.045847}};
  const double (*t)[3] = cs == ORC_CS_OHTA ? ohta : cs == ORC_CS_REC601YCBCR ? r601 : cs == ORC_CS_REC709YCBCR ? r709 : NULL;
  if (!t) return -1;
  memcpy(c, t, sizeof(double) * 9);
  return 0;
}

/* inverse tables: row k of the result = x[k]*i_r + (0.5*y[k])*(2 i_g - MaxMap) + (0.5*z[k])*(2 i_b - MaxMap) */
static int lut_inverse_coeffs(int cs, double x[3], double y[3], double z[3])
{
  if (cs == ORC_CS_OHTA) {
    x[0] = x[1] = x[2] = 1.0;
    y[0] = 0.5 * 1.00000; y[1] = 0.5 * 0.00000; y[2] = -0.5 * 1.00000;
    z[0] = -0.5 * 0.66668; z[1] = 0.5 * 1.33333; z[2] = -0.5 * 0.66668;
  } else if (cs == ORC_CS_REC601YCBCR) {
    x[0] = 0.99999999999914679361; x[1] = 0.99999975910502514331; x[2] = 1.00000124040004623180;
    y[0] = 0.5 * (-1.2188941887145875e-06); y[1] = 0.5 * (-0.34413567816504303521); y[2] = 0.5 * 1.77200006607230409200;
    z[0] = 0.5 * 1.4019995886561440468; z[1] = 0.5 * (-0.71413649331646789076); z[2] = 0.5 * 2.1453384174593273e-06;
  } else if (cs == ORC_CS_REC709YCBCR) {
    x[0] = x[1] = x[2] = 1.0;
    y[0] = 0.5 * 0.000000; y[1] = 0.5 * (-0.187324); y[2] = 0.5 * 1.855600;
    z[0] = 0.5 * 1.574800; z[1] = 0.5 * (-0.468124); z[2] = 0.5 * 0.000000;
  } else return -1;
  return 0;
}

static int is_core_space(int cs) { return cs == ORC_CS_SRGB || cs == ORC_CS_LAB || cs == ORC_CS_XYZ || cs == ORC_CS_RGB; }

/* one leg: sRGB -> `to` (forward != 0) or `from` -> sRGB, for the matrix / LUT / CMY spaces */
static int colorspace_matrix_leg(float *buf, long n, int ch, int cs, int forward)
{
  long i;
  double c[3][3], ix[3], iy[3], iz[3];
  const cs_matrix *gm = forward ? generic_forward(cs) : generic_inverse(cs);
  const int lut = lut_forward_coeffs(cs, c) == 0;
  if (lut && !forward) lut_inverse_coeffs(cs, ix, iy, iz);
  if (!gm && !lut && cs != ORC_CS_CMY) return -1;
#pragma omp parallel for schedule(static)
  for (i = 0; i < n; i++) {
    float *q = buf + (size_t) i * ch;
    int k;
    if (lut) {
      const double r = (double) scale_quantum_to_map(q[0]), g = (double) scale_quantum_to_map(q[1]),
                   b = (double) scale_quantum_to_map(q[2]);
      float o[3];
      for (k = 0; k < 3; k++) {
        double v;
        if (forward) v = ((c[k][0] * r + c[k][1] * g) + c[k][2] * b) + (k == 0 ? 0.0 : 32768.0);
        else v = (ix[k] * r + iy[k] * (2.0 * g - 65535.0)) + iz[k] * (2.0 * b - 65535.0);
        o[k] = scale_map_to_quantum(v);
      }
      q[0] = o[0]; q[1] = o[1]; q[2] = o[2];
    } else if (cs == ORC_CS_CMY) {
      for (k = 0; k < 3; k++) {
        if (forward) q[k] = (float) (QR * (QS * (QR - (double) q[k])));
        else q[k] = (float) (QR * (1.0 - QS * (double) q[k]));
      }
    } else if (forward) {
      const double R = q[0], G = q[1], B = q[2];
      float o[3];
      for (k = 0; k < 3; k++) {
        double X = QS * ((gm->m[k][0] * R + gm->m[k][1] * G) + gm->m[k][2] * B);
        if (k) X += 0.5;
        o[k] = (float) (QR * X);
      }
      q[0] = o[0]; q[1] = o[1]; q[2] = o[2];
    } else {
      const double Y = QS * q[0], U = QS * q[1] - 0.5, V = QS * q[2] - 0.5;
      float o[3];
      for (k = 0; k < 3; k++) {
        const double t = gm->m[k][0] == 1.0 ? Y : gm->m[k][0] * Y;
        o[k] = (float) (QR * ((t + gm->m[k][1] * U) + gm->m[k][2] * V));
      }
      q[0] = o[0]; q[1] = o[1]; q[2] = o[2];
    }
  }
  return 0;
}

/* ------------------------------------------------------------------------------------------
   Hexcone colourspaces of the generic branch (colorspace.c:958-1054 forward, :2296-2390 inverse):
   HCL, HCLp, HSB, HSI, HSL, HSV, HWB.  Forward takes Quantum-range R, G, B and returns unit-range
   components that are stored as (float) (QuantumRange * X); inverse takes QuantumScale * sample and
   returns Quantum-range values that are cast to float (HDRI ClampToQuantum).
   ------------------------------------------------------------------------------------------ */
#define ORC_MAX(x, y) (((x) > (y)) ? (x) : (y))
#define ORC_MIN(x, y) (((x) < (y)) ? (x) : (y))

static void rgb_to_hcl(double red, double green, double blue, double *hue, double *chroma, double *luma)
{ /* colorspace-private.h:801-832 (HCL) and :834-865 (HCLp): identical forward transforms */
  double c, h, max;
  max = ORC_MAX(red, ORC_MAX(green, blue));
  c = max - (double) ORC_MIN(red, ORC_MIN(green, blue));
  h = 0.0;
  if (fabs(c) < EPS) h = 0.0;
  else if (fabs(red - max) < EPS) h = fmod((green - blue) / c + 6.0, 6.0);
  else if (fabs(green - max) < EPS) h = ((blue - red) / c) + 2.0;
  else if (fabs(blue - max) < EPS) h = ((red - green) / c) + 4.0;
  *hue = (h / 6.0);
  *chroma = QS * c;
  *luma = QS * (0.298839 * red + 0.586811 * green + 0.114350 * blue);
}

static void hcl_to_rgb(double hue, double chroma, double luma, int clip, double *red, double *green, double *blue)
{ /* colorspace-private.h:149-212 (HCL), :214-290 (HCLp: clip != 0) */
  double b = 0.0, c, g = 0.0, h, m, r = 0.0, x, z;
  h = 6.0 * hue;
  c = chroma;
  x = c * (1.0 - fabs(fmod(h, 2.0) - 1.0));
  if ((0.0 <= h) && (h < 1.0)) { r = c; g = x; }
  else if ((1.0 <= h) && (h < 2.0)) { r = x; g = c; }
  else if ((2.0 <= h) && (h < 3.0)) { g = c; b = x; }
  else if ((3.0 <= h) && (h < 4.0)) { g = x; b = c; }
  else if ((4.0 <= h) && (h < 5.0)) { r = x; b = c; }
  else if ((5.0 <= h) && (h < 6.0)) { r = c; b = x; }
  m = luma - (0.298839 * r + 0.586811 * g + 0.114350 * b);
  if (!clip) {
    *red = QR * (r + m); *green = QR * (g + m); *blue = QR * (b + m);
    return;
  }
  z = 1.0;
  if (m < 0.0) { z = luma / (luma - m); m = 0.0; }
  else if (m + c > 1.0) { z = (1.0 - luma) / (m + c - luma); m = 1.0 - z * c; }
  *red = QR * (z * r + m); *green = QR * (z * g + m); *blue = QR * (z * b + m);
}

static void rgb_to_hsb(double red, double green, double blue, double *hue, double *saturation, double *brightness)
{ /* colorspace-private.h:867-907 */
  double delta, max, min;
  *hue = 0.0; *saturation = 0.0; *brightness = 0.0;
  min = red < green ? red : green;
  if (blue < min) min = blue;
  max = red > green ? red : green;
  if (blue > max) max = blue;
  if (fabs(max) < EPS) return;
  delta = max - min;
  *saturation = delta / max;
  *brightness = QS * max;
  if (fabs(delta) < EPS) return;
  if (fabs(red - max) < EPS) *hue = (green - blue) / delta;
  else if (fabs(green - max) < EPS) *hue = 2.0 + (blue - red) / delta;
  else *hue = 4.0 + (red - green) / delta;
  *hue /= 6.0;
  if (*hue < 0.0) *hue += 1.0;
}

static void hsb_to_rgb(double hue, double saturation, double brightness, double *red, double *green, double *blue)
{ /* colorspace-private.h:292-366 */
  double f, h, p, q, t;
  if (fabs(saturation) < EPS) {
    *red = QR * brightness; *green = (*red); *blue = (*red);
    return;
  }
  h = 6.0 * (hue - floor(hue));
  f = h - floor((double) h);
  p = brightness * (1.0 - saturation);
  q = brightness * (1.0 - saturation * f);
  t = brightness * (1.0 - (saturation * (1.0 - f)));
  switch ((int) h) {
    case 0: default: *red = QR * brightness; *green = QR * t; *blue = QR * p; break;
    case 1: *red = QR * q; *green = QR * brightness; *blue = QR * p; break;
    case 2: *red = QR * p; *green = QR * brightness; *blue = QR * t; break;
    case 3: *red = QR * p; *green = QR * q; *blue = QR * brightness; break;
    case 4: *red = QR * t; *green = QR * p; *blue = QR * brightness; break;
    case 5: *red = QR * brightness; *green = QR * p; *blue = QR * q; break;
  }
}

static void rgb_to_hsi(double red, double green, double blue, double *hue, double *saturation, double *intensity)
{ /* colorspace-private.h:909-936 */
  double alpha, beta;
  *intensity = (QS * red + QS * green + QS * blue) / 3.0;
  if (*intensity <= 0.0) { *hue = 0.0; *saturation = 0.0; return; }
  *saturation = 1.0 - ORC_MIN(QS * red, ORC_MIN(QS * green, QS * blue)) / (*intensity);
  alpha = 0.5 * (2.0 * QS * red - QS * green - QS * blue);
  beta = 0.8660254037844385 * (QS * green - QS * blue);
  *hue = atan2(beta, alpha) * (180.0 / PI_) / 360.0;
  if (*hue < 0.0) *hue += 1.0;
}

static void hsi_to_rgb(double hue, double saturation, double intensity, double *red, double *green, double *blue)
{ /* colorspace-private.h:368-412 */
  double b, g, h, r;
  h = 360.0 * hue;
  h -= 360.0 * floor(h / 360.0);
  if (h < 120.0) {
    b = intensity * (1.0 - saturation);
    r = intensity * (1.0 + saturation * cos(h * (PI_ / 180.0)) / cos((60.0 - h) * (PI_ / 180.0)));
    g = 3.0 * intensity - r - b;
  } else if (h < 240.0) {
    h -= 120.0;
    r = intensity * (1.0 - saturation);
    g = intensity * (1.0 + saturation * cos(h * (PI_ / 180.0)) / cos((60.0 - h) * (PI_ / 180.0)));
    b = 3.0 * intensity - r - g;
  } else {
    h -= 240.0;
    g = intensity * (1.0 - saturation);
    b = intensity * (1.0 + saturation * cos(h * (PI_ / 180.0)) / cos((60.0 - h) * (PI_ / 180.0)));
    r = 3.0 * intensity - g - b;
  }
  *red = QR * r; *green = QR * g; *blue = QR * b;
}

static void rgb_to_hsl_hsv(double red, double green, double blue, int hsv, double *hue, double *saturation, double *third)
{ /* ConvertRGBToHSL colorspace.c:597-640, ConvertRGBToHSV colorspace-private.h:994-1033 */
  double c, max, min;
  max = ORC_MAX(QS * red, ORC_MAX(QS * green, QS * blue));
  min = ORC_MIN(QS * red, ORC_MIN(QS * green, QS * blue));
  c = max - min;
  *third = hsv ? max : (max + min) / 2.0;
  if (c <= 0.0) { *hue = 0.0; *saturation = 0.0; return; }
  if (fabs(max - QS * red) < EPS) {
    *hue = (QS * green - QS * blue) / c;
    if ((QS * green) < (QS * blue)) *hue += 6.0;
  } else if (fabs(max - QS * green) < EPS) *hue = 2.0 + (QS * blue - QS * red) / c;
  else *hue = 4.0 + (QS * red - QS * green) / c;
  *hue *= 60.0 / 360.0;
  if (hsv) *saturation = c * precip(max);
  else if (*third <= 0.5) *saturation = c * precip(2.0 * (*third));
  else *saturation = c * precip(2.0 - 2.0 * (*third));
}

static void hsl_hsv_to_rgb(double hue, double saturation, double third, int hsv, double *red, double *green, double *blue)
{ /* ConvertHSLToRGB colorspace.c:307-385, ConvertHSVToRGB colorspace-private.h:414-481 */
  double c, h, min, x;
  h = hue * 360.0;
  if (hsv) { c = third * saturation; min = third - c; }
  else {
    if (third <= 0.5) c = 2.0 * third * saturation;
    else c = (2.0 - 2.0 * third) * saturation;
    min = third - 0.5 * c;
  }
  h -= 360.0 * floor(h / 360.0);
  h /= 60.0;
  x = c * (1.0 - fabs(h - 2.0 * floor(h / 2.0) - 1.0));
  switch ((int) floor(h)) {
    case 0: default: *red = QR * (min + c); *green = QR * (min + x); *blue = QR * min; break;
    case 1: *red = QR * (min + x); *green = QR * (min + c); *blue = QR * min; break;
    case 2: *red = QR * min; *green = QR * (min + c); *blue = QR * (min + x); break;
    case 3: *red = QR * min; *green = QR * (min + x); *blue = QR * (min + c); break;
    case 4: *red = QR * (min + x); *green = QR * min; *blue = QR * (min + c); break;
    case 5: *red = QR * (min + c); *green = QR * min; *blue = QR * (min + x); break;
  }
}

static void rgb_to_hwb(double red, double green, double blue, double *hue, double *whiteness, double *blackness)
{ /* colorspace-private.h:1035-1064 */
  double f, p, v, w;
  w = ORC_MIN(red, ORC_MIN(green, blue));
  v = ORC_MAX(red, ORC_MAX(green, blue));
  *blackness = 1.0 - QS * v;
  *whiteness = QS * w;
  if (fabs(v - w) < EPS) { *hue = (-1.0); return; }
  f = (fabs(red - w) < EPS) ? green - blue : ((fabs(green - w) < EPS) ? blue - red : red - green);
  p = (fabs(red - w) < EPS) ? 3.0 : ((fabs(green - w) < EPS) ? 5.0 : 1.0);
  *hue = (p - f / (v - 1.0 * w)) / 6.0;
}

static void hwb_to_rgb(double hue, double whiteness, double blackness, double *red, double *green, double *blue)
{ /* colorspace-private.h:483-529; CastDoubleToLong image-private.h:67 (NaN -> 0, saturating) */
  double b, f, g, n, r, v, fl;
  long i;
  v = 1.0 - blackness;
  if (fabs(hue - (-1.0)) < EPS) { *red = QR * v; *green = QR * v; *blue = QR * v; return; }
  fl = floor(6.0 * hue);
  if (fl != fl) i = 0;
  else if (fl < -9223372036854775808.0) i = (-9223372036854775807L - 1);
  else if (fl > 9223372036854775807.0) i = 9223372036854775807L;
  else i = (long) fl;
  f = 6.0 * hue - i;
  if ((i & 0x01) != 0) f = 1.0 - f;
  n = whiteness + f * (v - whiteness);
  switch (i) {
    case 0: default: r = v; g = n; b = whiteness; break;
    case 1: r = n; g = v; b = whiteness; break;
    case 2: r = whiteness; g = v; b = n; break;
    case 3: r = whiteness; g = n; b = v; break;
    case 4: r = n; g = whiteness; b = v; break;
    case 5: r = v; g = whiteness; b = n; break;
  }
  *red = QR * r; *green = QR * g; *blue = QR * b;
}

static int is_hexcone_space(int cs)
{
  return cs == ORC_CS_HCL || cs == ORC_CS_HCLP || cs == ORC_CS_HSB || cs == ORC_CS_HSI || cs == ORC_CS_HSL ||
         cs == ORC_CS_HSV || cs == ORC_CS_HWB;
}

/* one leg: sRGB -> `cs` (forward != 0, colorspace.c:1038-1043) or `cs` -> sRGB (:2373-2379) */
static int colorspace_hexcone_leg(float *buf, long n, int ch, int cs, int forward)
{
  long i;
  if (!is_hexcone_space(cs)) return -1;
#pragma omp parallel for schedule(static)
  for (i = 0; i < n; i++) {
    float *q = buf + (size_t) i * ch;
    double X, Y, Z;
    if (forward) {
      const double R = (double) q[0], G = (double) q[1], B = (double) q[2];
      switch (cs) {
        case ORC_CS_HCL: case ORC_CS_HCLP: rgb_to_hcl(R, G, B, &X, &Y, &Z); break;
        case ORC_CS_HSB: rgb_to_hsb(R, G, B, &X, &Y, &Z); break;
        case ORC_CS_HSI: rgb_to_hsi(R, G, B, &X, &Y, &Z); break;
        case ORC_CS_HSL: rgb_to_hsl_hsv(R, G, B, 0, &X, &Y, &Z); break;
        case ORC_CS_HSV: rgb_to_hsl_hsv(R, G, B, 1, &X, &Y, &Z); break;
        default: rgb_to_hwb(R, G, B, &X, &Y, &Z); break;
      }
      q[0] = (float) (QR * X); q[1] = (float) (QR * Y); q[2] = (float) (QR * Z);
    } else {
      const double a = QS * q[0], b = QS * q[1], c = QS * q[2];
      switch (cs) {
        case ORC_CS_HCL: hcl_to_rgb(a, b, c, 0, &X, &Y, &Z); break;
        case ORC_CS_HCLP: hcl_to_rgb(a, b, c, 1, &X, &Y, &Z); break;
        case ORC_CS_HSB: hsb_to_rgb(a, b, c, &X, &Y, &Z); break;
        case ORC_CS_HSI: hsi_to_rgb(a, b, c, &X, &Y, &Z); break;
        case ORC_CS_HSL: hsl_hsv_to_rgb(a, b, c, 0, &X, &Y, &Z); break;
        case ORC_CS_HSV: hsl_hsv_to_rgb(a, b, c, 1, &X, &Y, &Z); break;
        default: hwb_to_rgb(a, b, c, &X, &Y, &Z); break;
      }
      q[0] = (float) X; q[1] = (float) Y; q[2] = (float) Z;
    }
  }
  return 0;
}

/* ------------------------------------------------------------------------------------------
   XYZ-derived colourspaces of the generic branch (colorspace.c:958-1054 / :2296-2390): Adobe98, DisplayP3, ProPhoto
   (an RGB matrix + the sRGB transfer curve on either side of XYZ), LMS, CAT02LMS, xyY, Luv.
   ------------------------------------------------------------------------------------------ */
typedef struct { double m[3][3]; } mat3;
/* colorspace-private.h:53-70 / :675-692 / :719-737 (X is assigned twice there: the second row set counts) */
static const mat3 adobe98_to_xyz = {{{0.57666904291013050, 0.18555823790654630, 0.18822864623499470},
                                     {0.29734497525053605, 0.62736356625546610, 0.07529145849399788},
                                     {0.02703136138641234, 0.07068885253582723, 0.99133753683763880}}};
static const mat3 displayp3_to_xyz = {{{0.4865709486482162, 0.26566769316909306, 0.1982172852343625},
                                       {0.2289745640697488, 0.69173852183650640, 0.0792869140937450},
                                       {0.0000000000000000, 0.04511338185890264, 1.0439443689009760}}};
static const mat3 prophoto_to_xyz = {{{0.7977604896723027, 0.13518583717574031, 0.03134934958152480000},
                                      {0.2880711282292934, 0.71184321781010140, 0.00008565396060525902},
                                      {0.0000000000000000, 0.00000000000000000, 0.82510460251046010000}}};
/* :938-952 / :966-980 / :1197-1211 */
static const mat3 xyz_to_adobe98 = {{{2.041587903810746500, -0.56500697427885960, -0.34473135077832956},
                                     {-0.969243636280879500, 1.87596750150772020, 0.04155505740717557},
                                     {0.013444280632031142, -0.11836239223101838, 1.01517499439120540}}};
static const mat3 xyz_to_displayp3 = {{{2.49349691194142500, -0.93138361791912390, -0.402710784450716840},
                                       {-0.82948896956157470, 1.76266406031834630, 0.023624685841943577},
                                       {0.03584583024378447, -0.07617238926804182, 0.956884524007687200}}};
static const mat3 xyz_to_prophoto = {{{1.3457989731028281, -0.25558010007997534, -0.05110628506753401},
                                      {-0.5446224939028347, 1.50823274131327810, 0.02053603239147973},
                                      {0.0000000000000000, 0.0000000000000000, 1.21196754563894540}}};
/* a*x + b*y + c*z exactly as the reference writes it: negative coefficients appear as subtractions there, which is the
   same IEEE result as adding the product with the negated constant */
static double row3(const double *r, double x, double y, double z) { return r[0] * x + r[1] * y + r[2] * z; }

static void xyz_to_lms(double x, double y, double z, double *L, double *M, double *S)
{ /* colorspace-private.h:1225-1231 (LMS) == :751-757 (CAT02LMS) */
  *L = 0.7328 * x + 0.4296 * y - 0.1624 * z;
  *M = (-0.7036 * x + 1.6975 * y + 0.0061 * z);
  *S = 0.0030 * x + 0.0136 * y + 0.9834 * z;
}
static void lms_to_xyz(double L, double M, double S, double *X, double *Y, double *Z)
{ /* :655-661 == :108-117 */
  *X = 1.096123820835514 * L - 0.278869000218287 * M + 0.182745179382773 * S;
  *Y = 0.454369041975359 * L + 0.473533154307412 * M + 0.072097803717229 * S;
  *Z = (-0.009627608738429) * L - 0.005698031216113 * M + 1.015325639954543 * S;
}

#define LUV_UN (4.0 * ILL_X / (ILL_X + 15.0 * ILL_Y + 3.0 * ILL_Z))
#define LUV_VN (9.0 * ILL_Y / (ILL_X + 15.0 * ILL_Y + 3.0 * ILL_Z))
static void xyz_to_luv(double X, double Y, double Z, double *L, double *u, double *v)
{ /* :1138-1161 */
  double alpha;
  if ((Y / ILL_Y) > CIE_EPS) *L = (double) (116.0 * pow(Y / ILL_Y, 1.0 / 3.0) - 16.0);
  else *L = CIE_K * (Y / ILL_Y);
  alpha = precip(X + 15.0 * Y + 3.0 * Z);
  *u = 13.0 * (*L) * ((4.0 * alpha * X) - LUV_UN);
  *v = 13.0 * (*L) * ((9.0 * alpha * Y) - LUV_VN);
  *L /= 100.0;
  *u = (*u + 134.0) / 354.0;
  *v = (*v + 140.0) / 262.0;
}
static void luv_to_xyz(double L, double u, double v, double *X, double *Y, double *Z)
{ /* :600-625 */
  double gamma;
  if (L > (CIE_K * CIE_EPS)) *Y = (double) pow((L + 16.0) / 116.0, 3.0);
  else *Y = L / CIE_K;
  gamma = precip((((52.0 * L * precip(u + 13.0 * L * LUV_UN)) - 1.0) / 3.0) - (-1.0 / 3.0));
  *X = gamma * ((*Y * ((39.0 * L * precip(v + 13.0 * L * LUV_VN)) - 5.0)) + 5.0 * (*Y));
  *Z = (*X * (((52.0 * L * precip(u + 13.0 * L * LUV_UN)) - 1.0) / 3.0)) - 5.0 * (*Y);
}

/* Oklab / Oklch (colorspace-private.h:1480-1549): cube roots of an LMS-like matrix of linear RGB; the polar form is taken
   of the OFFSET a, b (0.5 + ...), so the hue of an achromatic pixel is atan2(-0.5, -0.5), not noise */
static void rgb_to_oklab(double red, double green, double blue, double *L, double *a, double *b)
{
  double B, G, l, m, R, s;
  R = QS * decode_pixel_gamma(red);
  G = QS * decode_pixel_gamma(green);
  B = QS * decode_pixel_gamma(blue);
  l = cbrt(0.4122214708 * R + 0.5363325363 * G + 0.0514459929 * B);
  m = cbrt(0.2119034982 * R + 0.6806995451 * G + 0.1073969566 * B);
  s = cbrt(0.0883024619 * R + 0.2817188376 * G + 0.6299787005 * B);
  *L = 0.2104542553 * l + 0.7936177850 * m - 0.0040720468 * s;
  *a = 1.9779984951 * l - 2.4285922050 * m + 0.4505937099 * s + 0.5;
  *b = 0.0259040371 * l + 0.7827717662 * m - 0.8086757660 * s + 0.5;
}
static void oklab_to_rgb(double L, double a, double b, double *red, double *green, double *blue)
{
  double B, G, l, m, R, s;
  l = L + 0.3963377774 * (a - 0.5) + 0.2158037573 * (b - 0.5);
  m = L - 0.1055613458 * (a - 0.5) - 0.0638541728 * (b - 0.5);
  s = L - 0.0894841775 * (a - 0.5) - 1.2914855480 * (b - 0.5);
  l *= l * l;
  m *= m * m;
  s *= s * s;
  R = 4.0767416621 * l - 3.3077115913 * m + 0.2309699292 * s;
  G = (-1.2684380046) * l + 2.6097574011 * m - 0.3413193965 * s;
  B = (-0.0041960863) * l - 0.7034186147 * m + 1.7076147010 * s;
  *red = encode_pixel_gamma(QR * R);
  *green = encode_pixel_gamma(QR * G);
  *blue = encode_pixel_gamma(QR * B);
}
/* Jzazbz (colorspace-private.h:1274-1478; white_luminance = 10000 unless the "white-luminance" property says otherwise,
   colorspace.c:995-998).  Quirks kept: RGB -> XYZ is called with green and blue swapped, and so is XYZ -> RGB. */
#define JZ_B 1.15
#define JZ_G 0.66
#define JZ_C1 (3424.0 / 4096.0)
#define JZ_C2 (2413.0 / 128.0)
#define JZ_C3 (2392.0 / 128.0)
#define JZ_N (2610.0 / 16384.0)
#define JZ_P (1.7 * 2523.0 / 32.0)
#define JZ_D (-0.56)
#define JZ_D0 1.6295499532821566e-11
static void xyz_to_jzazbz(double X, double Y, double Z, double white_luminance, double *Jz, double *az, double *bz)
{
  double a, b, dL, dM, dS, gL, gM, gS, nL, nM, nS, Iz, J, JdI, L, Lp, M, Mp, S, Sp, WLr, Xp, Yp;
  WLr = precip(white_luminance);
  Xp = Z + JZ_B * (X - Z);
  Yp = X + JZ_G * (Y - X);
  L = 0.0146480 * Z; M = 0.0531008 * Z; S = 0.6684799 * Z;
  L += 0.41478972 * Xp; M += (-0.2015100) * Xp; S += (-0.0166008) * Xp;
  L += 0.579999 * Yp; M += 1.120649 * Yp; S += 0.264800 * Yp;
  gL = pow(L * WLr, JZ_N); gM = pow(M * WLr, JZ_N); gS = pow(S * WLr, JZ_N);
  nL = JZ_C1 + JZ_C2 * gL; nM = JZ_C1 + JZ_C2 * gM; nS = JZ_C1 + JZ_C2 * gS;
  dL = 1.0 + JZ_C3 * gL; dM = 1.0 + JZ_C3 * gM; dS = 1.0 + JZ_C3 * gS;
  Lp = pow(nL / dL, JZ_P); Mp = pow(nM / dM, JZ_P); Sp = pow(nS / dS, JZ_P);
  Iz = (Lp + Mp) * 0.5;
  JdI = JZ_D * Iz;
  J = (JdI + Iz) / (JdI + 1.0) - JZ_D0;
  a = 0.5 + 3.52400 * Lp; b = 0.5 + 0.199076 * Lp;
  a += (-4.066708) * Mp; b += 1.096799 * Mp;
  a += 0.542708 * Sp; b += (-1.295875) * Sp;
  *Jz = isnan(J) ? 0.0 : J;
  *az = isnan(a) ? 0.5 : a;
  *bz = isnan(b) ? 0.5 : b;
}
static void jzazbz_to_xyz(double Jz, double az, double bz, double white_luminance, double *X, double *Y, double *Z)
{
  double azz, bzz, C, dL, dM, dS, g, gL, gM, gS, Jnr, Jpr, L, Lp, M, Mp, S, Sp, nL, nM, nS, Xp, Zp, Yp;
  g = Jz + JZ_D0;
  azz = az - 0.5; bzz = bz - 0.5;
  C = 0.138605043271539 * azz + 0.0580473161561189 * bzz;
  Sp = g / (1.0 + JZ_D * (1.0 - g));
  Lp = Sp + C; Mp = Sp - C;
  Sp += (-0.0960192420263189) * azz;
  Sp += (-0.811891896056039) * bzz;
  Jpr = 1.0 / JZ_P;
  gL = pow(Lp, Jpr); gM = pow(Mp, Jpr); gS = pow(Sp, Jpr);
  Jnr = 1.0 / JZ_N;
  nL = gL - JZ_C1; nM = gM - JZ_C1; nS = gS - JZ_C1;
  dL = JZ_C2 + (-2392.0 / 128.0) * gL; dM = JZ_C2 + (-2392.0 / 128.0) * gM; dS = JZ_C2 + (-2392.0 / 128.0) * gS;
  L = pow(nL / dL, Jnr); M = pow(nM / dM, Jnr); S = pow(nS / dS, Jnr);
  L *= white_luminance; M *= white_luminance; S *= white_luminance;
  Zp = (-0.0909828109828476) * L; Xp = 1.92422643578761 * L; Yp = 0.350316762094999 * L;
  Zp += (-0.312728290523074) * M; Xp += (-1.00479231259537) * M; Yp += 0.726481193931655 * M;
  Zp += 1.52276656130526 * S; Xp += 0.037651404030618 * S; Yp += (-0.065384422948085) * S;
  Zp = isnan(Zp) ? 0.0 : Zp;
  Xp = Zp + (Xp - Zp) / JZ_B;
  Xp = isnan(Xp) ? 0.0 : Xp;
  Yp = Xp + (Yp - Xp) / JZ_G;
  Yp = isnan(Yp) ? 0.0 : Yp;
  *Z = Zp; *X = Xp; *Y = Yp;
}
static double degrees_to_radians(double degrees) { return (double) (PI_ * degrees / 180.0); }   /* image-private.h:142 */

static int is_xyz_family_space(int cs)
{
  if (cs == ORC_CS_OKLAB || cs == ORC_CS_OKLCH || cs == ORC_CS_LCH || cs == ORC_CS_LCHAB || cs == ORC_CS_LCHUV ||
      cs == ORC_CS_JZAZBZ) return 1;
  return cs == ORC_CS_ADOBE98 || cs == ORC_CS_DISPLAYP3 || cs == ORC_CS_PROPHOTO || cs == ORC_CS_LMS ||
         cs == ORC_CS_CAT02LMS || cs == ORC_CS_XYY || cs == ORC_CS_LUV;
}

static int colorspace_xyz_family_leg(float *buf, long n, int ch, int cs, int forward)
{
  long i;
  if (!is_xyz_family_space(cs)) return -1;
#pragma omp parallel for schedule(static)
  for (i = 0; i < n; i++) {
    float *q = buf + (size_t) i * ch;
    double X, Y, Z, a, b, c;
    if (cs == ORC_CS_JZAZBZ) {                               /* :1365-1376, :1467-1478: note the swapped arguments */
      if (forward) {
        rgb_to_xyz((double) q[0], (double) q[2], (double) q[1], &X, &Y, &Z);
        xyz_to_jzazbz(X, Y, Z, cs_white_luminance, &a, &b, &c);
        q[0] = (float) (QR * a); q[1] = (float) (QR * b); q[2] = (float) (QR * c);
      } else {
        double R, G, B;
        jzazbz_to_xyz(QS * q[0], QS * q[1], QS * q[2], cs_white_luminance, &X, &Y, &Z);
        xyz_to_rgb(X, Y, Z, &R, &B, &G);
        q[0] = (float) R; q[1] = (float) G; q[2] = (float) B;
      }
      continue;
    }
    if (cs == ORC_CS_OKLAB || cs == ORC_CS_OKLCH) {          /* not routed through XYZ */
      if (forward) {
        rgb_to_oklab((double) q[0], (double) q[1], (double) q[2], &a, &b, &c);
        if (cs == ORC_CS_OKLCH) {                            /* :1539-1549 */
          const double C = sqrt(b * b + c * c), h = 0.5 + 0.5 * atan2(-c, -b) / PI_;
          b = C; c = h;
        }
        q[0] = (float) (QR * a); q[1] = (float) (QR * b); q[2] = (float) (QR * c);
      } else {
        double R, G, B;
        a = QS * q[0]; b = QS * q[1]; c = QS * q[2];
        if (cs == ORC_CS_OKLCH) {                            /* :1527-1537 */
          const double ca = b * cos(2.0 * PI_ * c), cb = b * sin(2.0 * PI_ * c);
          b = ca; c = cb;
        }
        oklab_to_rgb(a, b, c, &R, &G, &B);
        q[0] = (float) R; q[1] = (float) G; q[2] = (float) B;
      }
      continue;
    }
    if (forward) {                       /* ConvertRGBToGeneric :411 -> (float) (QR * component) */
      rgb_to_xyz((double) q[0], (double) q[1], (double) q[2], &X, &Y, &Z);
      switch (cs) {
        case ORC_CS_LCH: case ORC_CS_LCHAB: {                /* :1104-1117: polar Lab */
          double L, la, lb;
          xyz_to_lab(X, Y, Z, &L, &la, &lb);
          a = L;
          b = hypot(la - 0.5, lb - 0.5) / 1.0 + 0.5;
          c = 180.0 * atan2(lb - 0.5, la - 0.5) / PI_ / 360.0;
          if (c < 0.0) c += 1.0;
          break;
        }
        case ORC_CS_LCHUV: {                                 /* :1163-1176: polar Luv */
          double L, u, v;
          xyz_to_luv(X, Y, Z, &L, &u, &v);
          a = L;
          b = hypot(354.0 * u - 134.0, 262.0 * v - 140.0) / 255.0 + 0.5;
          c = 180.0 * atan2(262.0 * v - 140.0, 354.0 * u - 134.0) / PI_ / 360.0;
          if (c < 0.0) c += 1.0;
          break;
        }
        case ORC_CS_ADOBE98: case ORC_CS_DISPLAYP3: case ORC_CS_PROPHOTO: {
          const mat3 *m = cs == ORC_CS_ADOBE98 ? &xyz_to_adobe98 : cs == ORC_CS_DISPLAYP3 ? &xyz_to_displayp3 : &xyz_to_prophoto;
          a = QS * encode_pixel_gamma(QR * row3(m->m[0], X, Y, Z));
          b = QS * encode_pixel_gamma(QR * row3(m->m[1], X, Y, Z));
          c = QS * encode_pixel_gamma(QR * row3(m->m[2], X, Y, Z));
          break;
        }
        case ORC_CS_LMS: xyz_to_lms(X, Y, Z, &a, &b, &c); break;
        case ORC_CS_CAT02LMS: { double L, M, S; xyz_to_lms(X, Y, Z, &L, &M, &S); lms_to_xyz(L, M, S, &a, &b, &c); break; }  /* :424-433 */
        case ORC_CS_XYY: { const double gamma = precip(X + Y + Z); a = gamma * X; b = gamma * Y; c = Y; break; }      /* :1258-1272 */
        default: xyz_to_luv(X, Y, Z, &a, &b, &c); break;
      }
      q[0] = (float) (QR * a); q[1] = (float) (QR * b); q[2] = (float) (QR * c);
    } else {                             /* ConvertGenericToRGB :122 on QuantumScale * sample */
      double R, G, B;
      a = QS * q[0]; b = QS * q[1]; c = QS * q[2];
      switch (cs) {
        case ORC_CS_ADOBE98: case ORC_CS_DISPLAYP3: case ORC_CS_PROPHOTO: {
          const mat3 *m = cs == ORC_CS_ADOBE98 ? &adobe98_to_xyz : cs == ORC_CS_DISPLAYP3 ? &displayp3_to_xyz : &prophoto_to_xyz;
          const double r = QS * decode_pixel_gamma(QR * a), g = QS * decode_pixel_gamma(QR * b), bl = QS * decode_pixel_gamma(QR * c);
          X = row3(m->m[0], r, g, bl); Y = row3(m->m[1], r, g, bl); Z = row3(m->m[2], r, g, bl);
          break;
        }
        case ORC_CS_LCH: case ORC_CS_LCHAB: {                /* :572-598 */
          const double luma = 100.0 * a, chroma = 255.0 * (b - 0.5), hue = 360.0 * c;
          lab_to_xyz(luma, chroma * cos(degrees_to_radians(hue)), chroma * sin(degrees_to_radians(hue)), &X, &Y, &Z);
          break;
        }
        case ORC_CS_LCHUV: {                                 /* :627-653 */
          const double luma = 100.0 * a, chroma = 255.0 * (b - 0.5), hue = 360.0 * c;
          luv_to_xyz(luma, chroma * cos(degrees_to_radians(hue)), chroma * sin(degrees_to_radians(hue)), &X, &Y, &Z);
          break;
        }
        case ORC_CS_LMS: lms_to_xyz(a, b, c, &X, &Y, &Z); break;
        case ORC_CS_CAT02LMS: { double L, M, S; xyz_to_lms(a, b, c, &L, &M, &S); lms_to_xyz(L, M, S, &X, &Y, &Z); break; }  /* :135-143 */
        case ORC_CS_XYY: { const double gamma = precip(b); X = gamma * c * a; Y = c; Z = gamma * c * (1.0 - a - b); break; }  /* :1676-1690 */
        default: luv_to_xyz(100.0 * a, 354.0 * b - 134.0, 262.0 * c - 140.0, &X, &Y, &Z); break;                        /* :706-717 */
      }
      xyz_to_rgb(X, Y, Z, &R, &G, &B);
      q[0] = (float) R; q[1] = (float) G; q[2] = (float) B;
    }
  }
  return 0;
}

/* ---- Log (colorspace.c:1055-1163 forward, :2391-2500 inverse): a 65536-entry table of Quantum values indexed by
   ScaleQuantumToMap of the linearised (forward) or stored (inverse) sample.  DisplayGamma = 1/1.7 is both the density and
   the default gamma (the "gamma" property lookup of :1081 never succeeds: SetImageProperty diverts that key to image->gamma,
   property.c:4583). */
typedef struct { double gamma, film_gamma, reference_black, reference_white; } log_settings;
static log_settings cs_log = {1.0 / 1.7, 0.6, 95.0, 685.0};

static void log_forward_table(float *logmap)
{
  const double density = 1.0 / 1.7;
  const double black = pow(10.0, (cs_log.reference_black - cs_log.reference_white) * (cs_log.gamma / density) * 0.002 *
                                     precip(cs_log.film_gamma));
  long i;
  for (i = 0; i <= 65535; i++)
    logmap[i] = scale_map_to_quantum(((double) 65535.0 * (cs_log.reference_white +
                  log10(black + (1.0 * (double) i / 65535.0) * (1.0 - black)) / ((cs_log.gamma / density) * 0.002 *
                  precip(cs_log.film_gamma))) / 1024.0));
}

static void log_inverse_table(float *logmap)
{
  const double density = 1.0 / 1.7;
  const double black = pow(10.0, (cs_log.reference_black - cs_log.reference_white) * (cs_log.gamma / density) * 0.002 *
                                     precip(cs_log.film_gamma));
  long i;
  for (i = 0; i <= 65535 && i <= (long) (cs_log.reference_black * 65535.0 / 1024.0); i++) logmap[i] = 0.0f;
  for (; i <= 65535 && i < (long) (cs_log.reference_white * 65535.0 / 1024.0); i++)
    logmap[i] = (float) ((double) QR / (1.0 - black) * (pow(10.0, (1024.0 * (double) i / 65535.0 - cs_log.reference_white) *
                  (cs_log.gamma / density) * 0.002 * precip(cs_log.film_gamma)) - black));
  for (; i <= 65535; i++) logmap[i] = (float) QR;
}

static int colorspace_log_leg(float *buf, long n, int ch, int forward)
{
  long i;
  float *logmap = (float *) malloc(65536 * sizeof(float));
  if (!logmap) return -1;
  if (forward) log_forward_table(logmap); else log_inverse_table(logmap);
#pragma omp parallel for schedule(static)
  for (i = 0; i < n; i++) {
    float *q = buf + (size_t) i * ch;
    int k;
    for (k = 0; k < 3; k++) {
      if (forward) q[k] = logmap[scale_quantum_to_map((float) decode_pixel_gamma((double) q[k]))];
      else q[k] = (float) encode_pixel_gamma((double) logmap[scale_quantum_to_map(q[k])]);
    }
  }
  free(logmap);
  return 0;
}

/* ---- YCC (PhotoYCC; colorspace.c:1347-1389 forward, :2681-2711 and :2788-2796 inverse) in the LUT branch: the forward
   tables are piecewise (linear toe up to 0.018 * MaxMap, then the 1.099 * i - 0.099 curve), offsets 156 and 137 on the
   8-bit scale; the inverse ends in a 1389-entry table of floats that is the sequence "%.6f" of (float) i / 1388 -- the
   values are regenerated from that rule and compared with the compiled reference by tests/test_oracle_vs_ref.py. */
#define YCC_C1_ZERO 40092.0      /* ScaleQuantumToMap(ScaleCharToQuantum(156)) = 156 * 257 */
#define YCC_C2_ZERO 35209.0      /* 137 * 257 */
static void ycc_map(float *table)
{
  int i;
  char text[32];
  for (i = 0; i < 1389; i++) {
    snprintf(text, sizeof(text), "%.6f", (double) ((float) i / 1388.0f));
    table[i] = strtof(text, NULL);
  }
}

static int colorspace_ycc_leg(float *buf, long n, int ch, int forward)
{
  static const double toe[3][3] = {{0.005382, -0.003296, 0.009410}, {0.010566, -0.006471, -0.007880}, {0.002052, 0.009768, -0.001530}};
  static const double curve[3][3] = {{0.298839, -0.298839, 0.70100}, {0.586811, -0.586811, -0.586811}, {0.114350, 0.88600, -0.114350}};
  float ycc[1389];
  long i;
  ycc_map(ycc);
#pragma omp parallel for schedule(static)
  for (i = 0; i < n; i++) {
    float *q = buf + (size_t) i * ch;
    const unsigned int idx[3] = {scale_quantum_to_map(q[0]), scale_quantum_to_map(q[1]), scale_quantum_to_map(q[2])};
    double v[3];
    int k, c;
    if (forward) {
      for (k = 0; k < 3; k++) {           /* k: output component (.x, .y, .z); c: input channel (x_map, y_map, z_map) */
        double e[3];
        for (c = 0; c < 3; c++) {
          const double di = (double) idx[c];
          e[c] = idx[c] <= 1179u ? toe[c][k] * di : curve[c][k] * (1.099 * di - 0.099);     /* (ssize_t) (0.018 * MaxMap) = 1179 */
        }
        v[k] = ((e[0] + e[1]) + e[2]) + (k == 0 ? 0.0 : k == 1 ? YCC_C1_ZERO : YCC_C2_ZERO);
        v[k] = (double) scale_map_to_quantum(v[k]);
      }
    } else {
      const double r = (double) idx[0], g = (double) idx[1], b = (double) idx[2];
      v[0] = (1.3584000 * r + 0.0000000) + 1.8215000 * (1.0 * b - YCC_C2_ZERO);
      v[1] = (1.3584000 * r + (-0.4302726) * (1.0 * g - YCC_C1_ZERO)) + (-0.9271435) * (1.0 * b - YCC_C2_ZERO);
      v[2] = (1.3584000 * r + 2.2179000 * (1.0 * g - YCC_C1_ZERO)) + 0.0000000;
      for (k = 0; k < 3; k++) {
        const double t = 1024.0 * v[k] / 65535.0;
        const long at = t <= 0.0 ? 0 : t >= 1388.0 ? 1388 : (long) (t + 0.5);               /* RoundToYCC :1814 */
        v[k] = (double) QR * (double) ycc[at];
      }
    }
    q[0] = (float) v[0]; q[1] = (float) v[1]; q[2] = (float) v[2];
  }
  return 0;
}

/* colorspace.c:1751-1783 TransformImageColorspace: anything that is not sRGB goes back to sRGB
   first (TransformsRGBImage), then forward (sRGBTransformImage). */
static int colorspace_leg(float *buf, size_t w, size_t h, int ch, int cs, int forward)
{
  const long n = (long) (w * h);
  if (cs == ORC_CS_LOG) return colorspace_log_leg(buf, n, ch, forward);
  if (cs == ORC_CS_YCC) return colorspace_ycc_leg(buf, n, ch, forward);
  if (is_hexcone_space(cs)) return colorspace_hexcone_leg(buf, n, ch, cs, forward);
  if (is_xyz_family_space(cs)) return colorspace_xyz_family_leg(buf, n, ch, cs, forward);
  if (is_core_space(cs)) return forward ? colorspace_core(buf, w, h, ch, ORC_CS_SRGB, cs) : colorspace_core(buf, w, h, ch, cs, ORC_CS_SRGB);
  return colorspace_matrix_leg(buf, n, ch, cs, forward);
}

int orc_colorspace_ex(float *buf, size_t w, size_t h, int ch, int from, int to, const orc_colorspace_options *o)
{
  int rc = 0;
  if (ch < 3) return -1;
  if (from == to) return 0;
  {
    const int ill = (o && (o->set & ORC_CO_ILLUMINANT) && o->illuminant >= 0 && o->illuminant <= 10) ? o->illuminant : 5;
    cs_ill[0] = illuminant_table[ill][0]; cs_ill[1] = illuminant_table[ill][1]; cs_ill[2] = illuminant_table[ill][2];
    cs_white_luminance = (o && (o->set & ORC_CO_WHITE_LUMINANCE)) ? o->white_luminance : 10000.0;
    cs_log.gamma = 1.0 / 1.7;
    cs_log.film_gamma = (o && (o->set & ORC_CO_FILM_GAMMA)) ? o->film_gamma : 0.6;
    cs_log.reference_black = (o && (o->set & ORC_CO_REFERENCE_BLACK)) ? o->reference_black : 95.0;
    cs_log.reference_white = (o && (o->set & ORC_CO_REFERENCE_WHITE)) ? o->reference_white : 685.0;
  }
  if (is_core_space(from) && is_core_space(to)) rc = colorspace_core(buf, w, h, ch, from, to);
  else {
    if (from != ORC_CS_SRGB) rc = colorspace_leg(buf, w, h, ch, from, 0);
    if (rc == 0 && to != ORC_CS_SRGB) rc = colorspace_leg(buf, w, h, ch, to, 1);
  }
  cs_ill[0] = illuminant_table[5][0]; cs_ill[1] = illuminant_table[5][1]; cs_ill[2] = illuminant_table[5][2];
  cs_white_luminance = 10000.0;
  return rc;
}

int orc_colorspace(float *buf, size_t w, size_t h, int ch, int from, int to)
{
  return orc_colorspace_ex(buf, w, h, ch, from, to, NULL);
}

/* the two tables on their own (pinned to the reference through the images above) */
void orc_log_table(int forward, const orc_colorspace_options *o, float *table)
{
  cs_log.gamma = 1.0 / 1.7;
  cs_log.film_gamma = (o && (o->set & ORC_CO_FILM_GAMMA)) ? o->film_gamma : 0.6;
  cs_log.reference_black = (o && (o->set & ORC_CO_REFERENCE_BLACK)) ? o->reference_black : 95.0;
  cs_log.reference_white = (o && (o->set & ORC_CO_REFERENCE_WHITE)) ? o->reference_white : 685.0;
  if (forward) log_forward_table(table); else log_inverse_table(table);
}

void orc_ycc_table(float *table) { ycc_map(table); }

/* ------------------------------------------------------------------------------------------
   threshold.c point operators (in place).
   BilevelImage :805-897, BlackThresholdImage :927-1053, WhiteThresholdImage :2518-2644,
   ClampImage :1087-1190; GetPixelIntensity pixel.c:2356-2451 with the default
   (Rec709Luma) method on an sRGB / gray image: 0.212656*R+0.715158*G+0.072186*B evaluated
   left to right in double (no contraction); one-channel images return the gray value itself
   (:2366); for Gray+Alpha the green/blue accessors resolve to the gray sample (channel map
   offsets default to 0), so the same expression is evaluated on (g,g,g).
   image->channel_mask == AllChannels, so every channel (alpha included: it carries the Update
   trait, pixel.c:6370) is compared through the pixel's INTENSITY, against its own threshold.
   op: 0 bilevel (thr[0]); 1 black, 2 white (thr = red, green, blue, alpha as left by the
   ParseGeometry step :955-985); 3 clamp (pixel-accessor.h:35-46, HDRI: no rounding).
   ------------------------------------------------------------------------------------------ */
static double pixel_intensity(const float *q, int ch)
{
  double red = (double) q[0], green, blue;
  if (ch == 1) return red;
  green = ch >= 3 ? (double) q[1] : red;
  blue = ch >= 3 ? (double) q[2] : red;
  return 0.212656 * red + 0.715158 * green + 0.072186 * blue;
}

int orc_threshold(float *buf, size_t w, size_t h, int ch, int op, const double *thr)
{
  long i, n = (long) (w * h);
  if (ch < 1 || ch > 4 || op < 0 || op > 3) return -1;
  if ((op == 1 || op == 2) && ch < 3) return -1;   /* gray images are promoted to sRGB there (:949) */
#pragma omp parallel for schedule(static)
  for (i = 0; i < n; i++) {
    float *q = buf + (size_t) i * ch;
    int c;
    if (op == 3) {
      for (c = 0; c < ch; c++) {
        double pixel = (double) q[c];
        if (pixel < 0.0) q[c] = 0.0f;
        else if (pixel >= QR) q[c] = (float) QR;
        else q[c] = (float) pixel;
      }
      continue;
    }
    {
      const double pixel = pixel_intensity(q, ch);
      for (c = 0; c < ch; c++) {
        const int is_alpha = (ch == 2 || ch == 4) && c == ch - 1;
        const double t = op == 0 ? thr[0] : (is_alpha ? thr[3] : thr[c]);
        if (op == 0) q[c] = (float) (pixel <= t ? 0.0 : QR);
        else if (op == 1) { if (pixel < t) q[c] = 0.0f; }
        else { if (pixel > t) q[c] = (float) QR; }
      }
    }
  }
  return 0;
}


/* effect.c:3991-4063 SharpenImage, :1520-1570 EdgeImage: inline kernel + ConvolveImage */
int orc_sharpen(const float *src, float *dst, size_t w, size_t h, int ch, double radius, double sigma)
{
  const size_t width = orc_optimal_kernel_width_2d(radius, sigma);
  const double s = fabs(sigma) < EPS ? EPS : sigma;                 /* MagickSigma */
  double *vals = (double *) malloc(width * width * sizeof(double)), normalize = 0.0, gamma;
  const long j = (long) (width - 1) / 2;
  long u, v;
  size_t i = 0;
  orc_kernel k;
  int rc;
  if (!vals) return -1;
  for (v = -j; v <= j; v++)
    for (u = -j; u <= j; u++) {
      vals[i] = -exp(-((double) u * u + v * v) / (2.0 * s * s)) / (2.0 * PI_ * s * s);
      normalize += vals[i];
      i++;
    }
  vals[i / 2] = (-2.0) * normalize;
  normalize = 0.0;
  for (i = 0; i < width * width; i++) normalize += vals[i];
  gamma = perceptible_reciprocal(normalize);
  for (i = 0; i < width * width; i++) vals[i] *= gamma;
  rc = orc_kernel_user(width, width, j, j, vals, &k);
  free(vals);
  if (rc) return rc;
  rc = orc_morphology_apply(src, dst, w, h, ch, ORC_CONVOLVE, 1, &k, 1, 0.0);
  orc_kernel_free(&k);
  return rc;
}

int orc_edge(const float *src, float *dst, size_t w, size_t h, int ch, double radius)
{
  const size_t width = orc_optimal_kernel_width_1d(radius, 0.5), n = width * width;
  double *vals = (double *) malloc(n * sizeof(double));
  orc_kernel k;
  size_t i;
  int rc;
  if (!vals) return -1;
  for (i = 0; i < n; i++) vals[i] = -1.0;
  vals[n / 2] = (double) width * width - 1.0;
  rc = orc_kernel_user(width, width, (long) (width - 1) / 2, (long) (width - 1) / 2, vals, &k);
  free(vals);
  if (rc) return rc;
  rc = orc_morphology_apply(src, dst, w, h, ch, ORC_CONVOLVE, 1, &k, 1, 0.0);
  orc_kernel_free(&k);
  return rc;
}

/* enhance.c:2040-2290 EqualizeImage, Q16-HDRI (MaxMap 65535), default traits.  sync != 0: the channel mask carries
   SyncChannels (AllChannels, the default mask, does: pixel.h:62,74): every channel's histogram is indexed by the pixel
   INTENSITY (:2125-2129); 0: by the channel's own value.  ScaleQuantumToMap / ScaleMapToQuantum: quantum-private.h:504, :464. */
int orc_equalize(float *buf, size_t w, size_t h, int ch, int sync)
{
  const size_t n = w * h, bins = 65536;
  double *histogram, *map, *equalize_map, black[4], white[4];
  size_t i, j;
  int c;
  if (ch < 1 || ch > 4) return -1;
  histogram = (double *) calloc(bins * (size_t) ch, sizeof(double));
  map = (double *) malloc(bins * (size_t) ch * sizeof(double));
  equalize_map = (double *) calloc(bins * (size_t) ch, sizeof(double));
  if (!histogram || !map || !equalize_map) { free(histogram); free(map); free(equalize_map); return -1; }
  for (i = 0; i < n; i++) {
    const float *p = buf + i * (size_t) ch;
    for (c = 0; c < ch; c++) {
      double intensity = (double) p[c];
      if (sync) intensity = pixel_intensity(p, ch);
      histogram[(size_t) ch * scale_quantum_to_map((float) intensity) + (size_t) c]++;     /* ClampToQuantum: the float cast */
    }
  }
  for (c = 0; c < ch; c++) {
    double intensity = 0.0;
    for (j = 0; j < bins; j++) {
      intensity += histogram[(size_t) ch * j + (size_t) c];
      map[(size_t) ch * j + (size_t) c] = intensity;
    }
  }
  for (c = 0; c < ch; c++) {
    black[c] = map[c];
    white[c] = map[(size_t) ch * (bins - 1) + (size_t) c];
    if (black[c] != white[c])
      for (j = 0; j < bins; j++) {
        const double value = (65535.0 * (map[(size_t) ch * j + (size_t) c] - black[c])) / (white[c] - black[c]);
        equalize_map[(size_t) ch * j + (size_t) c] =
            (double) (value <= 0.0 ? 0.0f : value >= 65535.0 ? 65535.0f : (float) value);      /* ScaleMapToQuantum */
      }
  }
  for (i = 0; i < n; i++) {
    float *q = buf + i * (size_t) ch;
    for (c = 0; c < ch; c++) {
      if (black[c] == white[c]) continue;
      q[c] = (float) equalize_map[(size_t) ch * scale_quantum_to_map(q[c]) + (size_t) c];
    }
  }
  free(histogram); free(map); free(equalize_map);
  return 0;
}

/* effect.c:1600-1681 EmbossImage: anti-diagonal kernel (:1649-1665) + ConvolveImage + EqualizeImage */
int orc_emboss_kernel(double radius, double sigma, orc_kernel *out)
{
  const size_t width = orc_optimal_kernel_width_1d(radius, sigma);
  const double s = fabs(sigma) < EPS ? EPS : sigma;                 /* MagickSigma */
  double *vals = (double *) malloc(width * width * sizeof(double)), normalize = 0.0, gamma;
  const long j = (long) (width - 1) / 2;
  long u, v, k = j;
  size_t i = 0;
  int rc;
  if (!vals) return -1;
  for (v = -j; v <= j; v++) {
    for (u = -j; u <= j; u++) {
      vals[i] = ((u < 0) || (v < 0) ? -8.0 : 8.0) * exp(-((double) u * u + v * v) / (2.0 * s * s)) / (2.0 * PI_ * s * s);
      if (u != k) vals[i] = 0.0;
      i++;
    }
    k--;
  }
  for (i = 0; i < width * width; i++) normalize += vals[i];
  gamma = perceptible_reciprocal(normalize);
  for (i = 0; i < width * width; i++) vals[i] *= gamma;
  rc = orc_kernel_user(width, width, j, j, vals, out);
  free(vals);
  return rc;
}

int orc_emboss(const float *src, float *dst, size_t w, size_t h, int ch, double radius, double sigma)
{
  orc_kernel k;
  int rc = orc_emboss_kernel(radius, sigma, &k);
  if (rc) return rc;
  rc = orc_morphology_apply(src, dst, w, h, ch, ORC_CONVOLVE, 1, &k, 1, 0.0);
  orc_kernel_free(&k);
  if (rc) return rc;
  return orc_equalize(dst, w, h, ch, 1);
}

/* ------------------------------------------------------------------------------------------
   resize.c:4106-4530 ScaleImage: box scaling as a sequential state machine -- rows are accumulated into y_vector with
   the running (span.y, scale.y) pair, each finished scanline is then accumulated along x with (span.x, scale.x); colour
   channels of images with alpha are premultiplied by QS*alpha on the way in (:4199-4215) and divided by the scaled alpha
   on the way out (:4482-4503).  Restated literally (same state updates, same multiply-then-add order).
   ------------------------------------------------------------------------------------------ */
int orc_scale(const float *src, size_t w, size_t h, int ch, float *dst, size_t ow, size_t oh)
{
  const int has_alpha = (ch == 2 || ch == 4);
  const size_t n = w * (size_t) ch, on = ow * (size_t) ch;
  double *x_vector, *y_vector, *scanline, *scale_scanline, pixel[4];
  double span_x, span_y = 1.0, scale_x, scale_y;
  long number_rows = 0, row = 0, y;
  int next_row = 1, next_column, c;
  if (ow == 0 || oh == 0 || ch < 1 || ch > 4) return -1;
  if (ow == w && oh == h) { memcpy(dst, src, n * h * sizeof(float)); return 0; }
  x_vector = (double *) malloc(n * sizeof(double));
  y_vector = (double *) calloc(n, sizeof(double));
  scanline = (h != oh) ? (double *) malloc(n * sizeof(double)) : x_vector;
  scale_scanline = (double *) malloc((on > n ? on : n) * sizeof(double) + 4 * sizeof(double));
  if (!x_vector || !y_vector || !scanline || !scale_scanline) return -1;
  scale_y = (double) oh / (double) h;
#define ORC_READ_ROW() do { const float *p = src + (size_t) row * n; size_t x_; double alpha_ = 1.0; row++; \
    for (x_ = 0; x_ < w; x_++, p += ch) { if (has_alpha) alpha_ = QS * (double) p[ch - 1]; \
      for (c = 0; c < ch; c++) x_vector[x_ * ch + c] = (has_alpha && c != ch - 1) ? alpha_ * (double) p[c] : (double) p[c]; } } while (0)
  for (y = 0; y < (long) oh; y++) {
    float *q = dst + (size_t) y * on;
    size_t x;
    if (oh == h) {
      ORC_READ_ROW();
    } else {
      while (scale_y < span_y) {
        if (next_row && number_rows < (long) h) { ORC_READ_ROW(); number_rows++; }
        for (x = 0; x < n; x++) y_vector[x] += scale_y * x_vector[x];
        span_y -= scale_y;
        scale_y = (double) oh / (double) h;
        next_row = 1;
      }
      if (next_row && number_rows < (long) h) { ORC_READ_ROW(); number_rows++; next_row = 0; }
      for (x = 0; x < n; x++) { scanline[x] = y_vector[x] + span_y * x_vector[x]; y_vector[x] = 0.0; }
      scale_y -= span_y;
      if (scale_y <= 0) { scale_y = (double) oh / (double) h; next_row = 1; }
      span_y = 1.0;
    }
    if (ow == w) {
      for (x = 0; x < ow; x++, q += ch) {
        double alpha = 1.0;
        if (has_alpha) alpha = perceptible_reciprocal(QS * scanline[x * ch + ch - 1]);
        for (c = 0; c < ch; c++)
          q[c] = (float) ((has_alpha && c != ch - 1) ? alpha * scanline[x * ch + c] : scanline[x * ch + c]);
      }
      continue;
    }
    {
      long t = 0;
      for (c = 0; c < ch; c++) pixel[c] = 0.0;
      next_column = 0;
      span_x = 1.0;
      for (x = 0; x < w; x++) {
        scale_x = (double) ow / (double) w;
        while (scale_x >= span_x) {
          if (next_column) { for (c = 0; c < ch; c++) pixel[c] = 0.0; t++; }
          for (c = 0; c < ch; c++) { pixel[c] += span_x * scanline[x * ch + c]; if (t < (long) ow) scale_scanline[t * ch + c] = pixel[c]; }
          scale_x -= span_x;
          span_x = 1.0;
          next_column = 1;
        }
        if (scale_x > 0) {
          if (next_column) { for (c = 0; c < ch; c++) pixel[c] = 0.0; next_column = 0; t++; }
          for (c = 0; c < ch; c++) pixel[c] += scale_x * scanline[x * ch + c];
          span_x -= scale_x;
        }
      }
      if (span_x > 0) for (c = 0; c < ch; c++) pixel[c] += span_x * scanline[(x - 1) * ch + c];
      if (!next_column && t < (long) ow) for (c = 0; c < ch; c++) scale_scanline[t * ch + c] = pixel[c];
      for (x = 0; x < ow; x++, q += ch) {
        double alpha = 1.0;
        if (has_alpha) alpha = perceptible_reciprocal(QS * scale_scanline[x * ch + ch - 1]);
        for (c = 0; c < ch; c++)
          q[c] = (float) ((has_alpha && c != ch - 1) ? alpha * scale_scanline[x * ch + c] : scale_scanline[x * ch + c]);
      }
    }
  }
#undef ORC_READ_ROW
  if (scanline != x_vector) free(scanline);
  free(x_vector); free(y_vector); free(scale_scanline);
  return 0;
}

/* resize.c:3907-4090 SampleImage (default sample:offset = 0.5 - MagickEpsilon) */
int orc_sample(const float *src, size_t w, size_t h, int ch, float *dst, size_t ow, size_t oh)
{
  const double off = 0.5 - EPS;
  long y;
  if (ow == 0 || oh == 0 || ch < 1 || ch > 4) return -1;
#pragma omp parallel for schedule(static)
  for (y = 0; y < (long) oh; y++) {
    const long yo = (long) ((((double) y + off) * (double) h) / (double) oh);
    size_t x;
    for (x = 0; x < ow; x++) {
      const long xo = (long) ((((double) x + off) * (double) w) / (double) ow);
      memcpy(dst + ((size_t) y * ow + x) * ch, src + ((size_t) yo * w + (size_t) xo) * ch, (size_t) ch * sizeof(float));
    }
  }
  return 0;
}


/* resize.c:4591-4650 ThumbnailImage, pixel path (image->filter undefined => LanczosSharp) */
int orc_thumbnail(const float *src, size_t w, size_t h, int ch, float *dst, size_t columns, size_t rows)
{
  const long xf = (long) w / (long) columns, yf = (long) h / (long) rows;
  const float *cur = src;
  float *a = NULL, *b = NULL;
  size_t cw = w, chh = h;
  int rc = 0;
  if (columns == w && rows == h) { memcpy(dst, src, w * h * (size_t) ch * sizeof(float)); return 0; }
  if (xf > 4 && yf > 4) {
    a = (float *) malloc(16 * columns * rows * (size_t) ch * sizeof(float));
    if (!a) return -1;
    rc = orc_sample(cur, cw, chh, ch, a, 4 * columns, 4 * rows);
    cur = a; cw = 4 * columns; chh = 4 * rows;
  }
  if (rc == 0 && xf > 2 && yf > 2) {
    b = (float *) malloc(4 * columns * rows * (size_t) ch * sizeof(float));
    if (!b) { free(a); return -1; }
    rc = orc_resize(cur, cw, chh, ch, b, 2 * columns, 2 * rows, ORC_F_BOX);
    cur = b; cw = 2 * columns; chh = 2 * rows;
  }
  if (rc == 0) rc = orc_resize(cur, cw, chh, ch, dst, columns, rows, ORC_F_LANCZOS_SHARP);
  free(a); free(b);
  return rc;
}


/* ------------------------------------------------------------------------------------------
   effect.c:2316-2345 GetMotionBlurKernel + :2347-2560 MotionBlurImage (groundwork for the next
   hot-path row, SURVEY 8f-4): a one-sided Gaussian of `width` taps walked along `angle` from the
   output pixel, integer offsets ceil(w*cos - 0.5) / ceil(w*sin - 0.5), edge-replicated source
   (cache.c:2663), alpha-weighted blend for the colour channels of images with alpha.
   ------------------------------------------------------------------------------------------ */
int orc_motion_blur(const float *src, float *dst, size_t w, size_t h, int ch, double radius, double sigma,
                    double angle)
{
  const size_t width = orc_optimal_kernel_width_1d(radius, sigma);
  const double s = fabs(sigma) < EPS ? EPS : sigma;                 /* MagickSigma */
  double *kernel = (double *) malloc(width * sizeof(double)), normalize = 0.0;
  long *ox = (long *) malloc(width * sizeof(long)), *oy = (long *) malloc(width * sizeof(long));
  const int has_alpha = (ch == 2 || ch == 4);
  double px, py;
  size_t i;
  long y;
  if (!kernel || !ox || !oy) { free(kernel); free(ox); free(oy); return -1; }
  for (i = 0; i < width; i++) {
    kernel[i] = exp((-((double) i * i) / (double) (2.0 * s * s))) / (SQ2PI_ * s);
    normalize += kernel[i];
  }
  for (i = 0; i < width; i++) kernel[i] /= normalize;
  px = (double) width * sin((double) (PI_ * angle / 180.0));
  py = (double) width * cos((double) (PI_ * angle / 180.0));
  for (i = 0; i < width; i++) {
    ox[i] = (long) ceil((double) ((double) i * py) / hypot(px, py) - 0.5);     /* CastDoubleToLong of a small value */
    oy[i] = (long) ceil((double) ((double) i * px) / hypot(px, py) - 0.5);
  }
#pragma omp parallel for schedule(static)
  for (y = 0; y < (long) h; y++) {
    size_t x;
    for (x = 0; x < w; x++) {
      int c;
      for (c = 0; c < ch; c++) {
        double pixel = 0.0, gamma = 0.0;
        size_t j;
        const int blend = has_alpha && c != ch - 1;
        for (j = 0; j < width; j++) {
          long xx = (long) x + ox[j], yy = y + oy[j];
          const float *r;
          xx = xx < 0 ? 0 : (xx >= (long) w ? (long) w - 1 : xx);
          yy = yy < 0 ? 0 : (yy >= (long) h ? (long) h - 1 : yy);
          r = src + ((size_t) yy * w + (size_t) xx) * ch;
          if (!blend) pixel += kernel[j] * (double) r[c];
          else {
            const double alpha = QS * (double) r[ch - 1];
            pixel += kernel[j] * alpha * (double) r[c];
            gamma += kernel[j] * alpha;
          }
        }
        if (blend) pixel = perceptible_reciprocal(gamma) * pixel;
        dst[((size_t) y * w + x) * ch + c] = (float) pixel;
      }
    }
  }
  free(kernel); free(ox); free(oy);
  return 0;
}


/* ------------------------------------------------------------------------------------------
   effect.c:821-1165 BilateralBlurImage (groundwork, SURVEY 8f-4).  Odd window sizes only: for even
   sizes the reference's reflected window index (2*mid - v) steps outside the window it fetched.
   Tonal weight = gaussian of the 8-bit intensity difference (ScaleQuantumToChar of the FLOAT-converted
   GetPixelIntensity, quantum.h:113-124), spatial weight = gaussian of the distance; colour channels of
   images with alpha accumulate w*r but normalise by sum w*alpha(p)*alpha(r) (:1108-1125), as written.
   The reference never initialises intensity_gaussian[510] (difference == +255, :935); the oracle uses
   BlurGaussian(255) there -- inputs with a full-range 8-bit jump inside one window are outside the pin.
   ------------------------------------------------------------------------------------------ */
static double blur_gaussian(double x, double sigma)
{
  return exp(-((double) x * x) * perceptible_reciprocal(2.0 * sigma * sigma)) *
         perceptible_reciprocal(TWOPI_ * sigma * sigma);
}

static unsigned char scale_quantum_to_char(float quantum)
{
  if (quantum != quantum || quantum <= 0.0f) return 0;
  if ((quantum / 257.0f) >= 255.0f) return 255;
  return (unsigned char) (quantum / 257.0f + 0.5f);
}

int orc_bilateral_blur(const float *src, float *dst, size_t w, size_t h, int ch, size_t width, size_t height,
                       double intensity_sigma, double spatial_sigma)
{
  const long W = (long) (width > 1 ? width : 1), Hh = (long) (height > 1 ? height : 1);
  const long midx = W / 2, midy = Hh / 2;
  const int has_alpha = (ch == 2 || ch == 4);
  double ig[512], *sg;
  long y, u, v, n = 0;
  if ((W % 2) == 0 || (Hh % 2) == 0) return -1;
  sg = (double *) malloc((size_t) (W * Hh) * sizeof(double));
  if (!sg) return -1;
  for (v = -255; v <= 255; v++) ig[v + 255] = blur_gaussian((double) v, intensity_sigma);
  for (v = 0; v < Hh; v++)
    for (u = 0; u < W; u++) {
      const double dx = (double) 0 - (double) (u - midx), dy = (double) 0 - (double) (v - midy);
      sg[n++] = blur_gaussian(sqrt(dx * dx + dy * dy), spatial_sigma);
    }
#pragma omp parallel for schedule(static) private(u, v)
  for (y = 0; y < (long) h; y++) {
    double *wt = (double *) malloc((size_t) (W * Hh) * sizeof(double));
    long x;
    for (x = 0; x < (long) w; x++) {
      const float *p = src + ((size_t) y * w + (size_t) x) * ch;
      const double ip = (double) scale_quantum_to_char((float) pixel_intensity(p, ch));
      long k = 0;
      int c;
      for (v = 0; v < Hh; v++)
        for (u = 0; u < W; u++) {
          long xx = x + midx - u, yy = y + midy - v;
          const float *r;
          double d;
          xx = xx < 0 ? 0 : (xx >= (long) w ? (long) w - 1 : xx);
          yy = yy < 0 ? 0 : (yy >= (long) h ? (long) h - 1 : yy);
          r = src + ((size_t) yy * w + (size_t) xx) * ch;
          d = (double) scale_quantum_to_char((float) pixel_intensity(r, ch)) - ip;
          wt[k] = ig[(long) d + 255] * sg[k];
          k++;
        }
      for (c = 0; c < ch; c++) {
        double pixel = 0.0, gamma = 0.0;
        const int blend = has_alpha && c != ch - 1;
        k = 0;
        for (v = 0; v < Hh; v++)
          for (u = 0; u < W; u++) {
            long xx = x + midx - u, yy = y + midy - v;
            const float *r;
            xx = xx < 0 ? 0 : (xx >= (long) w ? (long) w - 1 : xx);
            yy = yy < 0 ? 0 : (yy >= (long) h ? (long) h - 1 : yy);
            r = src + ((size_t) yy * w + (size_t) xx) * ch;
            pixel += wt[k] * (double) r[c];
            if (!blend) gamma += wt[k];
            else gamma += wt[k] * (double) (QS * (double) p[ch - 1]) * (double) (QS * (double) r[ch - 1]);
            k++;
          }
        dst[((size_t) y * w + (size_t) x) * ch + c] = (float) (perceptible_reciprocal(gamma) * pixel);
      }
    }
    free(wt);
  }
  free(sg);
  return 0;
}


/* ------------------------------------------------------------------------------------------
   effect.c:3406-3700 SelectiveBlurImage: a width x width Gaussian (GetOptimalKernelWidth1D, not normalised) of which only
   the taps whose intensity differs from the centre pixel's by less than `threshold` take part.  Channels without the
   Blend trait (no alpha, or the alpha channel) compare the neighbour's intensity in a clone transformed to GRAYColorspace
   (:3629) with the centre's double intensity: the clone holds the FLOAT-rounded intensity (colorspace.c:943-945; a gray
   image is left as it is), and with alpha it has two channels, so GetPixelIntensity (pixel.c:2366) returns
   0.212656 g + 0.715158 g + 0.072186 g of that sample rather than g.  The alpha-blended colour channels compare double
   intensities (:3657).  gamma == 0 (no tap qualifies) copies the centre.
   ------------------------------------------------------------------------------------------ */
int orc_selective_blur(const float *src, float *dst, size_t w, size_t h, int ch, double radius, double sigma, double threshold)
{
  const size_t width = orc_optimal_kernel_width_1d(radius, sigma);
  const double s = fabs(sigma) < EPS ? EPS : sigma;
  const long j = (long) (width - 1) / 2;
  const int has_alpha = (ch == 2 || ch == 4);
  double *kernel = (double *) malloc(width * width * sizeof(double));
  long u, v, y;
  size_t i = 0;
  if (!kernel) return -1;
  for (v = -j; v <= j; v++)
    for (u = -j; u <= j; u++)
      kernel[i++] = exp(-((double) u * u + v * v) / (2.0 * s * s)) / (2.0 * PI_ * s * s);
#pragma omp parallel for schedule(static) private(u, v)
  for (y = 0; y < (long) h; y++) {
    long x;
    for (x = 0; x < (long) w; x++) {
      const float *p = src + ((size_t) y * w + (size_t) x) * ch;
      const double intensity = pixel_intensity(p, ch);
      int c;
      for (c = 0; c < ch; c++) {
        const int blend = has_alpha && c != ch - 1;
        double pixel = 0.0, gamma = 0.0;
        const double *k = kernel;
        for (v = 0; v < (long) width; v++)
          for (u = 0; u < (long) width; u++, k++) {
            long xx = x - j + u, yy = y - j + v;
            const float *r;
            double contrast;
            xx = xx < 0 ? 0 : (xx >= (long) w ? (long) w - 1 : xx);
            yy = yy < 0 ? 0 : (yy >= (long) h ? (long) h - 1 : yy);
            r = src + ((size_t) yy * w + (size_t) xx) * ch;
            if (!blend) {
              /* the GRAY clone's sample is the float intensity (a gray image's own sample); with alpha the clone
                 keeps two channels, so GetPixelIntensity weighs that sample as (g, g, g) again */
              const float g = ch >= 3 ? (float) pixel_intensity(r, ch) : r[0];
              const double luminance = has_alpha ? 0.212656 * g + 0.715158 * g + 0.072186 * g : (double) g;
              contrast = luminance - intensity;
              if (fabs(contrast) < threshold) { pixel += (*k) * (double) r[c]; gamma += (*k); }
            } else {
              contrast = pixel_intensity(r, ch) - intensity;
              if (fabs(contrast) < threshold) {
                const double alpha = QS * (double) r[ch - 1];
                pixel += (*k) * alpha * (double) r[c];
                gamma += (*k) * alpha;
              }
            }
          }
        if (fabs(gamma) < EPS) dst[((size_t) y * w + (size_t) x) * ch + c] = p[c];
        else dst[((size_t) y * w + (size_t) x) * ch + c] = (float) (perceptible_reciprocal(gamma) * pixel);
      }
    }
  }
  free(kernel);
  return 0;
}

/* ------------------------------------------------------------------------------------------
   effect.c:3129-3400 RotationalBlurImage (groundwork, SURVEY 8f-4): n samples on the arc through the
   pixel about the image centre (cos/sin tables of theta*w - offset), every `step`-th one taken
   (step = blur_radius / radius, clamped to [1, n-1]); sample coordinates are (ssize_t)(value + 0.5)
   (truncation toward zero) with edge replication; plain average without alpha / for the alpha
   channel, alpha-weighted average for the colour channels of images with alpha.
   ------------------------------------------------------------------------------------------ */
int orc_rotational_blur(const float *src, float *dst, size_t w, size_t h, int ch, double angle)
{
  const double cx = (double) (w - 1) / 2.0, cy = (double) (h - 1) / 2.0;
  const double blur_radius = hypot(cx, cy);
  const double rad = (double) (PI_ * angle / 180.0);
  const size_t n = (size_t) fabs(4.0 * rad * sqrt((double) blur_radius) + 2UL);
  const double theta = rad / (double) (n - 1), offset = theta * (double) (n - 1) / 2.0;
  const int has_alpha = (ch == 2 || ch == 4);
  double *ct, *st;
  long y;
  size_t k;
  if (n < 2) return -1;
  ct = (double *) malloc(n * sizeof(double));
  st = (double *) malloc(n * sizeof(double));
  if (!ct || !st) { free(ct); free(st); return -1; }
  for (k = 0; k < n; k++) {
    ct[k] = cos((double) (theta * (double) (long) k - offset));
    st[k] = sin((double) (theta * (double) (long) k - offset));
  }
#pragma omp parallel for schedule(static)
  for (y = 0; y < (long) h; y++) {
    long x;
    for (x = 0; x < (long) w; x++) {
      const double dx = (double) x - cx, dy = (double) y - cy;
      const double radius = hypot(dx, dy);
      size_t step = 1;
      int c;
      if (radius != 0) {
        step = (size_t) (blur_radius / radius);
        if (step == 0) step = 1;
        else if (step >= n) step = n - 1;
      }
      for (c = 0; c < ch; c++) {
        double gamma = 0.0, pixel = 0.0;
        const int blend = has_alpha && c != ch - 1;
        size_t j;
        for (j = 0; j < n; j += step) {
          long xx = (long) (cx + dx * ct[j] - dy * st[j] + 0.5);
          long yy = (long) (cy + dx * st[j] + dy * ct[j] + 0.5);
          const float *r;
          xx = xx < 0 ? 0 : (xx >= (long) w ? (long) w - 1 : xx);
          yy = yy < 0 ? 0 : (yy >= (long) h ? (long) h - 1 : yy);
          r = src + ((size_t) yy * w + (size_t) xx) * ch;
          if (!blend) { pixel += (double) r[c]; gamma++; }
          else {
            const double alpha = QS * (double) r[ch - 1];
            pixel += alpha * (double) r[c];
            gamma += alpha;
          }
        }
        dst[((size_t) y * w + (size_t) x) * ch + c] = (float) (perceptible_reciprocal(gamma) * pixel);
      }
    }
  }
  free(ct); free(st);
  return 0;
}


/* ------------------------------------------------------------------------------------------
   statistic.c:2918-3160 StatisticImage (groundwork, SURVEY 8f-4): per channel (alpha included, every
   channel carries the Update trait) over the max(width,1) x max(height,1) window whose top-left corner is
   (x - width/2, y - height/2), edge-replicated.  Gradient / Maximum / Mean / Minimum / RootMeanSquare /
   StandardDeviation / Contrast accumulate in double in row-major window order; Median goes through the
   reference's 16-bit skip list (InsertPixelList :2878 -> ScaleQuantumToShort; GetMedianPixelList :2784
   returns the element at sorted index length/2), so its result is an integer Quantum.  Mode (:2809) walks the
   distinct values in ascending order and keeps the first one whose count is strictly the greatest; Nonpeak (:2843) is the
   median's value unless that value is the smallest (largest) distinct value of the window and a larger (smaller) one
   exists, in which case it steps to that neighbour.  type: statistic.h:141-151 numeric values.
   ------------------------------------------------------------------------------------------ */
static unsigned short scale_quantum_to_short(float q)
{
  if (q != q || q <= 0.0f) return 0;
  if (q >= 65535.0f) return 65535;
  return (unsigned short) (q + 0.5f);
}

static int cmp_ushort(const void *a, const void *b)
{
  const unsigned short x = *(const unsigned short *) a, y = *(const unsigned short *) b;
  return x < y ? -1 : (x > y ? 1 : 0);
}

int orc_statistic(const float *src, float *dst, size_t w, size_t h, int ch, int type, size_t width, size_t height)
{
  const long W = (long) (width > 1 ? width : 1), Hh = (long) (height > 1 ? height : 1);
  long y;
  if (type < 1 || type > 10) return -1;
#pragma omp parallel for schedule(static)
  for (y = 0; y < (long) h; y++) {
    unsigned short *list = (unsigned short *) malloc((size_t) (W * Hh) * sizeof(unsigned short));
    long x;
    for (x = 0; x < (long) w; x++) {
      int c;
      for (c = 0; c < ch; c++) {
        double area = 0.0, minimum = 0.0, maximum = 0.0, sum = 0.0, sum_squared = 0.0, pixel;
        long u, v, n = 0;
        for (v = 0; v < Hh; v++)
          for (u = 0; u < W; u++) {
            long xx = x - W / 2 + u, yy = y - Hh / 2 + v;
            double value;
            xx = xx < 0 ? 0 : (xx >= (long) w ? (long) w - 1 : xx);
            yy = yy < 0 ? 0 : (yy >= (long) h ? (long) h - 1 : yy);
            value = (double) src[((size_t) yy * w + (size_t) xx) * ch + c];
            if (n == 0) { minimum = value; maximum = value; }
            list[n++] = scale_quantum_to_short((float) value);
            area++;
            if (value < minimum) minimum = value;
            if (value > maximum) maximum = value;
            sum += value;
            sum_squared += value * value;
          }
        switch (type) {
          /* MagickAbsoluteValue (image-private.h:45), x < 0 ? -x : x, keeps the sign of a zero (and of a NaN) */
          case 1: pixel = maximum - minimum; pixel = pixel < 0 ? -pixel : pixel; break;              /* Gradient */
          case 2: pixel = maximum; break;
          case 4:
            qsort(list, (size_t) n, sizeof(unsigned short), cmp_ushort);
            pixel = (double) list[n >> 1];
            break;
          case 5: pixel = minimum; break;
          case 6: {                                                                                /* Mode */
            long i = 0, best = 0;
            qsort(list, (size_t) n, sizeof(unsigned short), cmp_ushort);
            pixel = 65536.0;                       /* the root node; unreachable for n >= 1 */
            while (i < n) {
              long j = i;
              while (j < n && list[j] == list[i]) j++;
              if (j - i > best) { best = j - i; pixel = (double) list[i]; }
              i = j;
            }
            break;
          }
          case 7: {                                                                                /* Nonpeak */
            long i, at = n >> 1;
            long previous = -1, next = -1;
            qsort(list, (size_t) n, sizeof(unsigned short), cmp_ushort);
            for (i = 0; i < n; i++) {
              if (list[i] < list[at]) previous = list[i];
              if (list[i] > list[at] && next < 0) next = list[i];
            }
            pixel = (double) list[at];
            if (previous < 0 && next >= 0) pixel = (double) next;
            else if (previous >= 0 && next < 0) pixel = (double) previous;
            break;
          }
          case 8: pixel = sqrt(sum_squared / area); break;
          case 9: pixel = sqrt(sum_squared / area - (sum / area * sum / area)); break;
          case 10:
            pixel = (maximum - minimum) * perceptible_reciprocal(maximum + minimum);
            pixel = pixel < 0 ? -pixel : pixel;
            break;
          default: pixel = sum / area; break;                                                      /* Mean */
        }
        dst[((size_t) y * w + (size_t) x) * ch + c] = (float) pixel;
      }
    }
    free(list);
  }
  return 0;
}

/* ------------------------------------------------------------------------------------------
   effect.c:128-416 AdaptiveBlurImage / :447-735 AdaptiveSharpenImage (sharpen != 0).
     edge  = EdgeImage(image, radius)                              (:181)
     AutoLevelImage(edge) = MinMaxStretchImage(edge, 0, 0, 1.0)    (enhance.c:266, histogram.c:927): the default channel
             mask is AllChannels, so ONE range over every channel (GetImageRange statistic.c:1851: plain comparisons seeded
             with each row's first sample, so NaN never wins but a row starting with NaN is dropped), LevelImage (enhance.c:2913: QuantumRange * (PerceptibleReciprocal(max - min) * (pixel - min)), gamma 1 so
             gamma_pow is the identity; skipped when |min - max| < MagickEpsilon) and ClampImage (threshold.c:1087)
     edge  = BlurImage(edge, radius, sigma); AutoLevelImage(edge)  (:188-194)
     width = GetOptimalKernelWidth2D(radius, sigma); kernel[j], j = 0, 2, ..: (width - j)^2 Gaussians, the centre absorbs
             1 - sum (blur) or is set to -2 * sum of the negated Gaussian (sharpen)                     (:199-236)
     per pixel: j = ceil(width * (1 - QS * intensity(edge)) - 0.5) clipped to [0, width], made even; the (width - j)^2
             window around the pixel is weighted with kernel[j] in plain (not reflected) order            (:279-372)
   ------------------------------------------------------------------------------------------ */
static void auto_level(float *buf, size_t w, size_t h, int ch)
{
  const size_t n = w * h * (size_t) ch, row = w * (size_t) ch;
  double minima = 1.7976931348623157e308, maxima = 2.2250738585072014e-308, scale;   /* MagickMaximumValue / Minimum */
  size_t i, y;
  /* GetImageRange seeds each row's extremes with the row's first sample, so a row that starts with NaN stays NaN and
     the merge drops it whole (statistic.c:1895-1896, :1921-1924) */
  for (y = 0; y < h; y++) {
    double row_minima = (double) buf[y * row], row_maxima = row_minima;
    for (i = y * row; i < (y + 1) * row; i++) {
      if ((double) buf[i] < row_minima) row_minima = (double) buf[i];
      if ((double) buf[i] > row_maxima) row_maxima = (double) buf[i];
    }
    if (row_minima < minima) minima = row_minima;
    if (row_maxima > maxima) maxima = row_maxima;
  }
  if (!(fabs(minima - maxima) >= EPS)) return;
  scale = perceptible_reciprocal(maxima - minima);
  for (i = 0; i < n; i++) {
    const double level = QR * (scale * ((double) buf[i] - minima));
    buf[i] = clamp_pixel((double) (float) level);
  }
}

static int adaptive_filter(const float *src, float *dst, size_t w, size_t h, int ch, double radius, double sigma, int sharpen)
{
  const size_t n = w * h * (size_t) ch, width = orc_optimal_kernel_width_2d(radius, sigma);
  const double s = fabs(sigma) < EPS ? EPS : sigma;
  const int has_alpha = (ch == 2 || ch == 4);
  float *edge, *tmp;
  double **kernel;
  long jw, y;
  int rc = -1;
  if (fabs(sigma) < EPS) { memcpy(dst, src, n * sizeof(float)); return 0; }
  edge = (float *) malloc(n * sizeof(float));
  tmp = (float *) malloc(n * sizeof(float));
  kernel = (double **) calloc(width, sizeof(*kernel));
  if (!edge || !tmp || !kernel) goto done;
  if (orc_edge(src, edge, w, h, ch, radius)) goto done;
  auto_level(edge, w, h, ch);
  if (orc_blur(edge, tmp, w, h, ch, radius, sigma)) goto done;
  auto_level(tmp, w, h, ch);
  for (jw = 0; jw < (long) width; jw += 2) {
    const long size = (long) width - jw, j = (size - 1) / 2;
    double normalize = 0.0;
    long u, v, k = 0;
    kernel[jw] = (double *) malloc((size_t) (size * size) * sizeof(double));
    if (!kernel[jw]) goto done;
    for (v = -j; v <= j; v++)
      for (u = -j; u <= j; u++) {
        const double g = exp(-((double) u * u + v * v) / (2.0 * s * s)) / (2.0 * PI_ * s * s);
        kernel[jw][k] = sharpen ? -g : g;
        normalize += kernel[jw][k];
        k++;
      }
    if (sharpen) kernel[jw][(k - 1) / 2] = (-2.0) * normalize;
    else kernel[jw][(k - 1) / 2] += 1.0 - normalize;
    if (sigma < EPS) kernel[jw][(k - 1) / 2] = 1.0;
  }
#pragma omp parallel for schedule(static)
  for (y = 0; y < (long) h; y++) {
    long x;
    for (x = 0; x < (long) w; x++) {
      const float *r = tmp + ((size_t) y * w + (size_t) x) * ch;
      double t = ceil((double) width * (1.0 - QS * pixel_intensity(r, ch)) - 0.5);
      long j, size, x0, y0, u, v;
      int c;
      j = t != t ? 0 : (t >= 9.2233720368547758e18 ? LONG_MAX : (t <= -9.2233720368547758e18 ? LONG_MIN : (long) t));
      if (j < 0) j = 0; else if (j > (long) width) j = (long) width;
      if ((j & 0x01) != 0) j--;
      size = (long) width - j;
      x0 = x - size / 2; y0 = y - size / 2;
      for (c = 0; c < ch; c++) {
        const int blend = has_alpha && c != ch - 1;
        const double *k = kernel[j];
        double pixel = 0.0, gamma = 0.0;
        for (v = 0; v < size; v++)
          for (u = 0; u < size; u++, k++) {
            const float *p = src + ((size_t) clampl(y0 + v, 0, (long) h - 1) * w + (size_t) clampl(x0 + u, 0, (long) w - 1)) * ch;
            if (!blend) { pixel += (*k) * (double) p[c]; gamma += (*k); }
            else {
              const double alpha = (double) (QS * (double) p[ch - 1]);
              pixel += (*k) * alpha * (double) p[c];
              gamma += (*k) * alpha;
            }
          }
        gamma = perceptible_reciprocal(gamma);
        dst[((size_t) y * w + (size_t) x) * ch + c] = (float) (gamma * pixel);
      }
    }
  }
  rc = 0;
done:
  if (kernel) { for (jw = 0; jw < (long) width; jw++) free(kernel[jw]); free(kernel); }
  free(edge); free(tmp);
  return rc;
}

int orc_adaptive_blur(const float *src, float *dst, size_t w, size_t h, int ch, double radius, double sigma)
{ return adaptive_filter(src, dst, w, h, ch, radius, sigma, 0); }
int orc_adaptive_sharpen(const float *src, float *dst, size_t w, size_t h, int ch, double radius, double sigma)
{ return adaptive_filter(src, dst, w, h, ch, radius, sigma, 1); }
