/*
  oracle/threshold_oracle.c -- TEST INFRASTRUCTURE ONLY.  Never linked into, imported by or executed from the product.

  The plain-C oracle of the threshold.c operators the GPU serves beyond Bilevel / Black / White / Clamp (ImageMagick
  7.1.1-45 Q16-HDRI): AdaptiveThresholdImage, AutoThresholdImage, RangeThresholdImage and PerceptibleImage, restated in
  the reference's operation order.  It builds on the main oracle's pixel_intensity, perceptible_reciprocal,
  scale_quantum_to_char and orc_threshold, which are file-local there, so this translation unit includes oracle.c.
  Built by oracle/Makefile into oracle/libthreshold_oracle.so with the main oracle's flags (no contraction, standard
  excess precision); pinned bit for bit against the reference compiled from source by
  tests/test_oracle_threshold_vs_ref.py.  Buffers as in oracle.h; `update_mask` bit c = channel c has the Update trait.

    int orc_adaptive_threshold(const float *src, float *dst, size_t w, size_t h, int ch, size_t ww, size_t wh,
                               double bias, unsigned update_mask);                       out of place, edge virtual pixels
    int orc_auto_threshold(float *buf, size_t w, size_t h, int ch, int method, double *threshold);    default mask
    int orc_range_threshold(float *buf, size_t w, size_t h, int ch, double low_black, double low_white,
                            double high_white, double high_black, int per_channel, unsigned update_mask);  3-4 channels
    int orc_perceptible(float *buf, size_t w, size_t h, int ch, double epsilon, unsigned update_mask);
*/
#include "oracle.c"

static long clamp_index(long v, long n) { return v < 0 ? 0 : (v >= n ? n - 1 : v); }

/* threshold.c:182-353 */
int orc_adaptive_threshold(const float *src, float *dst, size_t w, size_t h, int ch, size_t ww, size_t wh, double bias,
                           unsigned update_mask)
{
  long y;
  const unsigned long long number_pixels = (unsigned long long) ww * wh;
  if (ch < 1 || ch > 4) return -1;
  if (ww == 0 || wh == 0) { memcpy(dst, src, w * h * (size_t) ch * sizeof(float)); return 0; }
#pragma omp parallel for schedule(static)
  for (y = 0; y < (long) h; y++) {
    const long top = y - (long) (wh / 2), left = -(long) (ww / 2);
    int c;
    for (c = 0; c < ch; c++) {
      long x, u, v;
#define SAMPLE(vv, jj) ((double) src[((size_t) clamp_index(top + (vv), (long) h) * w + \
                                      (size_t) clamp_index(left + (jj), (long) w)) * ch + c])
      double sum = 0.0, bias_sum = 0.0;
      if (((update_mask >> c) & 1u) == 0) {
        for (x = 0; x < (long) w; x++) dst[((size_t) y * w + x) * ch + c] = src[((size_t) y * w + x) * ch + c];
        continue;
      }
      for (v = 0; v < (long) wh; v++)
        for (u = 0; u < (long) ww; u++) {
          if (u == (long) ww - 1) bias_sum += SAMPLE(v, u);
          sum += SAMPLE(v, u);
        }
      for (x = 0; x < (long) w; x++) {
        double mean;
        sum -= bias_sum;
        bias_sum = 0.0;
        for (v = 0; v < (long) wh; v++) {
          bias_sum += SAMPLE(v, x);
          sum += SAMPLE(v, x + (long) ww - 1);
        }
        mean = (double) (sum / number_pixels + bias);
        dst[((size_t) y * w + x) * ch + c] =
            (float) ((double) src[((size_t) y * w + x) * ch + c] <= mean ? 0 : QR);
      }
#undef SAMPLE
    }
  }
  return 0;
}

#define MAX_INTENSITY 255

static double kapur(const double *histogram)
{
  double cumulative[MAX_INTENSITY + 1], black[MAX_INTENSITY + 1], white[MAX_INTENSITY + 1], entropy, maximum, epsilon;
  long i, j;
  size_t threshold;
  cumulative[0] = histogram[0];
  for (i = 1; i <= MAX_INTENSITY; i++) cumulative[i] = cumulative[i - 1] + histogram[i];
  epsilon = 2.22507385850720140E-308;
  for (j = 0; j <= MAX_INTENSITY; j++) {
    black[j] = 0.0;
    if (cumulative[j] > epsilon) {
      entropy = 0.0;
      for (i = 0; i <= j; i++)
        if (histogram[i] > epsilon) entropy -= histogram[i] / cumulative[j] * log(histogram[i] / cumulative[j]);
      black[j] = entropy;
    }
    white[j] = 0.0;
    if ((1.0 - cumulative[j]) > epsilon) {
      entropy = 0.0;
      for (i = j + 1; i <= MAX_INTENSITY; i++)
        if (histogram[i] > epsilon)
          entropy -= histogram[i] / (1.0 - cumulative[j]) * log(histogram[i] / (1.0 - cumulative[j]));
      white[j] = entropy;
    }
  }
  maximum = black[0] + white[0];
  threshold = 0;
  for (j = 1; j <= MAX_INTENSITY; j++)
    if ((black[j] + white[j]) > maximum) { maximum = black[j] + white[j]; threshold = (size_t) j; }
  return 100.0 * threshold / MAX_INTENSITY;
}

static double otsu(const double *histogram)
{
  double myu[MAX_INTENSITY + 1], omega[MAX_INTENSITY + 1], sigma, max_sigma = 0.0, threshold = 0.0;
  long i;
  omega[0] = histogram[0];
  myu[0] = 0.0;
  for (i = 1; i <= MAX_INTENSITY; i++) { omega[i] = omega[i - 1] + histogram[i]; myu[i] = myu[i - 1] + i * histogram[i]; }
  for (i = 0; i < MAX_INTENSITY; i++) {
    sigma = 0.0;
    if ((omega[i] != 0.0) && (omega[i] != 1.0))
      sigma = pow(myu[MAX_INTENSITY] * omega[i] - myu[i], 2.0) / (omega[i] * (1.0 - omega[i]));
    if (sigma > max_sigma) { max_sigma = sigma; threshold = (double) i; }
  }
  return 100.0 * threshold / MAX_INTENSITY;
}

static double triangle(const double *histogram)
{
  double a, b, c, count, distance, inverse_ratio, max_distance, segment, x1, x2, y1, y2;
  long i, end = 0, max = 0, start = 0, threshold = 0;
  for (i = 0; i <= MAX_INTENSITY; i++) if (histogram[i] > 0.0) { start = i; break; }
  for (i = MAX_INTENSITY; i >= 0; i--) if (histogram[i] > 0.0) { end = i; break; }
  count = 0.0;
  for (i = 0; i <= MAX_INTENSITY; i++) if (histogram[i] > count) { max = i; count = histogram[i]; }
  x1 = (double) max; y1 = histogram[max]; x2 = (double) end;
  if ((max - start) >= (end - max)) x2 = (double) start;
  y2 = 0.0; a = y1 - y2; b = x2 - x1; c = (-1.0) * (a * x1 + b * y1);
  inverse_ratio = 1.0 / sqrt(a * a + b * b + c * c);
  max_distance = 0.0;
  if (x2 == (double) start)
    for (i = start; i < max; i++) {
      segment = inverse_ratio * (a * i + b * histogram[i] + c);
      distance = sqrt(segment * segment);
      if ((distance > max_distance) && (segment > 0.0)) { threshold = i; max_distance = distance; }
    }
  else
    for (i = end; i > max; i--) {
      segment = inverse_ratio * (a * i + b * histogram[i] + c);
      distance = sqrt(segment * segment);
      if ((distance > max_distance) && (segment < 0.0)) { threshold = i; max_distance = distance; }
    }
  return 100.0 * threshold / MAX_INTENSITY;
}

/* threshold.c:660-789; method: 0 Undefined (OTSU), 1 Kapur, 2 OTSU, 3 Triangle */
int orc_auto_threshold(float *buf, size_t w, size_t h, int ch, int method, double *threshold)
{
  double histogram[MAX_INTENSITY + 1], sum = 0.0, gamma, t[4] = {0, 0, 0, 0};
  size_t i, n = w * h;
  if (ch < 1 || ch > 4) return -1;
  memset(histogram, 0, sizeof(histogram));
  for (i = 0; i < n; i++) histogram[scale_quantum_to_char((float) pixel_intensity(buf + i * ch, ch))]++;
  for (i = 0; i <= MAX_INTENSITY; i++) sum += histogram[i];
  gamma = perceptible_reciprocal(sum);
  for (i = 0; i <= MAX_INTENSITY; i++) histogram[i] = gamma * histogram[i];
  *threshold = method == 1 ? kapur(histogram) : method == 3 ? triangle(histogram) : otsu(histogram);
  t[0] = (double) QR * *threshold / 100.0;
  return orc_threshold(buf, w, h, ch, 0, t);
}

/* threshold.c:2377-2481 on an sRGB image */
int orc_range_threshold(float *buf, size_t w, size_t h, int ch, double low_black, double low_white, double high_white,
                        double high_black, int per_channel, unsigned update_mask)
{
  long i, n = (long) (w * h);
  if (ch < 3 || ch > 4) return -1;
#pragma omp parallel for schedule(static)
  for (i = 0; i < n; i++) {
    float *q = buf + (size_t) i * ch;
    double pixel = pixel_intensity(q, ch);
    int c;
    for (c = 0; c < ch; c++) {
      if (((update_mask >> c) & 1u) == 0) continue;
      if (per_channel) pixel = (double) q[c];
      if (pixel < low_black) q[c] = 0.0f;
      else if ((pixel >= low_black) && (pixel < low_white))
        q[c] = (float) ((double) QR * perceptible_reciprocal(low_white - low_black) * (pixel - low_black));
      else if ((pixel >= low_white) && (pixel <= high_white)) q[c] = (float) QR;
      else if ((pixel > high_white) && (pixel <= high_black))
        q[c] = (float) ((double) QR * (double) perceptible_reciprocal(high_black - high_white) * (high_black - pixel));
      else q[c] = 0.0f;
    }
  }
  return 0;
}

/* threshold.c:2080-2090, :2138-2165 */
int orc_perceptible(float *buf, size_t w, size_t h, int ch, double epsilon, unsigned update_mask)
{
  size_t i, n = w * h * (size_t) ch;
  if (ch < 1 || ch > 4) return -1;
  for (i = 0; i < n; i++) {
    double sign;
    if (((update_mask >> (i % (size_t) ch)) & 1u) == 0) continue;
    sign = (double) buf[i] < 0.0 ? -1.0 : 1.0;
    if (!((sign * (double) buf[i]) >= epsilon)) buf[i] = (float) (sign * epsilon);
  }
  return 0;
}
