/*
  oracle/level_oracle.c -- TEST INFRASTRUCTURE ONLY.  Never linked into, imported by or executed from the product.

  The plain-C oracle of the level and stretch operators of enhance.c (ImageMagick 7.1.1-45 Q16-HDRI): LevelImage,
  LevelizeImage, MinMaxStretchImage (AutoLevelImage), ContrastStretchImage (NormalizeImage), LinearStretchImage and
  GammaImage, restated in the reference's operation order.  It builds on the main oracle's pixel_intensity,
  perceptible_reciprocal, scale_quantum_to_map and scale_map_to_quantum, which are file-local there, so this translation
  unit includes oracle.c.  Built by oracle/Makefile into oracle/liblevel_oracle.so with the main oracle's flags (no
  contraction, standard excess precision); pinned bit for bit against the reference compiled from source by
  tests/test_oracle_level_vs_ref.py.  Buffers as in oracle.h; `update_mask` bit c = channel c has the Update trait;
  `per_channel` = the image's channel mask is not AllChannels.

    int orc_level(float *buf, size_t w, size_t h, int ch, double black, double white, double gamma, unsigned update_mask);
    int orc_levelize(...same...);
    int orc_minmax_stretch(float *buf, size_t w, size_t h, int ch, double black, double white, double gamma,
                           int per_channel, unsigned update_mask);
    int orc_identify_gray(const float *buf, size_t w, size_t h, int ch);           0 not gray, 1 grayscale, 2 bilevel
    int orc_contrast_stretch(float *buf, size_t w, size_t h, int ch, double black_point, double white_point,
                             int per_channel, unsigned update_mask, char *property);
        IdentifyImageType's re-layout first (a gray-valued 3-4 channel image keeps channel 0 and alpha, and channel 0's
        and alpha's Update bits); returns the channel count of the result.  `property`: the "histogram:contrast-stretch"
        value (at least 64 bytes).
    int orc_linear_stretch(float *buf, size_t w, size_t h, int ch, double black_point, double white_point,
                           unsigned update_mask, char *property);
    int orc_gamma(float *buf, size_t w, size_t h, int ch, double gamma, unsigned update_mask);
*/
#include "oracle.c"

#include <stdio.h>

static double gamma_pow(double value, double gamma) { return value < 0.0 ? value : pow(value, gamma); }

/* enhance.c:2900-3018 LevelImage, then threshold.c:1087 ClampImage on the same channels */
int orc_level(float *buf, size_t w, size_t h, int ch, double black, double white, double gamma, unsigned update_mask)
{
  long i, n = (long) (w * h);
  if (ch < 1 || ch > 4) return -1;
#pragma omp parallel for schedule(static)
  for (i = 0; i < n; i++) {
    float *q = buf + (size_t) i * ch;
    int c;
    for (c = 0; c < ch; c++) {
      double scale;
      float v;
      if (((update_mask >> c) & 1u) == 0) continue;
      scale = perceptible_reciprocal(white - black);
      v = (float) ((double) QR * gamma_pow(scale * ((double) q[c] - black), perceptible_reciprocal(gamma)));
      if ((double) v < 0.0) v = 0.0f;
      else if ((double) v >= QR) v = (float) QR;
      q[c] = v;
    }
  }
  return 0;
}

/* enhance.c:3062-3168 LevelizeImage (no clamp) */
int orc_levelize(float *buf, size_t w, size_t h, int ch, double black, double white, double gamma, unsigned update_mask)
{
  long i, n = (long) (w * h);
  if (ch < 1 || ch > 4) return -1;
#pragma omp parallel for schedule(static)
  for (i = 0; i < n; i++) {
    float *q = buf + (size_t) i * ch;
    int c;
    for (c = 0; c < ch; c++) {
      if (((update_mask >> c) & 1u) == 0) continue;
      q[c] = (float) (gamma_pow(QS * (double) q[c], gamma) * (white - black) + black);
    }
  }
  return 0;
}

/* statistic.c:1851-1929 GetImageRange over the channels of `select`; each row starts from its first sample of channel 0 */
static void image_range(const float *buf, size_t w, size_t h, int ch, unsigned select, double *minima, double *maxima)
{
  size_t y, x;
  *maxima = 2.22507385850720140E-308;          /* MagickMinimumValue */
  *minima = 1.79769313486231570E+308;          /* MagickMaximumValue */
  for (y = 0; y < h; y++) {
    const float *p = buf + y * w * (size_t) ch;
    double row_maxima = (double) p[0], row_minima = (double) p[0];
    for (x = 0; x < w; x++) {
      int c;
      for (c = 0; c < ch; c++) {
        if (((select >> c) & 1u) == 0) continue;
        if ((double) p[c] < row_minima) row_minima = (double) p[c];
        if ((double) p[c] > row_maxima) row_maxima = (double) p[c];
      }
      p += ch;
    }
    if (row_minima < *minima) *minima = row_minima;
    if (row_maxima > *maxima) *maxima = row_maxima;
  }
}

/* histogram.c:927-975 MinMaxStretchImage.  Per channel, SetImageChannelMask(1 << offset) selects the PixelChannel of that
   number: the colour channel at the offset (gray / red 0, green 1, blue 2), never alpha (PixelChannel 4). */
int orc_minmax_stretch(float *buf, size_t w, size_t h, int ch, double black, double white, double gamma, int per_channel,
                       unsigned update_mask)
{
  double min, max;
  int c;
  if (ch < 1 || ch > 4) return -1;
  if (!per_channel) {
    image_range(buf, w, h, ch, update_mask, &min, &max);
    min += black;
    max -= white;
    if (fabs(min - max) >= EPS) orc_level(buf, w, h, ch, min, max, gamma, update_mask);
    return 0;
  }
  for (c = 0; c < (ch >= 3 ? 3 : 1); c++) {
    if (((update_mask >> c) & 1u) == 0) continue;
    image_range(buf, w, h, ch, 1u << c, &min, &max);
    min += black;
    max -= white;
    if (fabs(min - max) >= EPS) orc_level(buf, w, h, ch, min, max, gamma, 1u << c);
  }
  return 0;
}

/* attribute.c:1564-1626 IdentifyImageGray's scan: IsPixelGray / IsPixelMonochrome */
int orc_identify_gray(const float *buf, size_t w, size_t h, int ch)
{
  size_t i, n = w * h;
  int type = 2;
  for (i = 0; i < n; i++) {
    const float *p = buf + i * (size_t) ch;
    const double r = (double) p[0], g = (double) p[ch >= 3 ? 1 : 0], b = (double) p[ch >= 3 ? 2 : 0];
    if (!(fabs(r - g) < EPS && fabs(g - b) < EPS)) return 0;
    if (fabs(r) >= EPS && fabs(r - QR) >= EPS) type = 1;
  }
  return type;
}

/* SetImageColorspace(GRAY) of a 3-4 channel image: the cache keeps channel 0 (and alpha) */
static int gray_relayout(float *buf, size_t n, int ch, unsigned *update_mask)
{
  const int out = ch == 4 ? 2 : 1;
  size_t i;
  for (i = 0; i < n; i++) {
    const float g = buf[i * (size_t) ch], a = buf[i * (size_t) ch + (size_t) (ch - 1)];
    buf[i * (size_t) out] = g;
    if (out == 2) buf[i * (size_t) out + 1] = a;
  }
  *update_mask = (*update_mask & 1u) | (ch == 4 && ((*update_mask >> 3) & 1u) ? 2u : 0u);
  return out;
}

/* enhance.c:1544-1818 ContrastStretchImage */
int orc_contrast_stretch(float *buf, size_t w, size_t h, int ch, double black_point, double white_point, int per_channel,
                         unsigned update_mask, char *property)
{
  const size_t n = w * h;
  double *histogram;
  float *stretch_map, black[4] = {0, 0, 0, 0}, white[4] = {0, 0, 0, 0};
  size_t i;
  int c;
  if (ch < 1 || ch > 4) return -1;
  if (ch >= 3 && orc_identify_gray(buf, w, h, ch) != 0) ch = gray_relayout(buf, n, ch, &update_mask);
  histogram = (double *) calloc(65536 * (size_t) ch, sizeof(double));
  stretch_map = (float *) calloc(65536 * (size_t) ch, sizeof(float));
  if (histogram == NULL || stretch_map == NULL) { free(histogram); free(stretch_map); return -1; }
  for (i = 0; i < n; i++) {
    const float *p = buf + i * (size_t) ch;
    double pixel = pixel_intensity(p, ch);
    for (c = 0; c < ch; c++) {
      if (per_channel) pixel = (double) p[c];
      histogram[(size_t) ch * scale_quantum_to_map((float) pixel) + (size_t) c]++;
    }
  }
  for (c = 0; c < ch; c++) {
    double intensity = 0.0;
    long j;
    for (j = 0; j <= 65535; j++) {
      intensity += histogram[(long) ch * j + c];
      if (intensity > black_point) break;
    }
    black[c] = (float) j;
    intensity = 0.0;
    for (j = 65535; j != 0; j--) {
      intensity += histogram[(long) ch * j + c];
      if (intensity > ((double) w * h - white_point)) break;
    }
    white[c] = (float) j;
  }
  for (c = 0; c < ch; c++) {
    long j;
    for (j = 0; j <= 65535; j++) {
      const double gamma = perceptible_reciprocal(white[c] - black[c]);
      if (j < (long) black[c]) stretch_map[(long) ch * j + c] = 0.0f;
      else if (j > (long) white[c]) stretch_map[(long) ch * j + c] = (float) QR;
      else if (black[c] != white[c])
        stretch_map[(long) ch * j + c] = scale_map_to_quantum((double) (65535.0 * gamma * (j - (double) black[c])));
    }
  }
  for (i = 0; i < n; i++) {
    float *q = buf + i * (size_t) ch;
    for (c = 0; c < ch; c++) {
      if (((update_mask >> c) & 1u) == 0 || black[c] == white[c]) continue;
      q[c] = stretch_map[(size_t) ch * scale_quantum_to_map(q[c]) + (size_t) c];
    }
  }
  if (property != NULL)
    snprintf(property, 64, "%gx%g%%", 100.0 * QS * pixel_intensity(black, ch), 100.0 * QS * pixel_intensity(white, ch));
  free(histogram);
  free(stretch_map);
  return ch;
}

/* enhance.c:3347-3427 LinearStretchImage */
int orc_linear_stretch(float *buf, size_t w, size_t h, int ch, double black_point, double white_point,
                       unsigned update_mask, char *property)
{
  const size_t n = w * h;
  double *histogram, intensity;
  long black, white;
  size_t i;
  if (ch < 1 || ch > 4) return -1;
  histogram = (double *) calloc(65536, sizeof(double));
  if (histogram == NULL) return -1;
  for (i = 0; i < n; i++) histogram[scale_quantum_to_map((float) pixel_intensity(buf + i * (size_t) ch, ch))]++;
  intensity = 0.0;
  for (black = 0; black < 65535; black++) {
    intensity += histogram[black];
    if (intensity >= black_point) break;
  }
  intensity = 0.0;
  for (white = 65535; white != 0; white--) {
    intensity += histogram[white];
    if (intensity >= white_point) break;
  }
  free(histogram);
  orc_level(buf, w, h, ch, (double) scale_map_to_quantum((double) black), (double) scale_map_to_quantum((double) white),
            1.0, update_mask);
  if (property != NULL) snprintf(property, 64, "%gx%g%%", 100.0 * black / 65535, 100.0 * white / 65535);
  return 0;
}

/* enhance.c:2322-2445 GammaImage */
int orc_gamma(float *buf, size_t w, size_t h, int ch, double gamma, unsigned update_mask)
{
  const size_t n = w * h;
  float *map;
  size_t i;
  if (ch < 1 || ch > 4) return -1;
  if (gamma == 1.0) return 0;
  map = (float *) calloc(65536, sizeof(float));
  if (map == NULL) return -1;
  if (gamma != 0.0)
    for (i = 0; i <= 65535; i++)
      map[i] = scale_map_to_quantum((double) (65535.0 * pow((double) i / 65535.0, perceptible_reciprocal(gamma))));
  for (i = 0; i < n; i++) {
    float *q = buf + i * (size_t) ch;
    int c;
    for (c = 0; c < ch; c++)
      if ((update_mask >> c) & 1u) q[c] = map[scale_quantum_to_map(q[c])];
  }
  free(map);
  return 0;
}
