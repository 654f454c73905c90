/*
  oracle/layout_oracle.c -- TEST INFRASTRUCTURE ONLY.  Never linked into, imported by or executed from the product.

  The plain-C oracle of TransformImageColorspace (colorspace.c:1751) for the colourspaces that change the channel
  layout of the pixel cache -- GRAY, LinearGRAY and CMYK -- restated in the reference's operation order on top of the
  main oracle: its gamma curves (decode_pixel_gamma / encode_pixel_gamma), its PerceptibleReciprocal and, for every
  other space on either side of sRGB, orc_colorspace_ex itself.  Those are file-local there, so this translation unit
  includes oracle.c rather than carrying a second copy of them.  Built by oracle/layout.mk into
  oracle/liblayout_oracle.so with the main oracle's flags (no contraction, standard excess precision); pinned bit for
  bit against the reference compiled from source by tests/test_oracle_layout_vs_ref.py.

    int orc_colorspace_channels(int colorspace, int has_alpha);
        GRAY / LinearGRAY 1, CMYK 4, every other space 3; plus one for alpha
    int orc_colorspace_layout(const float *src, int src_ch, float *dst, int dst_ch, size_t w, size_t h, int from,
                              int to, const orc_colorspace_options *options);
        `src` (w x h x src_ch, tagged `from`) -> `dst` (w x h x dst_ch, tagged `to`); src is not written.
        0, or -1 for channel counts off the layout rule and for a space the main oracle does not serve.

  The legs (the reference's pixel loops):
    sRGB -> GRAY        :901-957    gray = 0.212656 R + 0.715158 G + 0.072186 B into channel 0, then the cache keeps gray
                                    (and alpha)
    sRGB -> LinearGRAY  :843-900    the same sum of DecodePixelGamma of each channel
    GRAY -> sRGB        :2224-2291  SetImageColorspace(sRGB) first (R = G = B = gray), then the same sum into all three
    LinearGRAY -> sRGB  :2171-2223  ... of EncodePixelGamma of each channel
    sRGB -> CMYK        :778-842    SetImageColorspace(CMYK) first, so ConvertRGBToCMYK sees a CMYK-tagged pixel and
                                    takes its linear branch (colorspace-private.h:1600-1611); K starts at 0
    CMYK -> sRGB        :2110-2170  ConvertCMYKToRGB (colorspace-private.h:131-139) on the CMYK layout, then the cache
                                    drops K
  Every other pair goes through sRGB (colorspace.c:1770-1781).  ClampToQuantum (HDRI) is a float cast; alpha is copied.
*/
#include "oracle.c"

#define ORC_CS_CMYK 2
#define ORC_CS_GRAY 3
#define ORC_CS_LINEAR_GRAY 33

static int is_layout_space(int cs) { return cs == ORC_CS_CMYK || cs == ORC_CS_GRAY || cs == ORC_CS_LINEAR_GRAY; }

int orc_colorspace_channels(int colorspace, int has_alpha)
{
  const int base = colorspace == ORC_CS_CMYK ? 4 : (colorspace == ORC_CS_GRAY || colorspace == ORC_CS_LINEAR_GRAY) ? 1 : 3;
  return base + (has_alpha != 0);
}

/* GRAY / LinearGRAY (g channels: gray[, alpha]) -> sRGB (3 + alpha) */
static void gray_to_srgb(const float *src, int src_ch, float *dst, int dst_ch, long n, int linear)
{
  long i;
#pragma omp parallel for schedule(static)
  for (i = 0; i < n; i++) {
    const float *p = src + (size_t) i * src_ch;
    float *q = dst + (size_t) i * dst_ch;
    const double red = (double) p[0], green = (double) p[0], blue = (double) p[0];
    double gray;
    if (linear)
      gray = 0.212656 * encode_pixel_gamma(red) + 0.715158 * encode_pixel_gamma(green) + 0.072186 * encode_pixel_gamma(blue);
    else
      gray = 0.212656 * red + 0.715158 * green + 0.072186 * blue;
    q[0] = (float) gray; q[1] = (float) gray; q[2] = (float) gray;
    if (dst_ch == 4) q[3] = p[1];
  }
}

/* sRGB (3 + alpha) -> GRAY / LinearGRAY (1 + alpha) */
static void srgb_to_gray(const float *src, int src_ch, float *dst, int dst_ch, long n, int linear)
{
  long i;
#pragma omp parallel for schedule(static)
  for (i = 0; i < n; i++) {
    const float *p = src + (size_t) i * src_ch;
    float *q = dst + (size_t) i * dst_ch;
    double gray;
    if (linear)
      gray = 0.212656 * decode_pixel_gamma((double) p[0]) + 0.715158 * decode_pixel_gamma((double) p[1]) +
             0.072186 * decode_pixel_gamma((double) p[2]);
    else
      gray = 0.212656 * (double) p[0] + 0.715158 * (double) p[1] + 0.072186 * (double) p[2];
    q[0] = (float) gray;
    if (dst_ch == 2) q[1] = p[3];
  }
}

/* sRGB (3 + alpha) -> CMYK (4 + alpha): ConvertRGBToCMYK's linear branch, SetPixelViaPixelInfo */
static void srgb_to_cmyk(const float *src, int src_ch, float *dst, int dst_ch, long n)
{
  long i;
#pragma omp parallel for schedule(static)
  for (i = 0; i < n; i++) {
    const float *p = src + (size_t) i * src_ch;
    float *q = dst + (size_t) i * dst_ch;
    const double red = QS * (double) p[0], green = QS * (double) p[1], blue = QS * (double) p[2];
    if ((fabs(red) < EPS) && (fabs(green) < EPS) && (fabs(blue) < EPS)) {
      q[0] = p[0]; q[1] = p[1]; q[2] = p[2]; q[3] = (float) QR;
    } else {
      double cyan = 1.0 - red, magenta = 1.0 - green, yellow = 1.0 - blue, black = cyan;
      if (magenta < black) black = magenta;
      if (yellow < black) black = yellow;
      cyan = perceptible_reciprocal(1.0 - black) * (cyan - black);
      magenta = perceptible_reciprocal(1.0 - black) * (magenta - black);
      yellow = perceptible_reciprocal(1.0 - black) * (yellow - black);
      q[0] = (float) (QR * cyan); q[1] = (float) (QR * magenta); q[2] = (float) (QR * yellow); q[3] = (float) (QR * black);
    }
    if (dst_ch == 5) q[4] = p[3];
  }
}

/* CMYK (4 + alpha) -> sRGB (3 + alpha): ConvertCMYKToRGB */
static void cmyk_to_srgb(const float *src, int src_ch, float *dst, int dst_ch, long n)
{
  long i;
#pragma omp parallel for schedule(static)
  for (i = 0; i < n; i++) {
    const float *p = src + (size_t) i * src_ch;
    float *q = dst + (size_t) i * dst_ch;
    const double black = (double) p[3];
    int c;
    for (c = 0; c < 3; c++) q[c] = (float) (QR - (QS * (double) p[c] * (QR - black) + black));
    if (dst_ch == 4) q[3] = p[4];
  }
}

int orc_colorspace_layout(const float *src, int src_ch, float *dst, int dst_ch, size_t w, size_t h, int from, int to,
                          const orc_colorspace_options *options)
{
  const long n = (long) (w * h);
  const int alpha = src_ch - orc_colorspace_channels(from, 0);
  const int rgb_ch = 3 + alpha;
  float *tmp;
  int rc = 0;
  if ((alpha != 0 && alpha != 1) || dst_ch != orc_colorspace_channels(to, alpha)) return -1;
  if (from == to) {
    memcpy(dst, src, (size_t) n * (size_t) src_ch * sizeof(float));
    return 0;
  }
  tmp = (float *) malloc((size_t) (n > 0 ? n : 1) * (size_t) rgb_ch * sizeof(float));
  if (tmp == NULL) return -1;
  /* back to sRGB (TransformsRGBImage) */
  if (from == ORC_CS_GRAY || from == ORC_CS_LINEAR_GRAY) gray_to_srgb(src, src_ch, tmp, rgb_ch, n, from == ORC_CS_LINEAR_GRAY);
  else if (from == ORC_CS_CMYK) cmyk_to_srgb(src, src_ch, tmp, rgb_ch, n);
  else {
    memcpy(tmp, src, (size_t) n * (size_t) rgb_ch * sizeof(float));
    if (from != ORC_CS_SRGB) rc = orc_colorspace_ex(tmp, w, h, rgb_ch, from, ORC_CS_SRGB, options);
  }
  /* ... and forward (sRGBTransformImage) */
  if (rc == 0) {
    if (to == ORC_CS_GRAY || to == ORC_CS_LINEAR_GRAY) srgb_to_gray(tmp, rgb_ch, dst, dst_ch, n, to == ORC_CS_LINEAR_GRAY);
    else if (to == ORC_CS_CMYK) srgb_to_cmyk(tmp, rgb_ch, dst, dst_ch, n);
    else if (to != ORC_CS_SRGB && !is_layout_space(to)) {
      float *out = (float *) malloc((size_t) (n > 0 ? n : 1) * (size_t) rgb_ch * sizeof(float));
      rc = out == NULL ? -1 : 0;
      if (rc == 0) {
        memcpy(out, tmp, (size_t) n * (size_t) rgb_ch * sizeof(float));
        rc = orc_colorspace_ex(out, w, h, rgb_ch, ORC_CS_SRGB, to, options);
        if (rc == 0) memcpy(dst, out, (size_t) n * (size_t) rgb_ch * sizeof(float));
        free(out);
      }
    } else memcpy(dst, tmp, (size_t) n * (size_t) rgb_ch * sizeof(float));
  }
  free(tmp);
  return rc;
}
