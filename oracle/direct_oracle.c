/*
  oracle/direct_oracle.c -- TEST INFRASTRUCTURE ONLY.  Never linked into, imported by or executed from the product.

  The plain-C oracle of the two "directly applied" morphology methods of ImageMagick 7.1.1-45 Q16-HDRI, Distance (21) and
  Voronoi (22): MorphologyApply's special branch (morphology.c:3736-3776) around MorphologyPrimitiveDirect (:3242-3623),
  restated loop for loop.  It uses the main oracle's kernel struct, pixel_intensity and clamp_pixel, which are file-local
  there, so this translation unit includes oracle.c.  Built by oracle/direct.mk into oracle/libdirect_oracle.so with the
  main oracle's flags (no contraction, standard excess precision); pinned bit for bit against the reference compiled from
  source by tests/test_oracle_direct_vs_ref.py.  Buffers as in oracle.h.

    int orc_morphology_direct(const float *src, float *dst, size_t w, size_t h, int ch, int method, const orc_kernel *k);

  `k` is the head of the kernel list (the only kernel MorphologyApply uses for these methods).  Returns the channel count
  of the result, or -1 on bad arguments.  The result has `ch` channels, except Voronoi on an image without alpha, whose
  result gains an alpha channel (ch + 1; dst must hold w*h*(ch+1) floats).  The result's alpha trait is the source's for
  Distance and CopyPixelTrait for Voronoi (:3766-3774).

  MorphologyPrimitiveDirect works in place on a clone of the source.  Every channel (alpha included) is swept on its own:
    pixel = QuantumRange; pixel = min(pixel, (double) sample + k) over the non-NaN kernel cells, a term replacing pixel only
    when it is strictly less; q = ClampToQuantum(pixel) (a float cast in HDRI).
  Forward pass (rows down, columns right), kernel reflected: ox = kw-kx-1, oy = kh-ky-1.
    1. The virtual region (edge virtual pixels) at columns x-ox .. x-ox+kw-1 of rows y-oy .. y (Voronoi: .. y-1), kernel
       index kw*kh-1 counting down.  It is read before row y is written: its row y holds the values the row had before the
       pass, the rows above are final.
    2. The live, updated values of the ox pixels to the left (x+u-ox >= 0), kernel index kw*(ky+1)-1 counting down.
  Reverse pass (rows up, columns left):
    1. Rows y .. y+ky of the forward result (row y before this pass, the rows below final), columns x-ox .. x-ox+kw-1,
       kernel index kw*(ky+1)-1 counting down.
    2. The live values of the pixels to the right (x+u-ox < columns), kernel index kw*ky+kx-1 (Voronoi: kw*(ky+1)-1)
       counting down.
  Voronoi then runs SetImageAlphaChannel(Deactivate), CompositeImage(result, source, CopyAlpha) and Deactivate again: the
  composite writes ClampPixel(QuantumRange*(QuantumScale*alpha)) of the source (its intensity when the source has no
  alpha) into the alpha channel and ClampPixel of the swept value into every other channel (composite.c:2606-2612,
  :2708-2709, :2860-2863, :3562).
*/
#include "oracle.c"

enum { ORC_DISTANCE = 21, ORC_VORONOI = 22 };

/* The value of channel i of the virtual pixel (xx, yy): edge virtual pixels clamp both coordinates. */
static double direct_virtual(const float *buf, const float *before, long y, long xx, long yy, long W, long H, int ch, int i)
{
  xx = clampl(xx, 0, W - 1);
  yy = clampl(yy, 0, H - 1);
  if (yy == y) return (double) before[(size_t) xx * ch + i];        /* the row as it was before this pass */
  return (double) buf[((size_t) yy * W + xx) * ch + i];
}

static void direct_forward(float *buf, float *before, long W, long H, int ch, int method, const orc_kernel *k, int sweep)
{
  const long kw = (long) k->width, kh = (long) k->height, ox = kw - k->x - 1, oy = kh - k->y - 1;
  const long rows = method == ORC_VORONOI ? oy : oy + 1;           /* :3371 v <= offset.y, :3402 v < offset.y */
  long x, y, u, v;
  int i;
  for (y = 0; y < H; y++) {
    float *q = buf + (size_t) y * W * ch;
    memcpy(before, q, (size_t) W * ch * sizeof(float));
    for (x = 0; x < W; x++)
      for (i = 0; i < sweep; i++) {
        double pixel = QR;
        const double *kv = k->values + kw * kh - 1;
        for (v = 0; v < rows; v++)
          for (u = 0; u < kw; u++, kv--) {
            if (!isnan(*kv)) {
              const double t = direct_virtual(buf, before, y, x - ox + u, y - oy + v, W, H, ch, i) + *kv;
              if (t < pixel) pixel = t;
            }
          }
        kv = k->values + kw * (k->y + 1) - 1;
        for (u = 0; u < ox; u++, kv--) {
          if (!isnan(*kv) && (x + u - ox) >= 0) {
            const double t = (double) q[(size_t) (x + u - ox) * ch + i] + *kv;
            if (t < pixel) pixel = t;
          }
        }
        q[(size_t) x * ch + i] = (float) pixel;
      }
  }
}

static void direct_reverse(float *buf, float *before, long W, long H, int ch, int method, const orc_kernel *k, int sweep)
{
  const long kw = (long) k->width, kh = (long) k->height, ox = kw - k->x - 1, oy = kh - k->y - 1;
  long x, y, u, v;
  int i;
  for (y = H - 1; y >= 0; y--) {
    float *q = buf + (size_t) y * W * ch;
    memcpy(before, q, (size_t) W * ch * sizeof(float));
    for (x = W - 1; x >= 0; x--)
      for (i = 0; i < sweep; i++) {
        double pixel = QR;
        const double *kv = k->values + kw * (k->y + 1) - 1;
        for (v = oy; v < kh; v++)
          for (u = 0; u < kw; u++, kv--) {
            if (!isnan(*kv)) {
              const double t = direct_virtual(buf, before, y, x - ox + u, y + v - oy, W, H, ch, i) + *kv;
              if (t < pixel) pixel = t;
            }
          }
        kv = method == ORC_VORONOI ? k->values + kw * (k->y + 1) - 1 : k->values + kw * k->y + k->x - 1;   /* :3580 */
        for (u = ox + 1; u < kw; u++, kv--) {
          if (!isnan(*kv) && (x + u - ox) < W) {
            const double t = (double) q[(size_t) (x + u - ox) * ch + i] + *kv;
            if (t < pixel) pixel = t;
          }
        }
        q[(size_t) x * ch + i] = (float) pixel;
      }
  }
}

int orc_morphology_direct(const float *src, float *dst, size_t w, size_t h, int ch, int method, const orc_kernel *k)
{
  const long W = (long) w, H = (long) h;
  const int has_alpha = ch == 2 || ch == 4;
  const size_t n = w * h;
  float *buf, *before;
  size_t p;
  int out_ch = ch, i;
  if (!src || !dst || !k || !k->values || w == 0 || h == 0 || ch < 1 || ch > 4) return -1;
  if (method != ORC_DISTANCE && method != ORC_VORONOI) return -1;
  if (k->x < 0 || k->y < 0 || k->x >= (long) k->width || k->y >= (long) k->height) return -1;
  buf = (float *) malloc(n * (size_t) ch * sizeof(float));
  before = (float *) malloc(w * (size_t) ch * sizeof(float));
  if (!buf || !before) { free(buf); free(before); return -1; }
  memcpy(buf, src, n * (size_t) ch * sizeof(float));                 /* CloneImage, :3749 */
  /* Every channel is swept; with Voronoi the source's alpha replaces the swept alpha below, so it is not swept. */
  direct_forward(buf, before, W, H, ch, method, k, method == ORC_VORONOI && has_alpha ? ch - 1 : ch);
  direct_reverse(buf, before, W, H, ch, method, k, method == ORC_VORONOI && has_alpha ? ch - 1 : ch);
  if (method == ORC_DISTANCE) {
    memcpy(dst, buf, n * (size_t) ch * sizeof(float));
  } else {
    out_ch = has_alpha ? ch : ch + 1;
    for (p = 0; p < n; p++) {
      const float *s = src + p * (size_t) ch, *b = buf + p * (size_t) ch;
      float *d = dst + p * (size_t) out_ch;
      const int colours = has_alpha ? ch - 1 : ch;
      for (i = 0; i < colours; i++) d[i] = clamp_pixel((double) b[i]);
      d[out_ch - 1] = clamp_pixel(has_alpha ? QR * (QS * (double) s[ch - 1]) : pixel_intensity(s, ch));
    }
  }
  free(buf);
  free(before);
  return out_ch;
}
