/*
  geometry_harness.c -- end-to-end check of the orientation and crop wraps of the drop-in boundary (test infrastructure).

  Linked like shim_harness (the UNMODIFIED reference MagickCore, the shim and libmagickb200, ld --wrap): each wrapped
  entry point -- FlipImage, FlopImage, TransposeImage, TransverseImage, IntegralRotateImage, CropImage, CropImageToTiles,
  ShaveImage, RollImage, AutoOrientImage -- is called through the shim and through __real_X with the shim disabled.
  Every image of the results must agree bit for bit, with the same size, page, type, orientation and channel count.  A
  ResizeImage -> CropImageToTiles -> FlopImage -> BlurImage chain is compared both ways within the ULP bar of the blur and
  resize kernels.  Without a device every wrap must decline ("gpu hits 0"); with one, the served cases must hit the GPU
  and the declines must fall back.  Exit code 0 == no FAIL.
*/
#include "MagickCore/studio.h"
#include "MagickCore/MagickCore.h"
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

extern Image *__real_FlipImage(const Image *, ExceptionInfo *);
extern Image *__real_FlopImage(const Image *, ExceptionInfo *);
extern Image *__real_TransposeImage(const Image *, ExceptionInfo *);
extern Image *__real_TransverseImage(const Image *, ExceptionInfo *);
extern Image *__real_IntegralRotateImage(const Image *, size_t, ExceptionInfo *);
extern Image *__real_CropImage(const Image *, const RectangleInfo *, ExceptionInfo *);
extern Image *__real_CropImageToTiles(const Image *, const char *, ExceptionInfo *);
extern Image *__real_ShaveImage(const Image *, const RectangleInfo *, ExceptionInfo *);
extern Image *__real_RollImage(const Image *, const ssize_t, const ssize_t, ExceptionInfo *);
extern Image *__real_AutoOrientImage(const Image *, const OrientationType, ExceptionInfo *);
extern Image *__real_RotateImage(const Image *, const double, ExceptionInfo *);
extern MagickBooleanType __real_TransformImageColorspace(Image *, const ColorspaceType, ExceptionInfo *);
extern int mb200_device_count(void);
extern long B200ShimHits(void), B200ShimFallbacks(void);
extern void B200ShimEnable(int);

enum { FLIP, FLOP, TRANSPOSE, TRANSVERSE, INTEGRAL_ROTATE, CROP, TILES, SHAVE, ROLL, AUTO_ORIENT, ROTATE };

typedef struct { int op; long a, b, c, d; const char *text; } op_args;

static Image *run(const Image *im, const op_args *o, int real, ExceptionInfo *ex)
{
  RectangleInfo r;
  r.width = (size_t) o->a; r.height = (size_t) o->b; r.x = o->c; r.y = o->d;
  switch (o->op) {
    case FLIP: return real ? __real_FlipImage(im, ex) : FlipImage(im, ex);
    case FLOP: return real ? __real_FlopImage(im, ex) : FlopImage(im, ex);
    case TRANSPOSE: return real ? __real_TransposeImage(im, ex) : TransposeImage(im, ex);
    case TRANSVERSE: return real ? __real_TransverseImage(im, ex) : TransverseImage(im, ex);
    case INTEGRAL_ROTATE: return real ? __real_IntegralRotateImage(im, (size_t) o->a, ex) : IntegralRotateImage(im, (size_t) o->a, ex);
    case CROP: return real ? __real_CropImage(im, &r, ex) : CropImage(im, &r, ex);
    case TILES: return real ? __real_CropImageToTiles(im, o->text, ex) : CropImageToTiles(im, o->text, ex);
    case SHAVE: return real ? __real_ShaveImage(im, &r, ex) : ShaveImage(im, &r, ex);
    case ROLL: return real ? __real_RollImage(im, (ssize_t) o->a, (ssize_t) o->b, ex) : RollImage(im, (ssize_t) o->a, (ssize_t) o->b, ex);
    case AUTO_ORIENT: return real ? __real_AutoOrientImage(im, (OrientationType) o->a, ex) : AutoOrientImage(im, (OrientationType) o->a, ex);
    default: return real ? __real_RotateImage(im, (double) o->a, ex) : RotateImage(im, (double) o->a, ex);
  }
}

/* 0 when both lists hold the same images: size, page, type, orientation, channels and every pixel word. */
static int same_lists(const Image *a, const Image *b, ExceptionInfo *ex)
{
  for (; a != (const Image *) NULL && b != (const Image *) NULL; a = GetNextImageInList(a), b = GetNextImageInList(b)) {
    const size_t n = a->columns * a->rows * GetPixelChannels(a);
    const Quantum *p, *q;
    if (a->columns != b->columns || a->rows != b->rows || GetPixelChannels(a) != GetPixelChannels(b) ||
        a->page.width != b->page.width || a->page.height != b->page.height || a->page.x != b->page.x ||
        a->page.y != b->page.y || a->type != b->type || a->orientation != b->orientation ||
        a->colorspace != b->colorspace || a->alpha_trait != b->alpha_trait)
      return 1;
    p = GetVirtualPixels(a, 0, 0, a->columns, a->rows, ex);
    q = GetVirtualPixels(b, 0, 0, b->columns, b->rows, ex);
    if (p == (const Quantum *) NULL || q == (const Quantum *) NULL || memcmp(p, q, n * sizeof(Quantum)) != 0) return 1;
  }
  return a != b;                                     /* both lists ended together (or both are empty) */
}

/* One case through the shim and through __real_: 1 on failure.  expect_fallback: the shim must decline. */
static int geometry_case(const char *name, const Image *src, op_args o, int expect_fallback, ExceptionInfo *ex)
{
  const long hits = B200ShimHits(), fb = B200ShimFallbacks();
  Image *a, *b;
  int bad;
  a = run(src, &o, 0, ex);
  B200ShimEnable(0);
  b = run(src, &o, 1, ex);
  B200ShimEnable(1);
  bad = same_lists(a, b, ex);
  if (mb200_device_count() > 0) {
    if (expect_fallback && B200ShimFallbacks() <= fb) bad = 1;
    if (!expect_fallback && B200ShimHits() <= hits) bad = 1;
  }
  printf("%-44s %s %lux%lu%+ld%+ld%s\n", name, a ? "image" : "none", a ? (unsigned long) a->columns : 0UL,
         a ? (unsigned long) a->rows : 0UL, a ? (long) a->page.x : 0L, a ? (long) a->page.y : 0L, bad ? "  FAIL" : "");
  if (a) a = DestroyImageList(a);
  if (b) b = DestroyImageList(b);
  return bad;
}

static Image *noise_image(size_t w, size_t h, MagickBooleanType alpha, ExceptionInfo *ex)
{
  ImageInfo *info = AcquireImageInfo();
  Image *im = AcquireImage(info, ex);
  Quantum *q;
  size_t i, n;
  unsigned long long s = 88172645463325252ULL ^ (w * 131 + h);
  info = DestroyImageInfo(info);
  (void) SetImageExtent(im, w, h, ex);
  if (alpha) im->alpha_trait = BlendPixelTrait;
  (void) SetImageStorageClass(im, DirectClass, ex);
  (void) SetImageColorspace(im, sRGBColorspace, ex);
  q = GetAuthenticPixels(im, 0, 0, w, h, ex);
  n = w * h * GetPixelChannels(im);
  for (i = 0; i < n; i++) { s ^= s << 13; s ^= s >> 7; s ^= s << 17; q[i] = (Quantum) ((s >> 40) * (65535.0 / 16777215.0)); }
  (void) SyncAuthenticPixels(im, ex);
  return im;
}

static long max_ulp(const Image *a, const Image *b, ExceptionInfo *ex)
{
  const Quantum *p, *q;
  size_t i, n;
  long worst = 0;
  if (!a || !b || a->columns != b->columns || a->rows != b->rows || GetPixelChannels(a) != GetPixelChannels(b))
    return 1L << 40;
  n = a->columns * a->rows * GetPixelChannels(a);
  p = GetVirtualPixels(a, 0, 0, a->columns, a->rows, ex);
  q = GetVirtualPixels(b, 0, 0, b->columns, b->rows, ex);
  for (i = 0; i < n; i++) {
    int ia, ib;
    float fa = (float) p[i], fb = (float) q[i];
    long d;
    memcpy(&ia, &fa, 4); memcpy(&ib, &fb, 4);
    if (ia < 0) ia = -(ia & 0x7fffffff);
    if (ib < 0) ib = -(ib & 0x7fffffff);
    d = labs((long) ia - (long) ib);
    if (d > worst) worst = d;
  }
  return worst;
}

/* ResizeImage -> CropImageToTiles -> FlopImage -> BlurImage with the shim on and with it off (every step on the CPU). */
static Image *chain(const Image *src, ExceptionInfo *ex)
{
  Image *r = ResizeImage(src, 400, 300, LanczosFilter, ex), *c, *f, *b;
  c = CropImageToTiles(r, "320x240+40+30", ex);
  f = FlopImage(c, ex);
  b = BlurImage(f, 0.0, 2.0, ex);
  r = DestroyImage(r); c = DestroyImageList(c); f = DestroyImage(f);
  return b;
}

int main(void)
{
  ExceptionInfo *ex;
  Image *rgba, *rgb, *gray, *paged, *canvas, *palette, *a, *b;
  int failures = 0, i;
  long d;
  MagickCoreGenesis("geometry_harness", MagickFalse);
  ex = AcquireExceptionInfo();
  rgba = noise_image(517, 389, MagickTrue, ex);
  rgb = noise_image(300, 200, MagickFalse, ex);
  gray = noise_image(97, 61, MagickFalse, ex);
  B200ShimEnable(0); (void) __real_TransformImageColorspace(gray, GRAYColorspace, ex); B200ShimEnable(1);
  gray->type = GrayscaleType;
  paged = noise_image(70, 45, MagickTrue, ex);
  paged->page.x = 7; paged->page.y = -3;
  canvas = noise_image(70, 45, MagickFalse, ex);
  canvas->page.width = 200; canvas->page.height = 150; canvas->page.x = 20; canvas->page.y = 30;
  palette = noise_image(64, 48, MagickFalse, ex);
  (void) SetImageType(palette, PaletteType, ex);

  {
    const Image *images[] = { rgba, rgb, gray, paged, canvas };
    const char *names[] = { "RGBA", "RGB", "gray", "RGBA page +7-3", "RGB canvas 200x150+20+30" };
    char name[128];
    for (i = 0; i < 5; i++) {
      const Image *im = images[i];
      const op_args ops[] = {
        { FLIP, 0, 0, 0, 0, NULL }, { FLOP, 0, 0, 0, 0, NULL }, { TRANSPOSE, 0, 0, 0, 0, NULL },
        { TRANSVERSE, 0, 0, 0, 0, NULL }, { INTEGRAL_ROTATE, 1, 0, 0, 0, NULL }, { INTEGRAL_ROTATE, 2, 0, 0, 0, NULL },
        { INTEGRAL_ROTATE, 3, 0, 0, 0, NULL }, { CROP, 40, 30, 10, 5, NULL }, { CROP, 60, 50, -3, -2, NULL },
        { SHAVE, 5, 3, 0, 0, NULL }, { ROLL, -13, 1000, 0, 0, NULL } };
      const char *op_names[] = { "FlipImage", "FlopImage", "TransposeImage", "TransverseImage", "IntegralRotateImage 1",
        "IntegralRotateImage 2", "IntegralRotateImage 3", "CropImage 40x30+10+5", "CropImage 60x50-3-2",
        "ShaveImage 5x3", "RollImage -13+1000" };
      size_t k;
      for (k = 0; k < sizeof(ops) / sizeof(ops[0]); k++) {
        (void) snprintf(name, sizeof(name), "%s %s", op_names[k], names[i]);
        failures += geometry_case(name, im, ops[k], 0, ex);
      }
      for (k = 2; k <= 8; k++) {
        const op_args o = { AUTO_ORIENT, (long) k, 0, 0, 0, NULL };
        (void) snprintf(name, sizeof(name), "AutoOrientImage %d %s", (int) k, names[i]);
        failures += geometry_case(name, im, o, 0, ex);
      }
    }
  }
  {
    /* CropImageToTiles: a region, an offset only, `!`, percent, fixed-size tiles (on the canvas image some of those
       tiles lie outside the image, where the reference makes 1x1 images: the loop declines), a gravity; `@` and the
       final clone decline */
    static const char *const served[] = { "100x80+10+20", "+10+20", "100x80+10+20!", "60%x80%+3+4" };
    static const char *const tiles[] = { "100x80", "120x100" };
    static const char *const declined[] = { "2x2@", "600x400" };
    char name[128];
    size_t k;
    for (k = 0; k < sizeof(served) / sizeof(served[0]); k++) {
      const op_args o = { TILES, 0, 0, 0, 0, served[k] };
      (void) snprintf(name, sizeof(name), "CropImageToTiles %s RGBA", served[k]);
      failures += geometry_case(name, rgba, o, 0, ex);
      (void) snprintf(name, sizeof(name), "CropImageToTiles %s canvas", served[k]);
      failures += geometry_case(name, canvas, o, 0, ex);
    }
    for (k = 0; k < sizeof(tiles) / sizeof(tiles[0]); k++) {
      const op_args o = { TILES, 0, 0, 0, 0, tiles[k] };
      (void) snprintf(name, sizeof(name), "CropImageToTiles %s RGBA", tiles[k]);
      failures += geometry_case(name, rgba, o, 0, ex);
      (void) snprintf(name, sizeof(name), "fallback: CropImageToTiles %s canvas", tiles[k]);
      failures += geometry_case(name, canvas, o, 1, ex);
    }
    for (k = 0; k < sizeof(declined) / sizeof(declined[0]); k++) {
      const op_args o = { TILES, 0, 0, 0, 0, declined[k] };
      (void) snprintf(name, sizeof(name), "fallback: CropImageToTiles %s", declined[k]);
      failures += geometry_case(name, rgba, o, 1, ex);
    }
    rgb->gravity = CenterGravity;
    {
      const op_args o = { TILES, 0, 0, 0, 0, "100x80+5+5" };
      failures += geometry_case("CropImageToTiles 100x80+5+5 -gravity center", rgb, o, 0, ex);
    }
    rgb->gravity = UndefinedGravity;
  }
  {
    const op_args outside = { CROP, 10, 10, 400, 10, NULL }, zero = { CROP, 10, 10, 300, 10, NULL };
    const op_args shave = { SHAVE, 150, 2, 0, 0, NULL }, rot0 = { INTEGRAL_ROTATE, 4, 0, 0, 0, NULL };
    const op_args top_left = { AUTO_ORIENT, TopLeftOrientation, 0, 0, 0, NULL }, flip = { FLIP, 0, 0, 0, 0, NULL };
    const op_args rot90 = { ROTATE, 90, 0, 0, 0, NULL }, rot180 = { ROTATE, 180, 0, 0, 0, NULL };
    failures += geometry_case("fallback: CropImage outside the canvas", rgb, outside, 1, ex);
    failures += geometry_case("fallback: CropImage zero area", rgb, zero, 1, ex);
    failures += geometry_case("fallback: ShaveImage half the width", rgb, shave, 1, ex);
    failures += geometry_case("fallback: IntegralRotateImage 4", rgb, rot0, 1, ex);
    failures += geometry_case("fallback: AutoOrientImage TopLeft", rgb, top_left, 1, ex);
    failures += geometry_case("fallback: FlipImage PseudoClass", palette, flip, 1, ex);
    /* RotateImage declines integral angles; its own call to IntegralRotateImage crosses objects and is served */
    failures += geometry_case("RotateImage 90 (IntegralRotateImage 1)", rgba, rot90, 0, ex);
    failures += geometry_case("RotateImage 180 (IntegralRotateImage 2)", rgb, rot180, 0, ex);
  }
  a = chain(rgba, ex);
  B200ShimEnable(0); b = chain(rgba, ex); B200ShimEnable(1);
  d = max_ulp(a, b, ex);
  printf("%-44s max ULP %ld (bar 4)%s\n", "chain Resize -> CropToTiles -> Flop -> Blur", d, d <= 4 ? "" : "  FAIL");
  if (d > 4) failures++;
  if (a) a = DestroyImage(a);
  if (b) b = DestroyImage(b);

  printf("gpu hits %ld, fallbacks %ld, failures %d\n", B200ShimHits(), B200ShimFallbacks(), failures);
  rgba = DestroyImage(rgba); rgb = DestroyImage(rgb); gray = DestroyImage(gray); paged = DestroyImage(paged);
  canvas = DestroyImage(canvas); palette = DestroyImage(palette);
  ex = DestroyExceptionInfo(ex);
  MagickCoreTerminus();
  return failures != 0;
}
