/*
  trim_harness.c -- end-to-end check of the GetImageBoundingBox and TrimImage wraps of the drop-in boundary (test
  infrastructure).

  Linked like shim_harness (the UNMODIFIED reference MagickCore, the shim and libmagickb200, ld --wrap): each case runs
  through the shim and through __real_X with the shim disabled, each with an exception of its own.  The boxes and the
  exceptions' severities must agree; the trimmed images must agree bit for bit, with the same size, page, type,
  colourspace, alpha trait and channel count.  Without a device every wrap must decline ("gpu hits 0"); with one, the
  served cases must hit the GPU and the declines must fall back.  Exit code 0 == no FAIL.
*/
#include "MagickCore/studio.h"
#include "MagickCore/MagickCore.h"
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

extern RectangleInfo __real_GetImageBoundingBox(const Image *, ExceptionInfo *);
extern Image *__real_TrimImage(const Image *, ExceptionInfo *);
extern MagickBooleanType __real_TransformImageColorspace(Image *, const ColorspaceType, ExceptionInfo *);
extern int mb200_device_count(void);
extern long B200ShimHits(void), B200ShimFallbacks(void);
extern void B200ShimEnable(int);

/* 0 when both images are the same: size, page, type, colourspace, alpha trait, channels and every pixel word. */
static int same_images(const Image *a, const Image *b, ExceptionInfo *ex)
{
  const Quantum *p, *q;
  if (a == (const Image *) NULL || b == (const Image *) NULL) return a != b;
  if (a->columns != b->columns || a->rows != b->rows || GetPixelChannels(a) != GetPixelChannels(b) ||
      a->page.width != b->page.width || a->page.height != b->page.height || a->page.x != b->page.x ||
      a->page.y != b->page.y || a->type != b->type || a->colorspace != b->colorspace || a->alpha_trait != b->alpha_trait)
    return 1;
  p = GetVirtualPixels(a, 0, 0, a->columns, a->rows, ex);
  q = GetVirtualPixels(b, 0, 0, b->columns, b->rows, ex);
  return p == (const Quantum *) NULL || q == (const Quantum *) NULL ||
         memcmp(p, q, a->columns * a->rows * GetPixelChannels(a) * sizeof(Quantum)) != 0;
}

/* The served / declined check of one call: with a device a served case must add a hit, a declined one a fallback. */
static int counted(int expect_fallback, long hits, long fallbacks)
{
  if (mb200_device_count() <= 0) return 0;
  if (expect_fallback) return B200ShimFallbacks() <= fallbacks;
  return B200ShimHits() <= hits;
}

static int box_case(const char *name, const Image *im, int expect_fallback)
{
  const long hits = B200ShimHits(), fb = B200ShimFallbacks();
  ExceptionInfo *ea = AcquireExceptionInfo(), *eb = AcquireExceptionInfo();
  RectangleInfo a, b;
  int bad;
  a = GetImageBoundingBox(im, ea);
  bad = counted(expect_fallback, hits, fb);
  B200ShimEnable(0);
  b = __real_GetImageBoundingBox(im, eb);
  B200ShimEnable(1);
  bad |= a.width != b.width || a.height != b.height || a.x != b.x || a.y != b.y || ea->severity != eb->severity;
  printf("%-52s box %lux%lu%+ld%+ld severity %d%s\n", name, (unsigned long) a.width, (unsigned long) a.height,
         (long) a.x, (long) a.y, (int) ea->severity, bad ? "  FAIL" : "");
  ea = DestroyExceptionInfo(ea); eb = DestroyExceptionInfo(eb);
  return bad;
}

static int trim_case(const char *name, const Image *im, int expect_fallback)
{
  const long hits = B200ShimHits(), fb = B200ShimFallbacks();
  ExceptionInfo *ea = AcquireExceptionInfo(), *eb = AcquireExceptionInfo();
  Image *a, *b;
  int bad;
  a = TrimImage(im, ea);
  bad = counted(expect_fallback, hits, fb);
  B200ShimEnable(0);
  b = __real_TrimImage(im, eb);
  B200ShimEnable(1);
  bad |= same_images(a, b, ea) || ea->severity != eb->severity;
  printf("%-52s %s %lux%lu%+ld%+ld ch %d severity %d%s\n", name, a ? "image" : "none",
         a ? (unsigned long) a->columns : 0UL, a ? (unsigned long) a->rows : 0UL, a ? (long) a->page.x : 0L,
         a ? (long) a->page.y : 0L, a ? (int) GetPixelChannels(a) : 0, (int) ea->severity, bad ? "  FAIL" : "");
  if (a) a = DestroyImage(a);
  if (b) b = DestroyImage(b);
  ea = DestroyExceptionInfo(ea); eb = DestroyExceptionInfo(eb);
  return bad;
}

/* A framed object: noise inside [w/5, w - w/4) x [h/6, h - h/3) on a flat background; `corners` makes the four corner
   pixels differ from it and from each other. */
static Image *framed_image(size_t w, size_t h, MagickBooleanType alpha, int corners, ExceptionInfo *ex)
{
  ImageInfo *info = AcquireImageInfo();
  Image *im = AcquireImage(info, ex);
  Quantum *q;
  size_t x, y, c, n;
  unsigned long long s = 88172645463325252ULL ^ (w * 131 + h);
  info = DestroyImageInfo(info);
  (void) SetImageExtent(im, w, h, ex);
  if (alpha) im->alpha_trait = BlendPixelTrait;
  (void) SetImageStorageClass(im, DirectClass, ex);
  (void) SetImageColorspace(im, sRGBColorspace, ex);
  (void) strcpy(im->filename, "framed");
  q = GetAuthenticPixels(im, 0, 0, w, h, ex);
  n = GetPixelChannels(im);
  for (y = 0; y < h; y++)
    for (x = 0; x < w; x++)
      for (c = 0; c < n; c++) {
        Quantum *v = q + (y * w + x) * n + c;
        *v = (Quantum) (c == 3 ? 65535.0 : 1000.0 + 20000.0 * c);
        if (x >= w / 5 && x < w - w / 4 && y >= h / 6 && y < h - h / 3) {
          s ^= s << 13; s ^= s >> 7; s ^= s << 17;
          *v = (Quantum) ((s >> 40) * (65535.0 / 16777215.0));
        }
      }
  if (corners) {
    const size_t at[4] = { 0, w - 1, (h - 1) * w, (h - 1) * w + w - 1 };
    for (c = 0; c < 4; c++) q[at[c] * n] = (Quantum) (7000.0 + 3000.0 * c);
  }
  (void) SyncAuthenticPixels(im, ex);
  return im;
}

int main(void)
{
  ExceptionInfo *ex;
  Image *rgba, *rgb, *corners, *gray, *canvas, *uniform, *palette, *cmyk, *profiled;
  int failures = 0;
  MagickCoreGenesis("trim_harness", MagickFalse);
  /* one thread: with several, the reference's box of an image of 512 rows or more whose bottom corners differ depends on
     the OpenMP schedule (attribute.c:484-535); the library gives the single-threaded result */
  (void) SetMagickResourceLimit(ThreadResource, 1);
  ex = AcquireExceptionInfo();
  rgba = framed_image(517, 389, MagickTrue, 0, ex);
  rgb = framed_image(300, 200, MagickFalse, 0, ex);
  corners = framed_image(300, 600, MagickFalse, 1, ex);
  gray = framed_image(97, 61, MagickFalse, 0, ex);
  B200ShimEnable(0); (void) __real_TransformImageColorspace(gray, GRAYColorspace, ex); B200ShimEnable(1);
  gray->type = GrayscaleType;
  canvas = framed_image(70, 45, MagickTrue, 0, ex);
  canvas->page.width = 200; canvas->page.height = 150; canvas->page.x = 20; canvas->page.y = 30;
  uniform = framed_image(40, 30, MagickTrue, 0, ex);
  (void) SetImageBackgroundColor(uniform, ex);
  palette = framed_image(64, 48, MagickFalse, 0, ex);
  (void) SetImageType(palette, PaletteType, ex);
  cmyk = framed_image(64, 48, MagickFalse, 0, ex);
  B200ShimEnable(0); (void) __real_TransformImageColorspace(cmyk, CMYKColorspace, ex); B200ShimEnable(1);
  profiled = framed_image(64, 48, MagickTrue, 0, ex);
  {
    StringInfo *profile = StringToStringInfo("8BIM");
    (void) SetImageProfile(profiled, "8bim", profile, ex);
    profile = DestroyStringInfo(profile);
  }

  {
    Image *images[] = { rgba, rgb, corners, gray, canvas };
    const char *names[] = { "RGBA", "RGB", "RGB 300x600 four corners", "gray", "RGBA canvas 200x150+20+30" };
    static const char *const gravities[] = { "NorthWest", "North", "NorthEast", "West", "Center", "East", "SouthWest",
                                             "South", "SouthEast" };
    char name[160];
    size_t i, k;
    for (i = 0; i < 5; i++) {
      Image *im = images[i];
      (void) snprintf(name, sizeof(name), "GetImageBoundingBox %s", names[i]);
      failures += box_case(name, im, 0);
      (void) snprintf(name, sizeof(name), "TrimImage %s", names[i]);
      failures += trim_case(name, im, 0);
      im->fuzz = 0.3 * 65535.0;
      (void) snprintf(name, sizeof(name), "GetImageBoundingBox %s fuzz 30%%", names[i]);
      failures += box_case(name, im, 0);
      (void) snprintf(name, sizeof(name), "TrimImage %s fuzz 30%%", names[i]);
      failures += trim_case(name, im, 0);
      im->fuzz = 0.0;
      (void) SetImageArtifact(im, "trim:edges", "North,west,bogus");
      (void) snprintf(name, sizeof(name), "GetImageBoundingBox %s trim:edges North,west,bogus", names[i]);
      failures += box_case(name, im, 0);
      (void) snprintf(name, sizeof(name), "TrimImage %s trim:edges North,west,bogus", names[i]);
      failures += trim_case(name, im, 0);
      (void) DeleteImageArtifact(im, "trim:edges");
      (void) SetImageArtifact(im, "trim:minSize", "400x300");
      for (k = 0; k < sizeof(gravities) / sizeof(gravities[0]); k++) {
        im->gravity = (GravityType) (k + 1);
        (void) snprintf(name, sizeof(name), "TrimImage %s minSize 400x300 %s", names[i], gravities[k]);
        failures += trim_case(name, im, 0);
      }
      im->gravity = UndefinedGravity;
      (void) DeleteImageArtifact(im, "trim:minSize");
    }
  }
  /* the zero box: the warning, and TrimImage's transparent 1x1 clone (served: the scan ran, no pixel is read after) */
  failures += box_case("GetImageBoundingBox uniform (zero box)", uniform, 0);
  failures += trim_case("TrimImage uniform (zero box)", uniform, 0);
  rgb->fuzz = 1.0e12;
  failures += box_case("GetImageBoundingBox RGB huge fuzz (zero box)", rgb, 0);
  failures += trim_case("TrimImage RGB huge fuzz (zero box)", rgb, 0);
  rgb->fuzz = 0.0;
  /* the declines */
  (void) SetImageArtifact(rgba, "trim:percent-background", "50");
  failures += box_case("fallback: GetImageBoundingBox percent-background", rgba, 1);
  failures += trim_case("fallback: TrimImage percent-background", rgba, 1);
  (void) DeleteImageArtifact(rgba, "trim:percent-background");
  failures += box_case("fallback: GetImageBoundingBox PseudoClass", palette, 1);
  failures += trim_case("fallback: TrimImage PseudoClass", palette, 1);
  failures += box_case("fallback: GetImageBoundingBox CMYK", cmyk, 1);
  failures += trim_case("fallback: TrimImage CMYK", cmyk, 1);
  failures += box_case("GetImageBoundingBox 8bim profile", profiled, 0);
  failures += trim_case("fallback: TrimImage 8bim profile", profiled, 1);

  printf("gpu hits %ld, fallbacks %ld, failures %d\n", B200ShimHits(), B200ShimFallbacks(), failures);
  rgba = DestroyImage(rgba); rgb = DestroyImage(rgb); corners = DestroyImage(corners); gray = DestroyImage(gray);
  canvas = DestroyImage(canvas); uniform = DestroyImage(uniform); palette = DestroyImage(palette);
  cmyk = DestroyImage(cmyk); profiled = DestroyImage(profiled);
  ex = DestroyExceptionInfo(ex);
  MagickCoreTerminus();
  return failures != 0;
}
