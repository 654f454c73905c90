/*
  shim_harness.c -- end-to-end check of the drop-in boundary (test infrastructure).

  Linked with the UNMODIFIED reference MagickCore (oracle/_ref/libMagickCoreRef.a), the shim and
  libmagickb200 using ld --wrap: every call below enters through ImageMagick's own exported entry
  point, is served by the GPU, and is compared against __real_X (the stock CPU path) on the same
  Image.  Exit code 0 == all within the parity bar and every operator actually hit the GPU path.
*/
#include "MagickCore/studio.h"
#include "MagickCore/MagickCore.h"
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>

extern Image *__real_BlurImage(const Image *, const double, const double, ExceptionInfo *);
extern Image *__real_GaussianBlurImage(const Image *, const double, const double, ExceptionInfo *);
extern Image *__real_UnsharpMaskImage(const Image *, const double, const double, const double, const double, ExceptionInfo *);
extern Image *__real_MorphologyImage(const Image *, const MorphologyMethod, const ssize_t, const KernelInfo *, ExceptionInfo *);
extern Image *__real_ResizeImage(const Image *, const size_t, const size_t, const FilterType, ExceptionInfo *);
extern MagickBooleanType __real_TransformImageColorspace(Image *, const ColorspaceType, ExceptionInfo *);
extern MagickBooleanType __real_ContrastImage(Image *, const MagickBooleanType, ExceptionInfo *);
extern MagickBooleanType __real_ModulateImage(Image *, const char *, ExceptionInfo *);
extern MagickBooleanType __real_GrayscaleImage(Image *, const PixelIntensityMethod, ExceptionInfo *);
extern MagickBooleanType __real_FunctionImage(Image *, const MagickFunction, const size_t, const double *, ExceptionInfo *);
extern Image *__real_SampleImage(const Image *, const size_t, const size_t, ExceptionInfo *);
extern Image *__real_ScaleImage(const Image *, const size_t, const size_t, ExceptionInfo *);
extern Image *__real_ThumbnailImage(const Image *, const size_t, const size_t, ExceptionInfo *);
extern Image *__real_MinifyImage(const Image *, ExceptionInfo *);
extern Image *__real_MotionBlurImage(const Image *, const double, const double, const double, ExceptionInfo *);
extern Image *__real_ConvolveImage(const Image *, const KernelInfo *, ExceptionInfo *);
extern Image *__real_ResampleImage(const Image *, const double, const double, const FilterType, ExceptionInfo *);
extern int mb200_device_count(void);
extern Image *__real_SharpenImage(const Image *, const double, const double, ExceptionInfo *);
extern Image *__real_EmbossImage(const Image *, const double, const double, ExceptionInfo *);
extern Image *__real_StatisticImage(const Image *, const StatisticType, const size_t, const size_t, ExceptionInfo *);
extern Image *__real_RotationalBlurImage(const Image *, const double, ExceptionInfo *);
extern Image *__real_AdaptiveBlurImage(const Image *, const double, const double, ExceptionInfo *);
extern Image *__real_AdaptiveSharpenImage(const Image *, const double, const double, ExceptionInfo *);
extern Image *__real_SelectiveBlurImage(const Image *, const double, const double, const double, ExceptionInfo *);
extern Image *__real_BilateralBlurImage(const Image *, const size_t, const size_t, const double, const double, ExceptionInfo *);
extern MagickBooleanType __real_EqualizeImage(Image *, ExceptionInfo *);
extern Image *__real_DespeckleImage(const Image *, ExceptionInfo *);
extern Image *__real_LocalContrastImage(const Image *, const double, const double, ExceptionInfo *);
extern Image *__real_WaveletDenoiseImage(const Image *, const double, const double, ExceptionInfo *);
extern Image *__real_EdgeImage(const Image *, const double, ExceptionInfo *);
extern MagickBooleanType __real_BilevelImage(Image *, const double, ExceptionInfo *);
extern MagickBooleanType __real_BlackThresholdImage(Image *, const char *, ExceptionInfo *);
extern MagickBooleanType __real_WhiteThresholdImage(Image *, const char *, ExceptionInfo *);
extern MagickBooleanType __real_ClampImage(Image *, ExceptionInfo *);
extern MagickBooleanType __real_ContrastStretchImage(Image *, const double, const double, ExceptionInfo *);
extern MagickBooleanType __real_NormalizeImage(Image *, ExceptionInfo *);
extern MagickBooleanType __real_LinearStretchImage(Image *, const double, const double, ExceptionInfo *);
extern MagickBooleanType __real_LevelImage(Image *, const double, const double, const double, ExceptionInfo *);
extern MagickBooleanType __real_LevelizeImage(Image *, const double, const double, const double, ExceptionInfo *);
extern MagickBooleanType __real_GammaImage(Image *, const double, ExceptionInfo *);
extern Image *__real_AdaptiveThresholdImage(const Image *, const size_t, const size_t, const double, ExceptionInfo *);
extern MagickBooleanType __real_AutoThresholdImage(Image *, const AutoThresholdMethod, ExceptionInfo *);
extern MagickBooleanType __real_RangeThresholdImage(Image *, const double, const double, const double, const double,
                                                    ExceptionInfo *);
extern MagickBooleanType __real_PerceptibleImage(Image *, const double, ExceptionInfo *);
extern long B200ShimHits(void), B200ShimFallbacks(void);
extern void B200ShimEnable(int);

static long ulp(float a, float b)
{
  int ia, ib;
  memcpy(&ia, &a, 4); memcpy(&ib, &b, 4);
  if (ia < 0) ia = -(ia & 0x7fffffff);
  if (ib < 0) ib = -(ib & 0x7fffffff);
  return labs((long) ia - (long) ib);
}

static long compare(const Image *a, const Image *b, ExceptionInfo *ex)
{
  const Quantum *p, *q;
  size_t i, n;
  long worst = 0;
  if (!a || !b || a->columns != b->columns || a->rows != b->rows) return 1L << 40;
  n = a->columns * a->rows * GetPixelChannels(a);
  p = GetVirtualPixels(a, 0, 0, a->columns, a->rows, ex);
  q = GetVirtualPixels(b, 0, 0, b->columns, b->rows, ex);
  for (i = 0; i < n; i++) { long d = ulp((float) p[i], (float) q[i]); if (d > worst) worst = d; }
  return worst;
}

static Image *noise_image(size_t w, size_t h, MagickBooleanType alpha, ExceptionInfo *ex)
{
  ImageInfo *info = AcquireImageInfo();
  Image *im = AcquireImage(info, ex);
  Quantum *q;
  size_t i, n;
  unsigned long long s = 88172645463325252ULL;
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

#define CPU(expr) (B200ShimEnable(0), cpu_tmp = (expr), B200ShimEnable(1), cpu_tmp)
#define CHECK(name, bar, gpu, cpu) do { Image *g_ = (gpu); Image *c_ = (cpu); long d_ = compare(g_, c_, ex); \
  printf("%-34s max ULP %ld (bar %d)%s\n", name, d_, bar, d_ <= bar ? "" : "  FAIL"); if (d_ > bar) failures++; \
  if (g_) DestroyImage(g_); if (c_) DestroyImage(c_); } while (0)

/* TransformImageColorspace(src -> to) through the shim and through __real_TransformImageColorspace, on clones of `src`:
   the pixels (within `bar` ULP), the channel count, the colourspace and the image type must agree.  1 on failure. */
static int layout_case(const char *name, int bar, const Image *src, ColorspaceType to, ExceptionInfo *ex)
{
  Image *a = CloneImage(src, 0, 0, MagickTrue, ex), *b = CloneImage(src, 0, 0, MagickTrue, ex);
  MagickBooleanType ra, rb;
  long d;
  ra = TransformImageColorspace(a, to, ex);
  B200ShimEnable(0); rb = __real_TransformImageColorspace(b, to, ex); B200ShimEnable(1);
  if (ra == MagickFalse || rb == MagickFalse || a->colorspace != to || b->colorspace != to ||
      GetPixelChannels(a) != GetPixelChannels(b) || a->type != b->type) {
    printf("%-34s channels %d/%d colorspace %d/%d type %d/%d  FAIL\n", name, (int) GetPixelChannels(a),
           (int) GetPixelChannels(b), (int) a->colorspace, (int) b->colorspace, (int) a->type, (int) b->type);
    d = 1L << 40;
  } else {
    d = compare(a, b, ex);
    printf("%-34s max ULP %ld (bar %d)%s\n", name, d, bar, d <= bar ? "" : "  FAIL");
  }
  a = DestroyImage(a); b = DestroyImage(b);
  return d > bar;
}

/* a clone of `src` converted by the stock CPU path */
static Image *converted(const Image *src, ColorspaceType to, ExceptionInfo *ex)
{
  Image *im = CloneImage(src, 0, 0, MagickTrue, ex);
  B200ShimEnable(0); (void) __real_TransformImageColorspace(im, to, ex); B200ShimEnable(1);
  return im;
}


/* The level and stretch operators on clones of `src` (under SetPixelChannelMask(mask) when mask >= 0): through the shim
   and through the stock CPU path.  The pixels (within `bar` ULP), the channel count, the colourspace, the "histogram:*"
   properties and image->gamma must agree; with `expect_fallback` the shim must have declined.  1 on failure.
   op: 0 Level, 1 Levelize, 2 Gamma, 3 AutoLevel (MinMaxStretchImage, wrapped), 4 ContrastStretch, 5 Normalize,
   6 LinearStretch. */
static MagickBooleanType level_op(Image *im, int op, double x, double y, double g, int cpu, ExceptionInfo *ex)
{
  switch (op) {
    case 0: return cpu ? __real_LevelImage(im, x, y, g, ex) : LevelImage(im, x, y, g, ex);
    case 1: return cpu ? __real_LevelizeImage(im, x, y, g, ex) : LevelizeImage(im, x, y, g, ex);
    case 2: return cpu ? __real_GammaImage(im, g, ex) : GammaImage(im, g, ex);
    case 3: return AutoLevelImage(im, ex);        /* its MinMaxStretchImage call is wrapped; the CPU side disables the shim */
    case 4: return cpu ? __real_ContrastStretchImage(im, x, y, ex) : ContrastStretchImage(im, x, y, ex);
    case 5: return cpu ? __real_NormalizeImage(im, ex) : NormalizeImage(im, ex);
    default: return cpu ? __real_LinearStretchImage(im, x, y, ex) : LinearStretchImage(im, x, y, ex);
  }
}

static int level_case(const char *name, int bar, const Image *src, int op, double x, double y, double g, long mask,
                      int expect_fallback, ExceptionInfo *ex)
{
  static const char *const props[] = { "histogram:contrast-stretch", "histogram:linear-stretch" };
  Image *a = CloneImage(src, 0, 0, MagickTrue, ex), *b = CloneImage(src, 0, 0, MagickTrue, ex);
  const long fb = B200ShimFallbacks();
  MagickBooleanType ra, rb;
  long d = 0;
  int k, bad = 0;
  if (mask >= 0) { (void) SetPixelChannelMask(a, (ChannelType) mask); (void) SetPixelChannelMask(b, (ChannelType) mask); }
  ra = level_op(a, op, x, y, g, 0, ex);
  B200ShimEnable(0); rb = level_op(b, op, x, y, g, 1, ex); B200ShimEnable(1);
  if (ra == MagickFalse || rb == MagickFalse || GetPixelChannels(a) != GetPixelChannels(b) ||
      a->colorspace != b->colorspace || a->gamma != b->gamma) bad = 1;
  for (k = 0; k < 2; k++) {
    const char *pa = GetImageProperty(a, props[k], ex), *pb = GetImageProperty(b, props[k], ex);
    if ((pa == NULL) != (pb == NULL) || (pa != NULL && strcmp(pa, pb) != 0)) bad = 1;
  }
  if (!bad) d = compare(a, b, ex);
  if (expect_fallback && mb200_device_count() > 0 && B200ShimFallbacks() <= fb) bad = 1;
  printf("%-34s max ULP %ld (bar %d) channels %d/%d%s\n", name, d, bar, (int) GetPixelChannels(a),
         (int) GetPixelChannels(b), bad || d > bar ? "  FAIL" : "");
  a = DestroyImage(a); b = DestroyImage(b);
  return bad || d > bar;
}

/* op: 0 AdaptiveThreshold (x = width, y = height, z = bias), 1 AutoThreshold (x = method), 2 RangeThreshold (x, y, z, t),
   3 Perceptible (x = epsilon) on a clone of `src` (channel mask `mask` unless negative), through the shim and through
   __real_: the pixels bit for bit, the channel count, the colourspace, the type and the "auto-threshold:threshold"
   property must agree; with `expect_fallback` the shim must have declined, otherwise it must have served the call.
   1 on failure. */
static int threshold_case(const char *name, const Image *src, int op, double x, double y, double z, double t, long mask,
                          int expect_fallback, ExceptionInfo *ex)
{
  Image *a = CloneImage(src, 0, 0, MagickTrue, ex), *b = CloneImage(src, 0, 0, MagickTrue, ex), *ra = a, *rb = b;
  const long fb = B200ShimFallbacks(), hits = B200ShimHits();
  MagickBooleanType oka = MagickFalse, okb = MagickFalse;
  const char *pa, *pb;
  long d = 0;
  int bad = 0;
  if (mask >= 0) { (void) SetPixelChannelMask(a, (ChannelType) mask); (void) SetPixelChannelMask(b, (ChannelType) mask); }
  switch (op) {
    case 0:
      ra = AdaptiveThresholdImage(a, (size_t) x, (size_t) y, z, ex);
      B200ShimEnable(0); rb = __real_AdaptiveThresholdImage(b, (size_t) x, (size_t) y, z, ex); B200ShimEnable(1);
      oka = ra != NULL ? MagickTrue : MagickFalse; okb = rb != NULL ? MagickTrue : MagickFalse;
      break;
    case 1:
      oka = AutoThresholdImage(a, (AutoThresholdMethod) (int) x, ex);
      B200ShimEnable(0); okb = __real_AutoThresholdImage(b, (AutoThresholdMethod) (int) x, ex); B200ShimEnable(1);
      break;
    case 2:
      oka = RangeThresholdImage(a, x, y, z, t, ex);
      B200ShimEnable(0); okb = __real_RangeThresholdImage(b, x, y, z, t, ex); B200ShimEnable(1);
      break;
    default:
      oka = PerceptibleImage(a, x, ex);
      B200ShimEnable(0); okb = __real_PerceptibleImage(b, x, ex); B200ShimEnable(1);
      break;
  }
  if (oka == MagickFalse || okb == MagickFalse || GetPixelChannels(ra) != GetPixelChannels(rb) ||
      ra->colorspace != rb->colorspace || ra->type != rb->type) bad = 1;
  else {
    pa = GetImageProperty(ra, "auto-threshold:threshold", ex); pb = GetImageProperty(rb, "auto-threshold:threshold", ex);
    if ((pa == NULL) != (pb == NULL) || (pa != NULL && strcmp(pa, pb) != 0)) bad = 1;
    d = compare(ra, rb, ex);
  }
  if (mb200_device_count() > 0 && (expect_fallback ? B200ShimFallbacks() <= fb : B200ShimHits() <= hits)) bad = 1;
  printf("%-34s max ULP %ld (bar 0) channels %d/%d%s\n", name, d, oka ? (int) GetPixelChannels(ra) : 0,
         okb ? (int) GetPixelChannels(rb) : 0, bad || d > 0 ? "  FAIL" : "");
  if (ra != NULL && ra != a) ra = DestroyImage(ra);
  if (rb != NULL && rb != b) rb = DestroyImage(rb);
  a = DestroyImage(a); b = DestroyImage(b);
  return bad || d > 0;
}

/* DistortImage (method >= 0) / RotateImage (method < 0) on `src` through the shim and through __real_: pixels (bit
   exact), size, page and channel count must agree; with `expect_fallback` the shim must have declined.  1 on failure. */
extern Image *__real_DistortImage(const Image *, const DistortMethod, const size_t, const double *, MagickBooleanType,
                                  ExceptionInfo *);
extern Image *__real_RotateImage(const Image *, const double, ExceptionInfo *);
static int distort_case(const char *name, const Image *src, int method, size_t n, const double *args,
                        MagickBooleanType bestfit, int expect_fallback, ExceptionInfo *ex)
{
  const long fb = B200ShimFallbacks();
  Image *a, *b;
  long d = 0;
  int bad = 0;
  a = method < 0 ? RotateImage(src, args[0], ex) : DistortImage(src, (DistortMethod) method, n, args, bestfit, ex);
  B200ShimEnable(0);
  b = method < 0 ? __real_RotateImage(src, args[0], ex) : __real_DistortImage(src, (DistortMethod) method, n, args, bestfit, ex);
  B200ShimEnable(1);
  if (!a || !b || GetPixelChannels(a) != GetPixelChannels(b) || a->page.x != b->page.x || a->page.y != b->page.y) bad = 1;
  else d = compare(a, b, ex);
  if (expect_fallback && mb200_device_count() > 0 && B200ShimFallbacks() <= fb) bad = 1;
  if (!expect_fallback && mb200_device_count() > 0 && B200ShimFallbacks() > fb) bad = 1;
  printf("%-34s max ULP %ld (bar 0) channels %d/%d%s\n", name, d, a ? (int) GetPixelChannels(a) : 0,
         b ? (int) GetPixelChannels(b) : 0, bad || d > 0 ? "  FAIL" : "");
  if (a) a = DestroyImage(a);
  if (b) b = DestroyImage(b);
  return bad || d > 0;
}

int main(void)
{
  ExceptionInfo *ex;
  Image *rgba, *rgb, *a, *b, *cpu_tmp;
  KernelInfo *k;
  int failures = 0;
  MagickCoreGenesis("shim_harness", MagickFalse);
  ex = AcquireExceptionInfo();
  rgba = noise_image(517, 389, MagickTrue, ex);
  rgb = noise_image(300, 200, MagickFalse, ex);

  {
    static const double srt[] = {0.8, 30.0}, rot30[] = {30.0}, rot90[] = {90.0}, polar_args[] = {20.0};
    static const double persp[] = {0, 0, 10, 5, 516, 0, 480, 30, 0, 388, 20, 360, 516, 388, 500, 380};
    /* Fresh images: a clone shares its pixel cache, and with it the virtual-pixel method, which RotateImage sets to
       Background on its clone (as the reference does), so a clone of rgba would change rgba for the cases below. */
    Image *rot = noise_image(517, 389, MagickTrue, ex), *persp4 = noise_image(517, 389, MagickTrue, ex);
    Image *none = noise_image(300, 200, MagickFalse, ex), *none2 = noise_image(300, 200, MagickFalse, ex);
    Image *g = noise_image(300, 200, MagickFalse, ex), *gray = converted(g, GRAYColorspace, ex);
    Image *point = noise_image(64, 48, MagickTrue, ex), *tile = noise_image(64, 48, MagickTrue, ex);
    Image *polar = noise_image(64, 48, MagickTrue, ex), *r90 = noise_image(64, 48, MagickTrue, ex);
    Image *c = noise_image(64, 48, MagickFalse, ex), *cmyk = converted(c, CMYKColorspace, ex);
    (void) QueryColorCompliance("none", AllCompliance, &none->background_color, ex);
    (void) QueryColorCompliance("none", AllCompliance, &none2->background_color, ex);
    point->filter = PointFilter;
    (void) SetImageVirtualPixelMethod(tile, TileVirtualPixelMethod, ex);
    failures += distort_case("RotateImage 30 RGBA", rot, -1, 1, rot30, MagickTrue, 0, ex);
    failures += distort_case("RotateImage 30 RGB -background none", none, -1, 1, rot30, MagickTrue, 0, ex);
    failures += distort_case("fallback: DistortImage SRT RGB -background none", none2, ScaleRotateTranslateDistortion,
                             2, srt, MagickTrue, 1, ex);
    failures += distort_case("RotateImage 30 gray", gray, -1, 1, rot30, MagickTrue, 0, ex);
    failures += distort_case("DistortImage Perspective RGBA", persp4, PerspectiveDistortion, 16, persp, MagickTrue, 0, ex);
    failures += distort_case("fallback: DistortImage Point filter", point, ScaleRotateTranslateDistortion, 2, srt,
                             MagickTrue, 1, ex);
    failures += distort_case("fallback: DistortImage Tile", tile, ScaleRotateTranslateDistortion, 2, srt, MagickTrue, 1, ex);
    failures += distort_case("fallback: DistortImage Polar", polar, PolarDistortion, 1, polar_args, MagickTrue, 1, ex);
    failures += distort_case("fallback: RotateImage 90", r90, -1, 1, rot90, MagickTrue, 1, ex);
    failures += distort_case("fallback: RotateImage CMYK", cmyk, -1, 1, rot30, MagickTrue, 1, ex);
    rot = DestroyImage(rot); persp4 = DestroyImage(persp4); none = DestroyImage(none); none2 = DestroyImage(none2);
    g = DestroyImage(g); gray = DestroyImage(gray); point = DestroyImage(point); tile = DestroyImage(tile);
    polar = DestroyImage(polar); r90 = DestroyImage(r90); c = DestroyImage(c); cmyk = DestroyImage(cmyk);
  }
  CHECK("BlurImage(0,4) RGBA", 1, BlurImage(rgba, 0.0, 4.0, ex), CPU(__real_BlurImage(rgba, 0.0, 4.0, ex)));
  CHECK("BlurImage(0,2) RGB", 1, BlurImage(rgb, 0.0, 2.0, ex), CPU(__real_BlurImage(rgb, 0.0, 2.0, ex)));
  CHECK("GaussianBlurImage(0,1.5) RGBA", 1, GaussianBlurImage(rgba, 0.0, 1.5, ex), CPU(__real_GaussianBlurImage(rgba, 0.0, 1.5, ex)));
  CHECK("UnsharpMaskImage RGBA", 1, UnsharpMaskImage(rgba, 0.0, 2.0, 1.5, 0.02, ex), CPU(__real_UnsharpMaskImage(rgba, 0.0, 2.0, 1.5, 0.02, ex)));
  CHECK("ResizeImage Lanczos 2x down RGBA", 1, ResizeImage(rgba, 258, 194, LanczosFilter, ex), CPU(__real_ResizeImage(rgba, 258, 194, LanczosFilter, ex)));
  CHECK("ResizeImage default up RGB", 1, ResizeImage(rgb, 450, 300, UndefinedFilter, ex), CPU(__real_ResizeImage(rgb, 450, 300, UndefinedFilter, ex)));
  CHECK("MotionBlurImage(0,3,30) RGBA", 1, MotionBlurImage(rgba, 0.0, 3.0, 30.0, ex), CPU(__real_MotionBlurImage(rgba, 0.0, 3.0, 30.0, ex)));
  CHECK("MinifyImage RGBA (Spline 2x)", 1, MinifyImage(rgba, ex), CPU(__real_MinifyImage(rgba, ex)));
  CHECK("ResampleImage 36 dpi RGB (Lanczos)", 1, ResampleImage(rgb, 36.0, 36.0, LanczosFilter, ex), CPU(__real_ResampleImage(rgb, 36.0, 36.0, LanczosFilter, ex)));
  CHECK("SampleImage 517x389 -> 100x77 RGBA", 0, SampleImage(rgba, 100, 77, ex), CPU(__real_SampleImage(rgba, 100, 77, ex)));
  CHECK("ScaleImage 517x389 -> 200x150 RGBA", 0, ScaleImage(rgba, 200, 150, ex), CPU(__real_ScaleImage(rgba, 200, 150, ex)));
  CHECK("ScaleImage 300x200 -> 450x333 RGB", 0, ScaleImage(rgb, 450, 333, ex), CPU(__real_ScaleImage(rgb, 450, 333, ex)));
  CHECK("SharpenImage(0,1) RGBA", 1, SharpenImage(rgba, 0.0, 1.0, ex), CPU(__real_SharpenImage(rgba, 0.0, 1.0, ex)));
  CHECK("EdgeImage(1) RGB", 1, EdgeImage(rgb, 1.0, ex), CPU(__real_EdgeImage(rgb, 1.0, ex)));
  CHECK("StatisticImage Median 3x3 RGBA", 0, StatisticImage(rgba, MedianStatistic, 3, 3, ex), CPU(__real_StatisticImage(rgba, MedianStatistic, 3, 3, ex)));
  CHECK("StatisticImage Mode 3x3 RGB", 0, StatisticImage(rgb, ModeStatistic, 3, 3, ex), CPU(__real_StatisticImage(rgb, ModeStatistic, 3, 3, ex)));
  CHECK("StatisticImage Nonpeak 5x5 RGBA", 0, StatisticImage(rgba, NonpeakStatistic, 5, 5, ex), CPU(__real_StatisticImage(rgba, NonpeakStatistic, 5, 5, ex)));
  CHECK("StatisticImage StdDev 5x3 RGB", 0, StatisticImage(rgb, StandardDeviationStatistic, 5, 3, ex), CPU(__real_StatisticImage(rgb, StandardDeviationStatistic, 5, 3, ex)));
  CHECK("RotationalBlurImage(7) RGBA", 0, RotationalBlurImage(rgba, 7.0, ex), CPU(__real_RotationalBlurImage(rgba, 7.0, ex)));
  CHECK("AdaptiveBlurImage 0x1.5 RGBA", 0, AdaptiveBlurImage(rgba, 0.0, 1.5, ex), CPU(__real_AdaptiveBlurImage(rgba, 0.0, 1.5, ex)));
  CHECK("AdaptiveSharpenImage 0x1 RGB", 0, AdaptiveSharpenImage(rgb, 0.0, 1.0, ex), CPU(__real_AdaptiveSharpenImage(rgb, 0.0, 1.0, ex)));
  CHECK("SelectiveBlurImage 0x1.5 t=10% RGBA", 0, SelectiveBlurImage(rgba, 0.0, 1.5, 6553.5, ex),
        CPU(__real_SelectiveBlurImage(rgba, 0.0, 1.5, 6553.5, ex)));
  CHECK("DespeckleImage RGBA", 0, DespeckleImage(rgba, ex), CPU(__real_DespeckleImage(rgba, ex)));
  CHECK("DespeckleImage RGB", 0, DespeckleImage(rgb, ex), CPU(__real_DespeckleImage(rgb, ex)));
  CHECK("LocalContrastImage 10x12.5 RGBA", 0, LocalContrastImage(rgba, 10.0, 12.5, ex), CPU(__real_LocalContrastImage(rgba, 10.0, 12.5, ex)));
  CHECK("LocalContrastImage 40x-30 RGB", 0, LocalContrastImage(rgb, 40.0, -30.0, ex), CPU(__real_LocalContrastImage(rgb, 40.0, -30.0, ex)));
  CHECK("WaveletDenoiseImage 10% RGBA", 0, WaveletDenoiseImage(rgba, 6553.5, 0.0, ex), CPU(__real_WaveletDenoiseImage(rgba, 6553.5, 0.0, ex)));
  CHECK("WaveletDenoiseImage 5%+0.3 RGB", 0, WaveletDenoiseImage(rgb, 3276.75, 0.3, ex), CPU(__real_WaveletDenoiseImage(rgb, 3276.75, 0.3, ex)));
  CHECK("BilateralBlurImage 5x5 RGB", 0, BilateralBlurImage(rgb, 5, 5, 20.0, 2.0, ex), CPU(__real_BilateralBlurImage(rgb, 5, 5, 20.0, 2.0, ex)));
  k = AcquireKernelInfo("Disk:3", ex);
  CHECK("MorphologyImage Dilate Disk:3", 0, MorphologyImage(rgba, DilateMorphology, 1, k, ex), CPU(__real_MorphologyImage(rgba, DilateMorphology, 1, k, ex)));
  CHECK("MorphologyImage Erode x2 Disk:3", 0, MorphologyImage(rgb, ErodeMorphology, 2, k, ex), CPU(__real_MorphologyImage(rgb, ErodeMorphology, 2, k, ex)));
  CHECK("MorphologyImage Edge Disk:3 RGBA", 0, MorphologyImage(rgba, EdgeMorphology, 1, k, ex), CPU(__real_MorphologyImage(rgba, EdgeMorphology, 1, k, ex)));
  CHECK("MorphologyImage TopHat Disk:3 RGB", 0, MorphologyImage(rgb, TopHatMorphology, 1, k, ex), CPU(__real_MorphologyImage(rgb, TopHatMorphology, 1, k, ex)));
  k = DestroyKernelInfo(k);
  k = AcquireKernelInfo("Corners", ex);
  CHECK("MorphologyImage HitAndMiss Corners", 0, MorphologyImage(rgb, HitAndMissMorphology, 1, k, ex), CPU(__real_MorphologyImage(rgb, HitAndMissMorphology, 1, k, ex)));
  k = DestroyKernelInfo(k);
  k = AcquireKernelInfo("Skeleton", ex);
  CHECK("MorphologyImage Thinning x3 Skeleton", 0, MorphologyImage(rgba, ThinningMorphology, 3, k, ex), CPU(__real_MorphologyImage(rgba, ThinningMorphology, 3, k, ex)));
  k = DestroyKernelInfo(k);
  k = AcquireKernelInfo("Disk:2", ex);
  CHECK("MorphologyImage OpenIntensity Disk:2", 0, MorphologyImage(rgba, OpenIntensityMorphology, 1, k, ex), CPU(__real_MorphologyImage(rgba, OpenIntensityMorphology, 1, k, ex)));
  k = DestroyKernelInfo(k);
  k = AcquireKernelInfo("Euclidean:2", ex);
  CHECK("MorphologyImage IterativeDistance x4", 0, MorphologyImage(rgb, IterativeDistanceMorphology, 4, k, ex), CPU(__real_MorphologyImage(rgb, IterativeDistanceMorphology, 4, k, ex)));
  k = DestroyKernelInfo(k);
  {
    /* Distance / Voronoi (MorphologyPrimitiveDirect): one run of the head kernel.  Voronoi leaves the alpha trait at
       Copy, and on an image without alpha (whose result gains an alpha channel) it must decline and still be right. */
    const long hits0 = B200ShimHits();
    Image *ga = converted(rgba, GRAYColorspace, ex);
    long fb;
    k = AcquireKernelInfo("Euclidean:4", ex);
    CHECK("MorphologyImage Distance Euclidean:4 RGBA", 0, MorphologyImage(rgba, DistanceMorphology, 1, k, ex), CPU(__real_MorphologyImage(rgba, DistanceMorphology, 1, k, ex)));
    CHECK("MorphologyImage Distance Euclidean:4 GA", 0, MorphologyImage(ga, DistanceMorphology, 3, k, ex), CPU(__real_MorphologyImage(ga, DistanceMorphology, 3, k, ex)));
    (void) SetPixelChannelMask(rgba, (ChannelType) (RedChannel | BlueChannel | AlphaChannel));
    CHECK("MorphologyImage Distance -channel RBA", 0, MorphologyImage(rgba, DistanceMorphology, 1, k, ex), CPU(__real_MorphologyImage(rgba, DistanceMorphology, 1, k, ex)));
    (void) SetPixelChannelMask(rgba, DefaultChannels);
    k = DestroyKernelInfo(k);
    k = AcquireKernelInfo("Chebyshev:2", ex);
    a = MorphologyImage(rgba, VoronoiMorphology, 1, k, ex); b = CPU(__real_MorphologyImage(rgba, VoronoiMorphology, 1, k, ex));
    if (!a || !b || a->alpha_trait != b->alpha_trait || GetPixelChannels(a) != GetPixelChannels(b)) {
      printf("MorphologyImage Voronoi RGBA: alpha trait / channels differ  FAIL\n"); failures++;
    }
    CHECK("MorphologyImage Voronoi Chebyshev:2 RGBA", 0, a, b);
    fb = B200ShimFallbacks();
    a = MorphologyImage(rgb, VoronoiMorphology, 1, k, ex); b = CPU(__real_MorphologyImage(rgb, VoronoiMorphology, 1, k, ex));
    if (!a || !b || a->alpha_trait != b->alpha_trait || GetPixelChannels(a) != GetPixelChannels(b)) {
      printf("MorphologyImage Voronoi RGB: alpha trait / channels differ  FAIL\n"); failures++;
    }
    CHECK("MorphologyImage Voronoi RGB (declines)", 0, a, b);
    if (mb200_device_count() > 0 && B200ShimFallbacks() <= fb) { printf("FAIL: Voronoi without alpha was not declined\n"); failures++; }
    if (mb200_device_count() > 0 && B200ShimHits() - hits0 < 4) { printf("FAIL: Distance / Voronoi did not reach the GPU path\n"); failures++; }
    k = DestroyKernelInfo(k);
    ga = DestroyImage(ga);
  }
  a = CloneImage(rgba, 0, 0, MagickTrue, ex); b = CloneImage(rgba, 0, 0, MagickTrue, ex);
  if (TransformImageColorspace(a, LabColorspace, ex) == MagickFalse || a->colorspace != LabColorspace) failures++;
  B200ShimEnable(0); (void) __real_TransformImageColorspace(b, LabColorspace, ex); B200ShimEnable(1);
  CHECK("TransformImageColorspace sRGB->Lab", 1, a, b);
  a = CloneImage(rgba, 0, 0, MagickTrue, ex); b = CloneImage(rgba, 0, 0, MagickTrue, ex);
  if (TransformImageColorspace(a, HSLColorspace, ex) == MagickFalse || a->colorspace != HSLColorspace) failures++;
  B200ShimEnable(0); (void) __real_TransformImageColorspace(b, HSLColorspace, ex); B200ShimEnable(1);
  CHECK("TransformImageColorspace sRGB->HSL", 0, a, b);
  a = CloneImage(rgb, 0, 0, MagickTrue, ex); b = CloneImage(rgb, 0, 0, MagickTrue, ex);
  (void) SetImageColorspace(a, HWBColorspace, ex); (void) SetImageColorspace(b, HWBColorspace, ex);
  if (TransformImageColorspace(a, HSVColorspace, ex) == MagickFalse || a->colorspace != HSVColorspace) failures++;
  B200ShimEnable(0); (void) __real_TransformImageColorspace(b, HSVColorspace, ex); B200ShimEnable(1);
  CHECK("TransformImageColorspace HWB->HSV", 0, a, b);
  a = CloneImage(rgba, 0, 0, MagickTrue, ex); b = CloneImage(rgba, 0, 0, MagickTrue, ex);
  if (TransformImageColorspace(a, LuvColorspace, ex) == MagickFalse || a->colorspace != LuvColorspace) failures++;
  B200ShimEnable(0); (void) __real_TransformImageColorspace(b, LuvColorspace, ex); B200ShimEnable(1);
  CHECK("TransformImageColorspace sRGB->Luv", 1, a, b);
  a = CloneImage(rgba, 0, 0, MagickTrue, ex); b = CloneImage(rgba, 0, 0, MagickTrue, ex);
  (void) SetImageArtifact(a, "color:illuminant", "D50"); (void) SetImageArtifact(b, "color:illuminant", "D50");
  if (TransformImageColorspace(a, LabColorspace, ex) == MagickFalse || a->colorspace != LabColorspace) failures++;
  B200ShimEnable(0); (void) __real_TransformImageColorspace(b, LabColorspace, ex); B200ShimEnable(1);
  CHECK("TransformImageColorspace sRGB->Lab (D50)", 1, a, b);
  a = CloneImage(rgb, 0, 0, MagickTrue, ex); b = CloneImage(rgb, 0, 0, MagickTrue, ex);
  (void) SetImageProperty(a, "reference-white", "700", ex); (void) SetImageProperty(b, "reference-white", "700", ex);
  if (TransformImageColorspace(a, LogColorspace, ex) == MagickFalse || a->colorspace != LogColorspace) failures++;
  B200ShimEnable(0); (void) __real_TransformImageColorspace(b, LogColorspace, ex); B200ShimEnable(1);
  CHECK("TransformImageColorspace sRGB->Log (reference-white 700)", 1, a, b);
  a = CloneImage(rgba, 0, 0, MagickTrue, ex); b = CloneImage(rgba, 0, 0, MagickTrue, ex);
  if (TransformImageColorspace(a, YCCColorspace, ex) == MagickFalse || a->colorspace != YCCColorspace) failures++;
  B200ShimEnable(0); (void) __real_TransformImageColorspace(b, YCCColorspace, ex); B200ShimEnable(1);
  CHECK("TransformImageColorspace sRGB->YCC", 0, a, b);
  a = CloneImage(rgba, 0, 0, MagickTrue, ex); b = CloneImage(rgba, 0, 0, MagickTrue, ex);
  (void) SetImageColorspace(a, YCCColorspace, ex); (void) SetImageColorspace(b, YCCColorspace, ex);
  if (TransformImageColorspace(a, sRGBColorspace, ex) == MagickFalse || a->colorspace != sRGBColorspace) failures++;
  B200ShimEnable(0); (void) __real_TransformImageColorspace(b, sRGBColorspace, ex); B200ShimEnable(1);
  CHECK("TransformImageColorspace YCC->sRGB", 0, a, b);
  {
    /* the colourspaces that change the channel layout; Lab -> GRAY adds the <= 1 ULP of the Lab leg in R, G and B to a
       weighted sum that can be several times smaller than one of them */
    Image *gray = converted(rgb, GRAYColorspace, ex), *cmyka = converted(rgba, CMYKColorspace, ex),
          *lab = converted(rgba, LabColorspace, ex);
    failures += layout_case("TransformImageColorspace sRGB->GRAY", 0, rgba, GRAYColorspace, ex);
    failures += layout_case("TransformImageColorspace sRGB->LinearGRAY", 1, rgb, LinearGRAYColorspace, ex);
    failures += layout_case("TransformImageColorspace sRGB->CMYK", 0, rgba, CMYKColorspace, ex);
    failures += layout_case("TransformImageColorspace CMYK->sRGB", 0, cmyka, sRGBColorspace, ex);
    failures += layout_case("TransformImageColorspace GRAY->sRGB", 0, gray, sRGBColorspace, ex);
    failures += layout_case("TransformImageColorspace Lab->GRAY", 4, lab, GRAYColorspace, ex);
    gray = DestroyImage(gray); cmyka = DestroyImage(cmyka); lab = DestroyImage(lab);
  }
  CHECK("ResizeImage Jinc 50% RGBA", 1, ResizeImage(rgba, rgba->columns / 2, rgba->rows / 2, JincFilter, ex),
        CPU(__real_ResizeImage(rgba, rgba->columns / 2, rgba->rows / 2, JincFilter, ex)));
  (void) SetImageArtifact(rgba, "filter:blur", "0.85"); (void) SetImageArtifact(rgba, "filter:lobes", "2");
  CHECK("ResizeImage Lanczos 50% blur=.85 lobes=2", 1, ResizeImage(rgba, rgba->columns / 2, rgba->rows / 2, LanczosFilter, ex),
        CPU(__real_ResizeImage(rgba, rgba->columns / 2, rgba->rows / 2, LanczosFilter, ex)));
  (void) DeleteImageArtifact(rgba, "filter:blur"); (void) DeleteImageArtifact(rgba, "filter:lobes");
  CHECK("ResizeImage Kaiser 150% RGB", 1, ResizeImage(rgb, rgb->columns * 3 / 2, rgb->rows * 3 / 2, KaiserFilter, ex),
        CPU(__real_ResizeImage(rgb, rgb->columns * 3 / 2, rgb->rows * 3 / 2, KaiserFilter, ex)));
  /* threshold.c point operators: in place, bit exact */
  a = CloneImage(rgba, 0, 0, MagickTrue, ex); b = CloneImage(rgba, 0, 0, MagickTrue, ex);
  if (BilevelImage(a, 30000.0, ex) == MagickFalse) failures++;
  B200ShimEnable(0); (void) __real_BilevelImage(b, 30000.0, ex); B200ShimEnable(1);
  CHECK("BilevelImage(30000) RGBA", 0, a, b);
  a = CloneImage(rgba, 0, 0, MagickTrue, ex); b = CloneImage(rgba, 0, 0, MagickTrue, ex);
  if (BlackThresholdImage(a, "40%,50%,60%", ex) == MagickFalse) failures++;
  B200ShimEnable(0); (void) __real_BlackThresholdImage(b, "40%,50%,60%", ex); B200ShimEnable(1);
  CHECK("BlackThresholdImage RGBA", 0, a, b);
  a = CloneImage(rgb, 0, 0, MagickTrue, ex); b = CloneImage(rgb, 0, 0, MagickTrue, ex);
  if (WhiteThresholdImage(a, "45000", ex) == MagickFalse) failures++;
  B200ShimEnable(0); (void) __real_WhiteThresholdImage(b, "45000", ex); B200ShimEnable(1);
  CHECK("WhiteThresholdImage RGB", 0, a, b);
  a = CloneImage(rgba, 0, 0, MagickTrue, ex); b = CloneImage(rgba, 0, 0, MagickTrue, ex);
  if (EqualizeImage(a, ex) == MagickFalse) failures++;
  B200ShimEnable(0); (void) __real_EqualizeImage(b, ex); B200ShimEnable(1);
  CHECK("EqualizeImage RGBA", 0, a, b);
  {
    /* EmbossImage ends in an equalisation of the convolved image: a discontinuous map, so a 1-ULP difference of one
       convolved sample may move many outputs a little; compared in absolute terms like the thumbnail cascade */
    Image *g = EmbossImage(rgb, 0.0, 1.0, ex), *c = CPU(__real_EmbossImage(rgb, 0.0, 1.0, ex));
    double worst = 0.0;
    if (!g || !c) { printf("EmbossImage: FAIL\n"); failures++; }
    else {
      const Quantum *p = GetVirtualPixels(g, 0, 0, g->columns, g->rows, ex), *q = GetVirtualPixels(c, 0, 0, c->columns, c->rows, ex);
      size_t i, n = g->columns * g->rows * GetPixelChannels(g);
      for (i = 0; i < n; i++) { double d = fabs((double) p[i] - (double) q[i]); if (d > worst) worst = d; }
      printf("%-34s max |diff| %.5f Quantum (bar 2.0)%s\n", "EmbossImage(0,1) RGB", worst, worst <= 2.0 ? "" : "  FAIL");
      if (worst > 2.0) failures++;
    }
    if (g) DestroyImage(g);
    if (c) DestroyImage(c);
  }
  /* the in-place enhance operators (enhance.c, statistic.c) */
  a = CloneImage(rgba, 0, 0, MagickTrue, ex); b = CloneImage(rgba, 0, 0, MagickTrue, ex);
  if (ContrastImage(a, MagickTrue, ex) == MagickFalse) failures++;
  B200ShimEnable(0); (void) __real_ContrastImage(b, MagickTrue, ex); B200ShimEnable(1);
  CHECK("ContrastImage(sharpen) RGBA", 1, a, b);
  a = CloneImage(rgb, 0, 0, MagickTrue, ex); b = CloneImage(rgb, 0, 0, MagickTrue, ex);
  if (ContrastImage(a, MagickFalse, ex) == MagickFalse) failures++;
  B200ShimEnable(0); (void) __real_ContrastImage(b, MagickFalse, ex); B200ShimEnable(1);
  CHECK("ContrastImage(dull) RGB", 1, a, b);
  a = CloneImage(rgba, 0, 0, MagickTrue, ex); b = CloneImage(rgba, 0, 0, MagickTrue, ex);
  if (ModulateImage(a, "90,130,150", ex) == MagickFalse) failures++;
  B200ShimEnable(0); (void) __real_ModulateImage(b, "90,130,150", ex); B200ShimEnable(1);
  CHECK("ModulateImage 90,130,150 RGBA", 0, a, b);
  a = CloneImage(rgb, 0, 0, MagickTrue, ex); b = CloneImage(rgb, 0, 0, MagickTrue, ex);
  (void) SetImageArtifact(a, "modulate:colorspace", "HWB"); (void) SetImageArtifact(b, "modulate:colorspace", "HWB");
  if (ModulateImage(a, "110x80,40", ex) == MagickFalse) failures++;
  B200ShimEnable(0); (void) __real_ModulateImage(b, "110x80,40", ex); B200ShimEnable(1);
  CHECK("ModulateImage HWB 110x80,40 RGB", 0, a, b);
  a = CloneImage(rgba, 0, 0, MagickTrue, ex); b = CloneImage(rgba, 0, 0, MagickTrue, ex);
  (void) SetImageArtifact(a, "modulate:colorspace", "LCHab"); (void) SetImageArtifact(b, "modulate:colorspace", "LCHab");
  (void) SetImageArtifact(a, "color:illuminant", "D50"); (void) SetImageArtifact(b, "color:illuminant", "D50");
  if (ModulateImage(a, "105,100,140", ex) == MagickFalse) failures++;
  B200ShimEnable(0); (void) __real_ModulateImage(b, "105,100,140", ex); B200ShimEnable(1);
  CHECK("ModulateImage LCHab D50 RGBA", 1, a, b);
  a = CloneImage(rgba, 0, 0, MagickTrue, ex); b = CloneImage(rgba, 0, 0, MagickTrue, ex);
  if (GrayscaleImage(a, Rec709LuminancePixelIntensityMethod, ex) == MagickFalse || a->colorspace != LinearGRAYColorspace ||
      GetPixelChannels(a) != 2) failures++;
  B200ShimEnable(0); (void) __real_GrayscaleImage(b, Rec709LuminancePixelIntensityMethod, ex); B200ShimEnable(1);
  CHECK("GrayscaleImage Rec709Luminance RGBA", 1, a, b);
  a = CloneImage(rgb, 0, 0, MagickTrue, ex); b = CloneImage(rgb, 0, 0, MagickTrue, ex);
  if (GrayscaleImage(a, AveragePixelIntensityMethod, ex) == MagickFalse || a->colorspace != GRAYColorspace ||
      GetPixelChannels(a) != 1) failures++;
  B200ShimEnable(0); (void) __real_GrayscaleImage(b, AveragePixelIntensityMethod, ex); B200ShimEnable(1);
  CHECK("GrayscaleImage Average RGB", 0, a, b);
  {
    const double poly[4] = { 0.5, -0.5, 0.75, 0.1 }, sine[2] = { 3.0, 45.0 };
    a = CloneImage(rgba, 0, 0, MagickTrue, ex); b = CloneImage(rgba, 0, 0, MagickTrue, ex);
    if (FunctionImage(a, PolynomialFunction, 4, poly, ex) == MagickFalse) failures++;
    B200ShimEnable(0); (void) __real_FunctionImage(b, PolynomialFunction, 4, poly, ex); B200ShimEnable(1);
    CHECK("FunctionImage Polynomial RGBA", 0, a, b);
    a = CloneImage(rgb, 0, 0, MagickTrue, ex); b = CloneImage(rgb, 0, 0, MagickTrue, ex);
    if (FunctionImage(a, SinusoidFunction, 2, sine, ex) == MagickFalse) failures++;
    B200ShimEnable(0); (void) __real_FunctionImage(b, SinusoidFunction, 2, sine, ex); B200ShimEnable(1);
    CHECK("FunctionImage Sinusoid RGB", 1, a, b);
  }
  {
    /* level and stretch operators (enhance.c, histogram.c:927): in place, the reference's control plane around them */
    const long hits0 = B200ShimHits();
    Image *gray = CloneImage(rgba, 0, 0, MagickTrue, ex), *t;
    Quantum *q = GetAuthenticPixels(gray, 0, 0, gray->columns, gray->rows, ex);
    size_t i;
    for (i = 0; i < gray->columns * gray->rows; i++) { q[4 * i + 1] = q[4 * i]; q[4 * i + 2] = q[4 * i]; }
    (void) SyncAuthenticPixels(gray, ex);
    failures += level_case("LevelImage 1000,60000,1 RGBA", 0, rgba, 0, 1000.0, 60000.0, 1.0, -1, 0, ex);
    failures += level_case("LevelImage 5000,50000,2.2 RGB", 1, rgb, 0, 5000.0, 50000.0, 2.2, -1, 0, ex);
    failures += level_case("LevelizeImage 1000,60000,0.45 RGBA", 1, rgba, 1, 1000.0, 60000.0, 0.45, -1, 0, ex);
    failures += level_case("LevelImage -channel RBA RGBA", 0, rgba, 0, 2000.0, 50000.0, 1.0,
                           RedChannel | BlueChannel | AlphaChannel, 0, ex);
    failures += level_case("GammaImage 2.2 RGBA", 0, rgba, 2, 0.0, 0.0, 2.2, -1, 0, ex);
    failures += level_case("GammaImage 0.45 RGB", 0, rgb, 2, 0.0, 0.0, 0.45, -1, 0, ex);
    failures += level_case("AutoLevelImage RGBA", 0, rgba, 3, 0.0, 0.0, 1.0, -1, 0, ex);
    failures += level_case("AutoLevelImage -channel RGBA", 0, rgba, 3, 0.0, 0.0, 1.0,
                           RedChannel | GreenChannel | BlueChannel | AlphaChannel, 0, ex);
    failures += level_case("ContrastStretchImage 1%,97% RGBA", 0, rgba, 4, 0.01 * 517 * 389, 0.97 * 517 * 389, 1.0, -1, 0, ex);
    failures += level_case("ContrastStretchImage -channel RGBA", 0, rgba, 4, 0.05 * 517 * 389, 0.9 * 517 * 389, 1.0,
                           RedChannel | GreenChannel | BlueChannel | AlphaChannel, 0, ex);
    failures += level_case("NormalizeImage RGB", 0, rgb, 5, 0.0, 0.0, 1.0, -1, 0, ex);
    failures += level_case("NormalizeImage gray sRGBA -> GA", 0, gray, 5, 0.0, 0.0, 1.0, -1, 0, ex);
    failures += level_case("LinearStretchImage 2%,1% RGBA", 0, rgba, 6, 0.02 * 517 * 389, 0.01 * 517 * 389, 1.0, -1, 0, ex);
    if (mb200_device_count() > 0 && B200ShimHits() - hits0 < 13) { printf("FAIL: level operators did not reach the GPU path\n"); failures++; }
    /* the fallbacks: PseudoClass, a linear-RGB image's intensity histogram, a non-default intensity method */
    t = CloneImage(rgb, 0, 0, MagickTrue, ex);
    (void) SetImageType(t, PaletteType, ex);         /* quantised to a colormap: PseudoClass */
    failures += level_case("fallback: LevelImage PseudoClass", 0, t, 0, 1000.0, 60000.0, 1.0, -1, 1, ex);
    t = DestroyImage(t);
    t = CloneImage(rgb, 0, 0, MagickTrue, ex);
    t->colorspace = RGBColorspace;
    failures += level_case("fallback: NormalizeImage linear RGB", 0, t, 5, 0.0, 0.0, 1.0, -1, 1, ex);
    t = DestroyImage(t);
    t = CloneImage(rgba, 0, 0, MagickTrue, ex);
    t->intensity = AveragePixelIntensityMethod;
    failures += level_case("fallback: LinearStretch Average", 0, t, 6, 0.02 * 517 * 389, 0.01 * 517 * 389, 1.0, -1, 1, ex);
    t = DestroyImage(t);
    gray = DestroyImage(gray);
  }
  a = CloneImage(rgba, 0, 0, MagickTrue, ex); b = CloneImage(rgba, 0, 0, MagickTrue, ex);
  if (ClampImage(a, ex) == MagickFalse) failures++;
  B200ShimEnable(0); (void) __real_ClampImage(b, ex); B200ShimEnable(1);
  CHECK("ClampImage RGBA", 0, a, b);
  {
    /* ThumbnailImage: the cascade is re-issued through the wrapped stages, the metadata comes from the real function.
       A cascade of <= 1 ULP stages is compared in absolute terms (a 1-ULP difference of a bright input sample is many
       ULPs of a dark output sample). */
    const char *const props[] = { "Thumb::URI", "Thumb::Image::Width", "Thumb::Image::Height", "Thumb::Document::Pages",
                                  "Thumb::Size", "software", (const char *) NULL };
    size_t sizes[3][2] = { { 100, 75 }, { 200, 150 }, { 400, 300 } };
    int s, pi;
    for (s = 0; s < 3; s++) {
      Image *g = ThumbnailImage(rgba, sizes[s][0], sizes[s][1], ex);
      Image *c = CPU(__real_ThumbnailImage(rgba, sizes[s][0], sizes[s][1], ex));
      double worst = 0.0;
      if (!g || !c || g->columns != c->columns || g->rows != c->rows) { printf("ThumbnailImage: geometry FAIL\n"); failures++; }
      else {
        const Quantum *p = GetVirtualPixels(g, 0, 0, g->columns, g->rows, ex), *q = GetVirtualPixels(c, 0, 0, c->columns, c->rows, ex);
        size_t i, n = g->columns * g->rows * GetPixelChannels(g);
        for (i = 0; i < n; i++) { double d = fabs((double) p[i] - (double) q[i]); if (d > worst) worst = d; }
        printf("%-34s max |diff| %.5f Quantum (bar 0.02)%s\n", "ThumbnailImage RGBA", worst, worst <= 0.02 ? "" : "  FAIL");
        if (worst > 0.02) failures++;
        if (g->depth != c->depth || g->page.width != c->page.width || g->interlace != c->interlace) { printf("ThumbnailImage: attributes FAIL\n"); failures++; }
        for (pi = 0; props[pi] != (const char *) NULL; pi++) {
          const char *a1 = GetImageProperty(g, props[pi], ex), *b1 = GetImageProperty(c, props[pi], ex);
          if ((a1 == NULL) != (b1 == NULL) || (a1 != NULL && strcmp(a1, b1) != 0)) { printf("ThumbnailImage: property %s FAIL\n", props[pi]); failures++; }
        }
      }
      if (g) DestroyImage(g);
      if (c) DestroyImage(c);
    }
  }
  {
    /* -channel selections: unselected channels carry the Copy trait and are handed through (nearest sample for resize) */
    const long hits0 = B200ShimHits();
    KernelInfo *uk = AcquireKernelInfo("3x3: 1,2,1, 2,4,2, 1,2,1", ex);
    (void) SetPixelChannelMask(rgba, (ChannelType) (RedChannel | BlueChannel | AlphaChannel));
    CHECK("BlurImage(0,2) -channel RBA RGBA", 1, BlurImage(rgba, 0.0, 2.0, ex), CPU(__real_BlurImage(rgba, 0.0, 2.0, ex)));
    CHECK("ResizeImage Lanczos -channel RBA RGBA", 1, ResizeImage(rgba, 258, 194, LanczosFilter, ex), CPU(__real_ResizeImage(rgba, 258, 194, LanczosFilter, ex)));
    CHECK("UnsharpMaskImage -channel RBA RGBA", 1, UnsharpMaskImage(rgba, 0.0, 2.0, 1.5, 0.02, ex), CPU(__real_UnsharpMaskImage(rgba, 0.0, 2.0, 1.5, 0.02, ex)));
    {
      /* alpha unselected: the second pass weights with the unfiltered alpha -- must decline, and still be right */
      const long fb0 = B200ShimFallbacks();
      (void) SetPixelChannelMask(rgba, (ChannelType) (RedChannel | BlueChannel));
      CHECK("BlurImage(0,2) -channel RB (declines)", 0, BlurImage(rgba, 0.0, 2.0, ex), CPU(__real_BlurImage(rgba, 0.0, 2.0, ex)));
      if (mb200_device_count() > 0 && B200ShimFallbacks() <= fb0) { printf("FAIL: alpha-less selection was not declined\n"); failures++; }
    }
    (void) SetPixelChannelMask(rgb, (ChannelType) (RedChannel | BlueChannel));
    CHECK("BlurImage(0,2) -channel RB RGB (no alpha)", 1, BlurImage(rgb, 0.0, 2.0, ex), CPU(__real_BlurImage(rgb, 0.0, 2.0, ex)));
    (void) SetPixelChannelMask(rgb, DefaultChannels);
    (void) SetPixelChannelMask(rgba, (ChannelType) (AlphaChannel | GreenChannel));
    CHECK("MorphologyImage Dilate -channel GA", 0, MorphologyImage(rgba, DilateMorphology, 1, uk, ex), CPU(__real_MorphologyImage(rgba, DilateMorphology, 1, uk, ex)));
    CHECK("ResizeImage up -channel GA RGBA", 1, ResizeImage(rgba, 700, 500, MitchellFilter, ex), CPU(__real_ResizeImage(rgba, 700, 500, MitchellFilter, ex)));
    (void) SetPixelChannelMask(rgba, DefaultChannels);
    if (mb200_device_count() > 0 && B200ShimHits() - hits0 < 5) { printf("FAIL: channel selections did not reach the GPU path\n"); failures++; }
    /* convolve:bias / convolve:scale (morphology.c:4156-4183) are restated by the wrapper */
    (void) SetImageArtifact(rgb, "convolve:bias", "10%");
    (void) SetImageArtifact(rgb, "convolve:scale", "0.05,20%");
    CHECK("ConvolveImage bias 10% scale 0.05,20% RGB", 1, ConvolveImage(rgb, uk, ex), CPU(__real_ConvolveImage(rgb, uk, ex)));
    (void) DeleteImageArtifact(rgb, "convolve:bias");
    (void) DeleteImageArtifact(rgb, "convolve:scale");
    if (mb200_device_count() > 0 && B200ShimHits() - hits0 < 6) { printf("FAIL: convolve artifacts did not reach the GPU path\n"); failures++; }
    uk = DestroyKernelInfo(uk);
  }
  {
    /* ADVICE r01: `-channel RGB -threshold` on an opaque RGB image leaves every trait at its default, but the reference
       then thresholds each channel on its own value -- the intensity-driven kernel must decline */
    const long fb = B200ShimFallbacks();
    (void) SetPixelChannelMask(rgb, (ChannelType) (RedChannel | GreenChannel | BlueChannel));
    a = CloneImage(rgb, 0, 0, MagickTrue, ex); b = CloneImage(rgb, 0, 0, MagickTrue, ex);
    (void) SetPixelChannelMask(a, (ChannelType) (RedChannel | GreenChannel | BlueChannel));
    (void) SetPixelChannelMask(b, (ChannelType) (RedChannel | GreenChannel | BlueChannel));
    if (BilevelImage(a, 30000.0, ex) == MagickFalse) failures++;
    B200ShimEnable(0); (void) __real_BilevelImage(b, 30000.0, ex); B200ShimEnable(1);
    CHECK("BilevelImage -channel RGB (declines)", 0, a, b);
    if (mb200_device_count() > 0 && B200ShimFallbacks() <= fb) { printf("FAIL: per-channel threshold was not declined\n"); failures++; }
    (void) SetPixelChannelMask(rgb, DefaultChannels);
  }
  {
    /* threshold.c: AdaptiveThreshold (-lat), AutoThreshold, RangeThreshold, Perceptible; bit exact */
    const long hits0 = B200ShimHits();
    const long rgb_mask = RedChannel | GreenChannel | BlueChannel;
    Image *gray = CloneImage(rgb, 0, 0, MagickTrue, ex), *t;
    (void) __real_TransformImageColorspace(gray, GRAYColorspace, ex);
    failures += threshold_case("AdaptiveThreshold 15x15+5% RGBA", rgba, 0, 15, 15, 0.05 * QuantumRange, 0, -1, 0, ex);
    failures += threshold_case("AdaptiveThreshold 4x6-500 RGB", rgb, 0, 4, 6, -500.0, 0, -1, 0, ex);
    failures += threshold_case("AdaptiveThreshold 7x5 -channel RGB", rgba, 0, 7, 5, 300.0, 0, rgb_mask, 0, ex);
    failures += threshold_case("AdaptiveThreshold 51x51 gray", gray, 0, 51, 51, 0.0, 0, -1, 0, ex);
    failures += threshold_case("AutoThreshold OTSU RGBA", rgba, 1, OTSUThresholdMethod, 0, 0, 0, -1, 0, ex);
    failures += threshold_case("AutoThreshold Kapur RGB", rgb, 1, KapurThresholdMethod, 0, 0, 0, -1, 0, ex);
    failures += threshold_case("AutoThreshold Triangle gray", gray, 1, TriangleThresholdMethod, 0, 0, 0, -1, 0, ex);
    failures += threshold_case("RangeThreshold RGBA", rgba, 2, 10000, 20000, 40000, 50000, -1, 0, ex);
    failures += threshold_case("RangeThreshold -channel RGB RGBA", rgba, 2, 10000, 20000, 40000, 50000, rgb_mask, 0, ex);
    failures += threshold_case("RangeThreshold gray -> sRGB", gray, 2, 10000, 10000, 40000, 50000, -1, 0, ex);
    failures += threshold_case("Perceptible 30000 RGBA", rgba, 3, 30000.0, 0, 0, 0, -1, 0, ex);
    failures += threshold_case("Perceptible -channel RGB RGBA", rgba, 3, 30000.0, 0, 0, 0, rgb_mask, 0, ex);
    if (mb200_device_count() > 0 && B200ShimHits() - hits0 < 12) { printf("FAIL: threshold operators did not reach the GPU path\n"); failures++; }
    failures += threshold_case("fallback: AdaptiveThreshold 0x5", rgba, 0, 0, 5, 0.0, 0, -1, 1, ex);
    t = CloneImage(rgb, 0, 0, MagickTrue, ex);
    t->colorspace = RGBColorspace;
    failures += threshold_case("fallback: AutoThreshold linear RGB", t, 1, OTSUThresholdMethod, 0, 0, 0, -1, 1, ex);
    t = DestroyImage(t);
    t = CloneImage(rgb, 0, 0, MagickTrue, ex);
    (void) SetImageType(t, PaletteType, ex);
    failures += threshold_case("fallback: Perceptible PseudoClass", t, 3, 1000.0, 0, 0, 0, -1, 1, ex);
    t = DestroyImage(t);
    gray = DestroyImage(gray);
  }
  {
    /* a declined case must silently take the CPU path: tiled virtual pixels are not eligible */
    long fb = B200ShimFallbacks();
    Image *t = CloneImage(rgb, 0, 0, MagickTrue, ex);
    (void) SetImageVirtualPixelMethod(t, TileVirtualPixelMethod, ex);
    a = BlurImage(t, 0.0, 1.0, ex); b = CPU(__real_BlurImage(t, 0.0, 1.0, ex));
    CHECK("fallback: tile virtual pixels", 0, a, b);
    if (B200ShimFallbacks() <= fb) { printf("expected a fallback\n"); failures++; }
    t = DestroyImage(t);
  }
  printf("gpu hits %ld, cpu fallbacks %ld\n", B200ShimHits(), B200ShimFallbacks());
  if (mb200_device_count() > 0 && B200ShimHits() < 32) { printf("FAIL: operators did not reach the GPU path\n"); failures++; }
  rgba = DestroyImage(rgba); rgb = DestroyImage(rgb);
  ex = DestroyExceptionInfo(ex);
  MagickCoreTerminus();
  return failures ? 1 : 0;
}
