/*
  magick_b200_shim.c -- the drop-in boundary: ImageMagick's own MagickCore entry points of
  the hot path, backed by libmagickb200 (include/magick_b200.h).

  Link an application / the MagickCore library with
      -Wl,--wrap=BlurImage,--wrap=GaussianBlurImage,--wrap=ConvolveImage,--wrap=UnsharpMaskImage,\
          --wrap=MorphologyImage,--wrap=ResizeImage,--wrap=TransformImageColorspace,\
          --wrap=BilevelImage,--wrap=BlackThresholdImage,--wrap=WhiteThresholdImage,--wrap=ClampImage,\
          --wrap=SharpenImage,--wrap=EdgeImage,--wrap=SampleImage,--wrap=ThumbnailImage,--wrap=MinifyImage,--wrap=ResampleImage,--wrap=MotionBlurImage,\
          --wrap=EmbossImage,--wrap=EqualizeImage,--wrap=StatisticImage,--wrap=RotationalBlurImage,--wrap=BilateralBlurImage,--wrap=ScaleImage,--wrap=SelectiveBlurImage,--wrap=AdaptiveBlurImage,--wrap=AdaptiveSharpenImage,\
          --wrap=DespeckleImage,--wrap=LocalContrastImage,--wrap=WaveletDenoiseImage,\
          --wrap=ContrastImage,--wrap=ModulateImage,--wrap=GrayscaleImage,--wrap=FunctionImage,\
          --wrap=ContrastStretchImage,--wrap=NormalizeImage,--wrap=LinearStretchImage,--wrap=LevelImage,\
          --wrap=LevelizeImage,--wrap=MinMaxStretchImage,--wrap=GammaImage,--wrap=DistortImage,--wrap=RotateImage,\
          --wrap=FlipImage,--wrap=FlopImage,--wrap=TransposeImage,--wrap=TransverseImage,--wrap=IntegralRotateImage,\
          --wrap=CropImage,--wrap=CropImageToTiles,--wrap=ShaveImage,--wrap=RollImage,--wrap=AutoOrientImage,\
          --wrap=AdaptiveThresholdImage,--wrap=AutoThresholdImage,--wrap=RangeThresholdImage,--wrap=PerceptibleImage
  and every caller of those exported functions (effect.c:765/1709/1170/4256, morphology.c:4129,
  resize.c:3761, colorspace.c:1751, threshold.c:805/927/2518/1087/182/660/2377/2092, effect.c:1308/2013, visual-effects.c:3515,
  enhance.c:1370/3461/2474/1544/4130/3347/2913/3062/2322, histogram.c:927, statistic.c:1064) reaches __wrap_X below.  Each wrapper follows the accelerate
  hook contract of effect.c:783-787 / resize.c:3818-3826: try the GPU; if the image is not
  eligible or the GPU path declines (returns NULL / MagickFalse without raising), run the stock
  CPU implementation (__real_X).  B200Accelerate*Image() are the same functions with the
  accelerate-private.h:35-62 signatures, for a build that patches the #if OPENCL call sites.

  Only public MagickCore API is used: GetVirtualPixels / GetAuthenticPixels return the pixel cache
  itself for full-frame requests on memory caches (cache.c:5126-5156), which is exactly the
  interleaved float Quantum layout the C-ABI takes.
*/
#include "MagickCore/studio.h"
#include "MagickCore/MagickCore.h"
#include "MagickCore/string-private.h"          /* StringToDoubleInterval (convolve:bias, morphology.c:4163) */
#include "MagickCore/colorspace-private.h"      /* IssRGBCompatibleColorspace (ModulateImage, enhance.c:3681) */
#include "magick_b200.h"
#include <math.h>
#include <string.h>

#if !defined(MAGICKCORE_HDRI_SUPPORT) || (MAGICKCORE_QUANTUM_DEPTH != 16)
# error "magick_b200_shim targets the reference's default Q16-HDRI build (Quantum == float)"
#endif

/* ---- eligibility: mirrors checkAccelerateCondition (accelerate.c:110-170) + SURVEY 8b --------- */
/* update_mask == NULL: every channel must carry its default traits (no `-channel` selection).  Otherwise unselected
   channels (Copy trait, pixel.c:6338-6393 SetPixelChannelMask) are accepted and reported: bit c set = channel c is updated. */
/* The channel layout test alone, whatever the virtual-pixel method (DistortImage serves several). */
/* single_stage: the operator reads each source sample of a channel only for that channel's result, so an unselected
   alpha channel feeds nothing and is simply copied (the multi-stage rule below does not apply). */
static int b200_layout_traits(const Image *image, unsigned *update_mask, int single_stage)
{
  const size_t n = GetPixelChannels(image);
  const MagickBooleanType gray = (image->colorspace == GRAYColorspace) ||
    (image->colorspace == LinearGRAYColorspace) ? MagickTrue : MagickFalse;
  if (image->storage_class != DirectClass) return 0;
  if ((image->channels & (ReadMaskChannel | WriteMaskChannel | CompositeMaskChannel)) != 0) return 0;
  if (image->number_meta_channels != 0) return 0;
  if (image->progress_monitor != (MagickProgressMonitor) NULL) return 0;
  if (n < 1 || n > 4) return 0;
  if (GetPixelChannelOffset(image, RedPixelChannel) != 0) return 0;
  {
    /* default traits (pixel.c:6356-6381), or Copy for the channels a -channel selection leaves out */
    ssize_t i;
    unsigned mask = 0;
    for (i = 0; i < (ssize_t) n; i++) {
      PixelChannel ch = GetPixelChannelChannel(image, i);
      PixelTrait want = (ch == AlphaPixelChannel || image->alpha_trait == UndefinedPixelTrait)
        ? UpdatePixelTrait : (PixelTrait) (UpdatePixelTrait | BlendPixelTrait);
      const PixelTrait have = GetPixelChannelTraits(image, ch);
      if (have == want) mask |= 1u << i;
      else if (have != CopyPixelTrait || update_mask == (unsigned *) NULL) return 0;
    }
    if (update_mask != (unsigned *) NULL) *update_mask = mask;
    if (mask == 0) return 0;                       /* nothing to compute: let the CPU path clone */
    /* An UNSELECTED alpha channel is copied by every stage of a multi-stage operator (row pass -> column pass, the two
       resize passes), so the later stages weight the colour channels with the ORIGINAL alpha instead of the filtered
       one: the selected channels then depend on the selection and a final restore pass cannot reproduce them.  Such
       selections stay on the CPU path; with alpha selected (or no alpha) the unselected channels feed nothing. */
    if (!single_stage && image->alpha_trait != UndefinedPixelTrait && mask != ((1u << n) - 1u) &&
        (mask >> (n - 1) & 1u) == 0) return 0;
  }
  if (gray != MagickFalse) {
    if (n == 1 && image->alpha_trait == UndefinedPixelTrait) return 1;
    if (n == 2 && image->alpha_trait != UndefinedPixelTrait &&
        GetPixelChannelOffset(image, AlphaPixelChannel) == 1) return 2;
    return 0;
  }
  if (image->colorspace == CMYKColorspace) return 0;
  if (GetPixelChannelOffset(image, GreenPixelChannel) != 1 ||
      GetPixelChannelOffset(image, BluePixelChannel) != 2) return 0;
  if (n == 3 && image->alpha_trait == UndefinedPixelTrait) return 3;
  if (n == 4 && image->alpha_trait != UndefinedPixelTrait &&
      GetPixelChannelOffset(image, AlphaPixelChannel) == 3) return 4;
  return 0;
}

static int b200_layout_masked(const Image *image, unsigned *update_mask)
{ return b200_layout_traits(image, update_mask, 0); }

static int b200_channels_stage(const Image *image, unsigned *update_mask, int single_stage)
{
  if ((GetImageVirtualPixelMethod(image) != UndefinedVirtualPixelMethod) &&
      (GetImageVirtualPixelMethod(image) != EdgeVirtualPixelMethod)) return 0;
  return b200_layout_traits(image, update_mask, single_stage);
}

static int b200_channels_masked(const Image *image, unsigned *update_mask)
{ return b200_channels_stage(image, update_mask, 0); }

static int b200_channels(const Image *image) { return b200_channels_masked(image, (unsigned *) NULL); }

/* CMYK images (TransformImageColorspace only): cyan, magenta, yellow, black at offsets 0-3 and alpha at 4, every channel
   with its default traits (pixel.c:6145-6170); 4 or 5 channels. */
static int b200_cmyk_channels(const Image *image)
{
  const size_t n = GetPixelChannels(image);
  ssize_t i;
  if (image->colorspace != CMYKColorspace || image->storage_class != DirectClass) return 0;
  if ((image->channels & (ReadMaskChannel | WriteMaskChannel | CompositeMaskChannel)) != 0) return 0;
  if (image->number_meta_channels != 0) return 0;
  if ((GetImageVirtualPixelMethod(image) != UndefinedVirtualPixelMethod) &&
      (GetImageVirtualPixelMethod(image) != EdgeVirtualPixelMethod)) return 0;
  if (image->progress_monitor != (MagickProgressMonitor) NULL) return 0;
  if (GetPixelChannelOffset(image, CyanPixelChannel) != 0 || GetPixelChannelOffset(image, MagentaPixelChannel) != 1 ||
      GetPixelChannelOffset(image, YellowPixelChannel) != 2 || GetPixelChannelOffset(image, BlackPixelChannel) != 3)
    return 0;
  if (!(n == 4 && image->alpha_trait == UndefinedPixelTrait) &&
      !(n == 5 && image->alpha_trait != UndefinedPixelTrait && GetPixelChannelOffset(image, AlphaPixelChannel) == 4))
    return 0;
  for (i = 0; i < (ssize_t) n; i++) {
    const PixelChannel ch = GetPixelChannelChannel(image, i);
    const PixelTrait want = (ch == AlphaPixelChannel || image->alpha_trait == UndefinedPixelTrait)
      ? UpdatePixelTrait : (PixelTrait) (UpdatePixelTrait | BlendPixelTrait);
    if (GetPixelChannelTraits(image, ch) != want) return 0;
  }
  return (int) n;
}

static MagickBooleanType has_artifact(const Image *image, const char *const *names)
{
  for (; *names != (const char *) NULL; names++)
    if (GetImageArtifact(image, *names) != (const char *) NULL) return MagickTrue;
  return MagickFalse;
}

static const char *const morphology_artifacts[] = { "convolve:bias", "convolve:scale",
  "morphology:compose", "morphology:showKernel", "debug", (const char *) NULL };
/* MorphologyImage itself restates convolve:bias / convolve:scale (B200AccelerateMorphologyImage); the others change the
   control flow (kernel-list merging, stderr output) */
static const char *const morphology_control_artifacts[] = { "morphology:compose", "morphology:showKernel", "debug",
  (const char *) NULL };
static const char *const compose_artifacts[] = { "compose:clamp", "compose:sync", "compose:args",
  "compose:outside-overlay", "compose:clip-to-self", (const char *) NULL };
static const char *const filter_artifacts[] = { "filter:filter", "filter:window", "filter:sigma",
  "filter:alpha", "filter:kaiser-beta", "filter:kaiser-alpha", "filter:lobes", "filter:blur",
  "filter:support", "filter:win-support", "filter:b", "filter:c", "filter:verbose",
  (const char *) NULL };

/* Output image with the reference's conventions (morphology.c:3926-3933, resize.c:3827, :3872). */
static Image *new_result(const Image *image, size_t columns, size_t rows, ExceptionInfo *exception)
{
  Image *out = CloneImage(image, columns, rows, MagickTrue, exception);
  if (out == (Image *) NULL) return out;
  if (SetImageStorageClass(out, DirectClass, exception) == MagickFalse) return DestroyImage(out);
  if (GetPixelChannels(out) != GetPixelChannels(image)) return DestroyImage(out);
  return out;
}

/* The pixel cache itself, for images whose cache is heap memory (cache.c:1273: the OpenCL path makes the same
   MemoryCache test; disk, map and distributed caches decline).  GetPixelCachePixels (cache.c:2310) hands out
   cache_info->pixels without passing one of the cache's sync sites -- what GetAuthenticOpenCLBuffer (cache.c:1259)
   is to the OpenCL path: in hook mode a result that still lives in HBM must not be pulled back just because the
   next operator asks where the pixels are. */
static float *b200_cache_pixels(const Image *image, int channels, ExceptionInfo *exception)
{
  MagickSizeType length = 0;
  void *pixels;
  if (GetImagePixelCacheType(image) != MemoryCache) return (float *) NULL;
  pixels = GetPixelCachePixels((Image *) image, &length, exception);
  if (pixels == (void *) NULL ||
      length != (MagickSizeType) image->columns * image->rows * (size_t) channels * sizeof(Quantum))
    return (float *) NULL;
  return (float *) pixels;
}

/* A GPU attempt reports into an ExceptionInfo of its own: when it declines, the CPU path must start with the
   caller's exception untouched (the "declined without raising" contract of effect.c:783-787). */
#define B200_ATTEMPT_BEGIN ExceptionInfo *attempt = AcquireExceptionInfo()
#define B200_ATTEMPT_END   attempt = DestroyExceptionInfo(attempt)

typedef int (*same_size_op)(const float *, float *, size_t, size_t, int, const void *);

/* src pixels -> new image through `op`; NULL == declined (caller falls back to the CPU).  allow_mask 1: the operator hands
   Copy-trait channels through from its source, so a -channel selection is served by one extra point pass; 2: the
   operator ignores the selection (it computes the same channels whatever their traits), so it is served as is; 3: as 1
   for a single-stage operator, whose unselected alpha channel feeds nothing (b200_layout_traits). */
static Image *run_same_size_masked(const Image *image, same_size_op op, const void *args, int allow_mask,
                                   ExceptionInfo *exception)
{
  unsigned update_mask = 0xfu;
  const int ch = allow_mask ? b200_channels_stage(image, &update_mask, allow_mask == 3) : b200_channels(image);
  const float *p;
  Quantum *q;
  Image *out;
  (void) exception;
  if (ch == 0 || mb200_device_count() <= 0) return (Image *) NULL;
  {
    B200_ATTEMPT_BEGIN;
    out = (Image *) NULL;
    p = b200_cache_pixels(image, ch, attempt);
    if (p != (const float *) NULL) out = new_result(image, image->columns, image->rows, attempt);
    if (out != (Image *) NULL) {
      q = GetAuthenticPixels(out, 0, 0, out->columns, out->rows, attempt);
      if (q == (Quantum *) NULL || b200_cache_pixels(out, ch, attempt) != (float *) q ||
          op(p, (float *) q, image->columns, image->rows, ch, args) != MB200_OK ||
          ((allow_mask == 1 || allow_mask == 3) && (update_mask & ((1u << ch) - 1u)) != ((1u << ch) - 1u) &&
           mb200_restore_channels((float *) q, p, image->columns, image->rows, ch, update_mask) != MB200_OK) ||
          SyncAuthenticPixels(out, attempt) == MagickFalse)
        out = DestroyImage(out);
    }
    B200_ATTEMPT_END;
  }
  if (out != (Image *) NULL) out->type = image->type;
  return out;
}

static Image *run_same_size(const Image *image, same_size_op op, const void *args, ExceptionInfo *exception)
{ return run_same_size_masked(image, op, args, 0, exception); }

/* ---- BlurImage / GaussianBlurImage / UnsharpMaskImage ------------------------------------------ */
typedef struct { double radius, sigma, gain, threshold; } blur_args;
static int op_blur(const float *s, float *d, size_t w, size_t h, int ch, const void *a)
{ const blur_args *b = (const blur_args *) a; return mb200_blur_image(s, d, w, h, ch, b->radius, b->sigma); }
static int op_gaussian(const float *s, float *d, size_t w, size_t h, int ch, const void *a)
{ const blur_args *b = (const blur_args *) a; return mb200_gaussian_blur_image(s, d, w, h, ch, b->radius, b->sigma); }
static int op_unsharp(const float *s, float *d, size_t w, size_t h, int ch, const void *a)
{ const blur_args *b = (const blur_args *) a;
  return mb200_unsharp_mask_image(s, d, w, h, ch, b->radius, b->sigma, b->gain, b->threshold); }

Image *B200AccelerateBlurImage(const Image *image, const double radius, const double sigma,
                               ExceptionInfo *exception)
{
  blur_args a = { radius, sigma, 0.0, 0.0 };
  if (has_artifact(image, morphology_artifacts) != MagickFalse) return (Image *) NULL;
  return run_same_size_masked(image, op_blur, &a, 1, exception);
}

Image *B200AccelerateGaussianBlurImage(const Image *image, const double radius, const double sigma,
                                       ExceptionInfo *exception)
{
  blur_args a = { radius, sigma, 0.0, 0.0 };
  if (has_artifact(image, morphology_artifacts) != MagickFalse) return (Image *) NULL;
  return run_same_size_masked(image, op_gaussian, &a, 1, exception);
}

Image *B200AccelerateUnsharpMaskImage(const Image *image, const double radius, const double sigma,
                                      const double gain, const double threshold, ExceptionInfo *exception)
{
  blur_args a = { radius, sigma, gain, threshold };
  if (has_artifact(image, morphology_artifacts) != MagickFalse) return (Image *) NULL;
  return run_same_size_masked(image, op_unsharp, &a, 1, exception);
}

/* ---- MorphologyImage / ConvolveImage --------------------------------------------------------------- */
static int map_kernel_type(KernelInfoType t)
{
  switch (t) {                       /* only what RotateKernelInfo distinguishes (morphology.c:4281-4305) */
    case BlurKernel: return MB200_BlurKernel;
    case GaussianKernel: case DoGKernel: case LoGKernel: case DiskKernel: case PeaksKernel:
    case LaplacianKernel: case ChebyshevKernel: case ManhattanKernel: case EuclideanKernel:
      return MB200_GaussianKernel;
    case SquareKernel: case DiamondKernel: case PlusKernel: case CrossKernel: return MB200_SquareKernel;
    default: return MB200_UserDefinedKernel;
  }
}

typedef struct { int method; long iterations; const KernelInfo *kernel; double bias; } morph_args;
static int op_morphology(const float *s, float *d, size_t w, size_t h, int ch, const void *a)
{
  const morph_args *m = (const morph_args *) a;
  mb200_kernel_info nodes[64];
  const KernelInfo *k;
  int n = 0, rc;
  for (k = m->kernel; k != (const KernelInfo *) NULL; k = k->next) {
    if (n == 64) return MB200_EUNSUPPORTED;
    memset(&nodes[n], 0, sizeof(nodes[n]));
    nodes[n].type = map_kernel_type(k->type);
    nodes[n].width = k->width; nodes[n].height = k->height;
    nodes[n].x = (long) k->x; nodes[n].y = (long) k->y;
    nodes[n].values = (double *) k->values;      /* MagickRealType == double; read-only use */
    nodes[n].minimum = k->minimum; nodes[n].maximum = k->maximum;
    nodes[n].negative_range = k->negative_range; nodes[n].positive_range = k->positive_range;
    nodes[n].angle = k->angle;
    if (n > 0) nodes[n - 1].next = &nodes[n];
    n++;
  }
  if (n == 0) return MB200_EINVAL;
  rc = mb200_morphology_image(s, d, w, h, ch, m->method, m->iterations, &nodes[0], m->bias);
  return rc;
}

/* Distance / Voronoi (morphology.c:3736-3776): one run of MorphologyPrimitiveDirect with the head kernel of the list,
   whatever the iteration count (0 aside) and bias. */
typedef struct { int method; const KernelInfo *kernel; } direct_args;
static int op_morphology_direct(const float *s, float *d, size_t w, size_t h, int ch, const void *a)
{
  const direct_args *m = (const direct_args *) a;
  mb200_kernel_info node;
  memset(&node, 0, sizeof(node));
  node.type = map_kernel_type(m->kernel->type);
  node.width = m->kernel->width; node.height = m->kernel->height;
  node.x = (long) m->kernel->x; node.y = (long) m->kernel->y;
  node.values = (double *) m->kernel->values;    /* MagickRealType == double; read-only use */
  return mb200_morphology_direct_image(s, d, w, h, ch, m->method, &node);
}

static Image *morphology_direct(const Image *image, const MorphologyMethod method, const KernelInfo *kernel,
                                ExceptionInfo *exception)
{
  direct_args a;
  Image *out;
  a.method = (int) method; a.kernel = kernel;
  if (method == DistanceMorphology)
    /* Copy-trait channels are skipped by the sweeps and so keep the clone's value: the restore pass gives the same */
    return run_same_size_masked(image, op_morphology_direct, &a, 1, exception);
  /* Voronoi ends in SetImageAlphaChannel(Deactivate), CompositeImage(CopyAlpha), Deactivate (:3766-3774).  The library
     computes the composite's result for the default compose settings and traits on an image with alpha; without alpha
     the result gains a channel, and a -channel selection would change what the composite writes. */
  if (image->alpha_trait == UndefinedPixelTrait) return (Image *) NULL;
  if (has_artifact(image, compose_artifacts) != MagickFalse) return (Image *) NULL;
  out = run_same_size_masked(image, op_morphology_direct, &a, 0, exception);
  if (out != (Image *) NULL) (void) SetImageAlphaChannel(out, DeactivateAlphaChannel, exception);   /* Blend -> Copy */
  return out;
}

Image *B200AccelerateMorphologyImage(const Image *image, const MorphologyMethod method,
                                     const ssize_t iterations, const KernelInfo *kernel,
                                     ExceptionInfo *exception)
{
  morph_args a;
  KernelInfo *scaled = (KernelInfo *) NULL;
  Image *out;
  int allow_mask = 1;
  const char *artifact;
  if (kernel == (const KernelInfo *) NULL || iterations == 0) return (Image *) NULL;
  if (has_artifact(image, morphology_control_artifacts) != MagickFalse) return (Image *) NULL;
  a.bias = 0.0;
  switch (method) {
    case ConvolveMorphology: case CorrelateMorphology:
      /* convolve:bias / convolve:scale apply to these two methods only (morphology.c:4156-4183) */
      artifact = GetImageArtifact(image, "convolve:bias");
      if (artifact != (const char *) NULL) {
        if (IsGeometry(artifact) == MagickFalse) return (Image *) NULL;      /* the reference warns: let it */
        a.bias = StringToDoubleInterval(artifact, (double) QuantumRange + 1.0);
      }
      artifact = GetImageArtifact(image, "convolve:scale");
      if (artifact != (const char *) NULL) {
        if (IsGeometry(artifact) == MagickFalse) return (Image *) NULL;
        scaled = CloneKernelInfo(kernel);
        if (scaled == (KernelInfo *) NULL) return (Image *) NULL;
        ScaleGeometryKernelInfo(scaled, artifact);
      }
      break;
    case ErodeMorphology: case DilateMorphology: case OpenMorphology: case CloseMorphology: case SmoothMorphology: break;
    case EdgeInMorphology: case EdgeOutMorphology: case EdgeMorphology: case TopHatMorphology:
    case BottomHatMorphology:                /* end in CompositeImage(Difference), morphology.c:3995-4012 */
      if (kernel->next != (KernelInfo *) NULL) return (Image *) NULL;
      if (has_artifact(image, compose_artifacts) != MagickFalse) return (Image *) NULL;
      allow_mask = 0;                        /* the composite step treats a channel selection on its own terms */
      break;
    case ErodeIntensityMorphology: case DilateIntensityMorphology: case OpenIntensityMorphology:
    case CloseIntensityMorphology:           /* GetPixelIntensity (pixel.c:2356): the kernel implements the default Rec709 luma */
      if (image->intensity != UndefinedPixelIntensityMethod && image->intensity != Rec709LumaPixelIntensityMethod)
        return (Image *) NULL;
      if (image->colorspace == RGBColorspace || image->colorspace == LinearGRAYColorspace) return (Image *) NULL;
      allow_mask = 0;                        /* the intensity is taken from the masked-out channels as well */
      break;
    case IterativeDistanceMorphology: case ThinningMorphology: case ThickenMorphology: break;
    case HitAndMissMorphology:               /* a kernel list is united with CompositeImage(Lighten), morphology.c:4044 */
      if (kernel->next != (KernelInfo *) NULL) {
        if (has_artifact(image, compose_artifacts) != MagickFalse) return (Image *) NULL;
        allow_mask = 0;
      }
      break;
    case DistanceMorphology: case VoronoiMorphology: return morphology_direct(image, method, kernel, exception);
    default: return (Image *) NULL;
  }
  a.method = (int) method; a.iterations = (long) iterations; a.kernel = scaled != (KernelInfo *) NULL ? scaled : kernel;
  out = run_same_size_masked(image, op_morphology, &a, allow_mask, exception);
  if (scaled != (KernelInfo *) NULL) scaled = DestroyKernelInfo(scaled);
  return out;
}

/* ---- ResizeImage -------------------------------------------------------------------------------------- */
/* The "filter:*" expert settings (-define filter:blur=0.8 ...), read exactly as AcquireResizeFilter reads them
   (resize.c:999-1226: GetImageArtifact + IsStringTrue / ParseCommandOption / StringToDouble / StringToLong) and handed to
   the library as values.  MagickFalse: a setting the GPU path does not serve (filter:verbose prints the filter). */
static MagickBooleanType b200_filter_options(const Image *image, mb200_filter_options *o)
{
  const char *a;
  (void) memset(o, 0, sizeof(*o));
  if (IsStringTrue(GetImageArtifact(image, "filter:verbose")) != MagickFalse) return MagickFalse;
  o->keep_filter = IsStringTrue(GetImageArtifact(image, "filter:filter")) != MagickFalse ? 1 : 0;
  if (o->keep_filter != 0) {
    /* :1000-1011: a truthy string is parsed as a filter name; a name that parses would replace the filter itself */
    ssize_t option = ParseCommandOption(MagickFilterOptions, MagickFalse, GetImageArtifact(image, "filter:filter"));
    if ((UndefinedFilter < option) && (option < SentinelFilter)) return MagickFalse;
  }
  a = GetImageArtifact(image, "filter:window");
  if (a != (const char *) NULL) {
    ssize_t option = ParseCommandOption(MagickFilterOptions, MagickFalse, a);
    if ((UndefinedFilter < option) && (option < SentinelFilter)) { o->window = (int) option; o->set |= MB200_FO_WINDOW; }
  }
  a = GetImageArtifact(image, "filter:sigma");
  if (a != (const char *) NULL) { o->sigma = StringToDouble(a, (char **) NULL); o->set |= MB200_FO_SIGMA; }
  a = GetImageArtifact(image, "filter:alpha");
  if (a != (const char *) NULL) { o->kaiser_beta = StringToDouble(a, (char **) NULL); o->set |= MB200_FO_KAISER_BETA; }
  a = GetImageArtifact(image, "filter:kaiser-beta");
  if (a != (const char *) NULL) { o->kaiser_beta = StringToDouble(a, (char **) NULL); o->set |= MB200_FO_KAISER_BETA; }
  a = GetImageArtifact(image, "filter:kaiser-alpha");
  if (a != (const char *) NULL) { o->kaiser_beta = StringToDouble(a, (char **) NULL) * 3.14159265358979323846264338327950288419716939937510; o->set |= MB200_FO_KAISER_BETA; }
  a = GetImageArtifact(image, "filter:lobes");
  if (a != (const char *) NULL) { o->lobes = (long) StringToLong(a); o->set |= MB200_FO_LOBES; }
  a = GetImageArtifact(image, "filter:blur");
  if (a != (const char *) NULL) { o->blur = StringToDouble(a, (char **) NULL); o->set |= MB200_FO_BLUR; }
  a = GetImageArtifact(image, "filter:support");
  if (a != (const char *) NULL) { o->support = StringToDouble(a, (char **) NULL); o->set |= MB200_FO_SUPPORT; }
  a = GetImageArtifact(image, "filter:win-support");
  if (a != (const char *) NULL) { o->win_support = StringToDouble(a, (char **) NULL); o->set |= MB200_FO_WIN_SUPPORT; }
  a = GetImageArtifact(image, "filter:b");
  if (a != (const char *) NULL) { o->b = StringToDouble(a, (char **) NULL); o->set |= MB200_FO_B; }
  a = GetImageArtifact(image, "filter:c");
  if (a != (const char *) NULL) { o->c = StringToDouble(a, (char **) NULL); o->set |= MB200_FO_C; }
  if ((o->set & MB200_FO_WINDOW) == 0) o->keep_filter = 0;
  return MagickTrue;
}

Image *B200AccelerateResizeImage(const Image *image, const size_t columns, const size_t rows,
                                 const FilterType filter, ExceptionInfo *exception)
{
  mb200_filter_options fopt;
  unsigned update_mask = 0xfu;
  const int ch = b200_channels_masked(image, &update_mask);
  const float *p;
  Quantum *q;
  Image *out;
  (void) exception;
  if (ch == 0 || columns == 0 || rows == 0 || mb200_device_count() <= 0) return (Image *) NULL;
  if (b200_filter_options(image, &fopt) == MagickFalse) return (Image *) NULL;       /* filter:verbose: stdout belongs to the CPU path */
  if (fopt.set != 0 && (update_mask & ((1u << ch) - 1u)) != ((1u << ch) - 1u)) return (Image *) NULL;
  if (image->storage_class == PseudoClass) return (Image *) NULL;
  {
    B200_ATTEMPT_BEGIN;
    out = (Image *) NULL;
    p = b200_cache_pixels(image, ch, attempt);
    if (p != (const float *) NULL) out = new_result(image, columns, rows, attempt);
    if (out != (Image *) NULL) {
      q = GetAuthenticPixels(out, 0, 0, columns, rows, attempt);
      if (q == (Quantum *) NULL || b200_cache_pixels(out, ch, attempt) != (float *) q ||
          mb200_resize_image_ex(p, image->columns, image->rows, ch, (float *) q, columns, rows, (int) filter,
                                fopt.set != 0 ? &fopt : (const mb200_filter_options *) NULL) != MB200_OK ||
          ((update_mask & ((1u << ch) - 1u)) != ((1u << ch) - 1u) &&
           mb200_resize_copy_channels(p, image->columns, image->rows, ch, (float *) q, columns, rows, (int) filter,
                                      update_mask) != MB200_OK) ||
          SyncAuthenticPixels(out, attempt) == MagickFalse)
        out = DestroyImage(out);
    }
    B200_ATTEMPT_END;
  }
  if (out != (Image *) NULL) out->type = image->type;
  return out;
}

/* ---- DistortImage / RotateImage (distort.c:1754, :2954) -------------------------------------------------------- */
/* The affine and perspective methods through the EWA sampler.  The output geometry comes from the library's planner;
   "distort:viewport" is parsed with the reference's ParseAbsoluteGeometry over the geometry it overrides, and
   "distort:scale" with StringToDouble.  A source without alpha whose result gains one inside DistortImage (a background
   or matte colour with an alpha trait, distort.c:2436-2437 and pixel.c:232-234) is declined; RotateImage's own
   SetImageVirtualPixelMethod adds that alpha before DistortImage, so its results are served.  NULL == declined, with
   the caller's exception untouched. */
static Image *b200_distort(const Image *image, const DistortMethod method, const size_t number_arguments,
                           const double *arguments, const MagickBooleanType bestfit, ExceptionInfo *exception)
{
  const VirtualPixelMethod vpm = GetImageVirtualPixelMethod(image);
  mb200_distort_params plan;
  mb200_resample_options o;
  mb200_filter_options fopt;
  const Image *src = image;
  Image *out = (Image *) NULL;
  const char *a;
  double scale = NAN;
  long viewport[4];
  int ch, viewport_given = 0;
  (void) exception;
  if (method != AffineDistortion && method != AffineProjectionDistortion && method != ScaleRotateTranslateDistortion &&
      method != PerspectiveDistortion && method != PerspectiveProjectionDistortion && method != RigidAffineDistortion)
    return (Image *) NULL;
  if (mb200_device_count() <= 0 || b200_layout_masked(image, (unsigned *) NULL) == 0) return (Image *) NULL;
  if (vpm != UndefinedVirtualPixelMethod && vpm != EdgeVirtualPixelMethod && vpm != BackgroundVirtualPixelMethod &&
      vpm != TransparentVirtualPixelMethod && vpm != BlackVirtualPixelMethod && vpm != GrayVirtualPixelMethod &&
      vpm != WhiteVirtualPixelMethod) return (Image *) NULL;
  if (image->interpolate != UndefinedInterpolatePixel && image->interpolate != BilinearInterpolatePixel)
    return (Image *) NULL;
  if (image->filter == PointFilter || b200_filter_options(image, &fopt) == MagickFalse) return (Image *) NULL;
  if (IsStringTrue(GetImageArtifact(image, "distort:verbose")) != MagickFalse) return (Image *) NULL;
  if (IsGrayColorspace(image->colorspace) != MagickFalse && IsPixelInfoGray(&image->background_color) == MagickFalse)
    return (Image *) NULL;                           /* the reference re-lays the result out to sRGB (:2433-2435) */
  if (image->alpha_trait == UndefinedPixelTrait && (image->background_color.alpha_trait != UndefinedPixelTrait ||
                                                    image->matte_color.alpha_trait != UndefinedPixelTrait))
    return (Image *) NULL;                           /* the result gains alpha inside DistortImage (:2436-2437) */
  a = GetImageArtifact(image, "distort:scale");
  if (a != (const char *) NULL) scale = StringToDouble(a, (char **) NULL);
  if (mb200_distort_plan((int) method, arguments, number_arguments, bestfit != MagickFalse ? 1 : 0, image->columns,
                         image->rows, (long) image->page.x, (long) image->page.y, (const long *) NULL, NAN, &plan) != MB200_OK)
    return (Image *) NULL;                           /* the reference raises its own argument errors */
  a = GetImageArtifact(image, "distort:viewport");
  if (a != (const char *) NULL) {
    RectangleInfo geometry;
    geometry.width = plan.columns; geometry.height = plan.rows; geometry.x = plan.page_x; geometry.y = plan.page_y;
    if (ParseAbsoluteGeometry(a, &geometry) == NoValue) return (Image *) NULL;     /* the reference warns */
    viewport[0] = (long) geometry.width; viewport[1] = (long) geometry.height;
    viewport[2] = (long) geometry.x; viewport[3] = (long) geometry.y;
    viewport_given = 1;
  }
  if (mb200_distort_plan((int) method, arguments, number_arguments, bestfit != MagickFalse ? 1 : 0, image->columns,
                         image->rows, (long) image->page.x, (long) image->page.y,
                         viewport_given ? viewport : (const long *) NULL, scale, &plan) != MB200_OK)
    return (Image *) NULL;
  (void) memset(&o, 0, sizeof(o));
  o.filter = (int) image->filter;
  o.filter_options = fopt.set != 0 ? &fopt : (const mb200_filter_options *) NULL;
  o.virtual_pixel = (int) vpm;
  o.interpolate = (int) image->interpolate;
  o.background[0] = image->background_color.red; o.background[1] = image->background_color.green;
  o.background[2] = image->background_color.blue; o.background[3] = image->background_color.alpha;
  o.matte[0] = image->matte_color.red; o.matte[1] = image->matte_color.green;
  o.matte[2] = image->matte_color.blue; o.matte[3] = image->matte_color.alpha;
  o.matte_alpha = image->matte_color.alpha_trait != UndefinedPixelTrait ? 1 : 0;
  {
    B200_ATTEMPT_BEGIN;
    ch = b200_layout_masked(src, (unsigned *) NULL);
    if (ch != 0) {
      const float *p = b200_cache_pixels(src, ch, attempt);
      if (p != (const float *) NULL) out = new_result(src, plan.columns, plan.rows, attempt);
      if (out != (Image *) NULL) {
        Quantum *q = GetAuthenticPixels(out, 0, 0, out->columns, out->rows, attempt);
        if (q == (Quantum *) NULL || b200_cache_pixels(out, ch, attempt) != (float *) q ||
            mb200_distort_image(p, src->columns, src->rows, ch, (float *) q, &plan, &o) != MB200_OK ||
            SyncAuthenticPixels(out, attempt) == MagickFalse)
          out = DestroyImage(out);
      }
    }
    B200_ATTEMPT_END;
  }
  if (out != (Image *) NULL) {
    out->page.x = plan.page_x;
    out->page.y = plan.page_y;
  }
  return out;
}

Image *B200AccelerateDistortImage(const Image *image, const DistortMethod method, const size_t number_arguments,
                                  const double *arguments, const MagickBooleanType bestfit, ExceptionInfo *exception)
{
  return b200_distort(image, method, number_arguments, arguments, bestfit, exception);
}

/* RotateImage: integral rotations stay with the reference (IntegralRotateImage); otherwise its own clone, its own
   SetImageVirtualPixelMethod(Background) -- which adds an opaque alpha or re-lays a gray image out as cache.c:5294-5309
   does -- and DistortImage(ScaleRotateTranslate, bestfit) on it. */
Image *B200AccelerateRotateImage(const Image *image, const double degrees, ExceptionInfo *exception)
{
  mb200_distort_params plan;
  Image *clone, *out = (Image *) NULL;
  (void) exception;
  if (mb200_device_count() <= 0 || b200_layout_masked(image, (unsigned *) NULL) == 0) return (Image *) NULL;
  if (mb200_rotate_plan(degrees, image->columns, image->rows, (long) image->page.x, (long) image->page.y, &plan) != MB200_OK)
    return (Image *) NULL;
  {
    B200_ATTEMPT_BEGIN;
    clone = CloneImage(image, 0, 0, MagickTrue, attempt);
    if (clone != (Image *) NULL) {
      (void) SetImageVirtualPixelMethod(clone, BackgroundVirtualPixelMethod, attempt);
      out = b200_distort(clone, ScaleRotateTranslateDistortion, 1, &degrees, MagickTrue, attempt);
      clone = DestroyImage(clone);
    }
    B200_ATTEMPT_END;
  }
  return out;
}

/* ---- SampleImage (resize.c:3907) ------------------------------------------------------------------------------ */
Image *B200AccelerateSampleImage(const Image *image, const size_t columns, const size_t rows, ExceptionInfo *exception)
{
  const int ch = b200_channels(image);
  const float *p;
  Quantum *q;
  Image *out;
  (void) exception;
  if (ch == 0 || columns == 0 || rows == 0 || mb200_device_count() <= 0) return (Image *) NULL;
  if ((columns == image->columns) && (rows == image->rows)) return (Image *) NULL;      /* plain clone: CPU */
  if (GetImageArtifact(image, "sample:offset") != (const char *) NULL) return (Image *) NULL;
  {
    B200_ATTEMPT_BEGIN;
    out = (Image *) NULL;
    p = b200_cache_pixels(image, ch, attempt);
    if (p != (const float *) NULL) out = new_result(image, columns, rows, attempt);
    if (out != (Image *) NULL) {
      q = GetAuthenticPixels(out, 0, 0, columns, rows, attempt);
      if (q == (Quantum *) NULL || b200_cache_pixels(out, ch, attempt) != (float *) q ||
          mb200_sample_image(p, image->columns, image->rows, ch, (float *) q, columns, rows) != MB200_OK ||
          SyncAuthenticPixels(out, attempt) == MagickFalse)
        out = DestroyImage(out);
    }
    B200_ATTEMPT_END;
  }
  if (out != (Image *) NULL) out->type = image->type;
  return out;
}

/* ---- ScaleImage (resize.c:4106) --------------------------------------------------------------------------------------------- */
Image *B200AccelerateScaleImage(const Image *image, const size_t columns, const size_t rows, ExceptionInfo *exception)
{
  const int ch = b200_channels(image);
  const float *p;
  Quantum *q;
  Image *out;
  (void) exception;
  if (ch == 0 || columns == 0 || rows == 0 || mb200_device_count() <= 0) return (Image *) NULL;
  if ((columns == image->columns) && (rows == image->rows)) return (Image *) NULL;      /* plain clone: CPU */
  {
    B200_ATTEMPT_BEGIN;
    out = (Image *) NULL;
    p = b200_cache_pixels(image, ch, attempt);
    if (p != (const float *) NULL) out = new_result(image, columns, rows, attempt);
    if (out != (Image *) NULL) {
      q = GetAuthenticPixels(out, 0, 0, columns, rows, attempt);
      if (q == (Quantum *) NULL || b200_cache_pixels(out, ch, attempt) != (float *) q ||
          mb200_scale_image(p, image->columns, image->rows, ch, (float *) q, columns, rows) != MB200_OK ||
          SyncAuthenticPixels(out, attempt) == MagickFalse)
        out = DestroyImage(out);
    }
    B200_ATTEMPT_END;
  }
  if (out != (Image *) NULL) out->type = image->type;
  return out;
}

/* ---- TransformImageColorspace (in place) ------------------------------------------------------------ */
static int map_colorspace(ColorspaceType c)
{
  switch (c) {
    case sRGBColorspace: return MB200_sRGBColorspace;
    case RGBColorspace: return MB200_RGBColorspace;
    case LabColorspace: return MB200_LabColorspace;
    case XYZColorspace: return MB200_XYZColorspace;
    case CMYColorspace: return MB200_CMYColorspace;
    case OHTAColorspace: return MB200_OHTAColorspace;
    case Rec601YCbCrColorspace: return MB200_Rec601YCbCrColorspace;
    case Rec709YCbCrColorspace: return MB200_Rec709YCbCrColorspace;
    case YCbCrColorspace: return MB200_YCbCrColorspace;
    case YDbDrColorspace: return MB200_YDbDrColorspace;
    case YIQColorspace: return MB200_YIQColorspace;
    case YPbPrColorspace: return MB200_YPbPrColorspace;
    case YUVColorspace: return MB200_YUVColorspace;
    case LCHColorspace: return MB200_LCHColorspace;
    case LCHabColorspace: return MB200_LCHabColorspace;
    case LCHuvColorspace: return MB200_LCHuvColorspace;
    case LogColorspace: return MB200_LogColorspace;
    case YCCColorspace: return MB200_YCCColorspace;
    case JzazbzColorspace: return MB200_JzazbzColorspace;
    case OklabColorspace: return MB200_OklabColorspace;
    case OklchColorspace: return MB200_OklchColorspace;
    case LMSColorspace: return MB200_LMSColorspace;
    case LuvColorspace: return MB200_LuvColorspace;
    case xyYColorspace: return MB200_xyYColorspace;
    case DisplayP3Colorspace: return MB200_DisplayP3Colorspace;
    case Adobe98Colorspace: return MB200_Adobe98Colorspace;
    case ProPhotoColorspace: return MB200_ProPhotoColorspace;
    case CAT02LMSColorspace: return MB200_CAT02LMSColorspace;
    case HCLColorspace: return MB200_HCLColorspace;
    case HCLpColorspace: return MB200_HCLpColorspace;
    case HSBColorspace: return MB200_HSBColorspace;
    case HSIColorspace: return MB200_HSIColorspace;
    case HSLColorspace: return MB200_HSLColorspace;
    case HSVColorspace: return MB200_HSVColorspace;
    case HWBColorspace: return MB200_HWBColorspace;
    case GRAYColorspace: return MB200_GRAYColorspace;
    case LinearGRAYColorspace: return MB200_LinearGRAYColorspace;
    case CMYKColorspace: return MB200_CMYKColorspace;
    default: return -1;
  }
}

/* The image settings sRGBTransformImage / TransformsRGBImage read (colorspace.c:761-773, :996, :1081-1095), parsed with
   the reference's own functions.  False: leave the image to the CPU path. */
static MagickBooleanType b200_colorspace_options(const Image *image, mb200_colorspace_options *o, ExceptionInfo *exception)
{
  const char *value;
  (void) memset(o, 0, sizeof(*o));
  value = GetImageArtifact(image, "color:illuminant");
  if (value != (const char *) NULL) {
    const ssize_t type = ParseCommandOption(MagickIlluminantOptions, MagickFalse, value);
    o->illuminant = type < 0 ? (int) UndefinedIlluminant : (int) type;      /* :769-772 */
    o->set |= MB200_CO_ILLUMINANT;
  }
  value = GetImageProperty(image, "white-luminance", exception);
  if (value != (const char *) NULL) { o->white_luminance = StringToDouble(value, (char **) NULL); o->set |= MB200_CO_WHITE_LUMINANCE; }
  if (GetImageProperty(image, "gamma", exception) != (const char *) NULL) return MagickFalse;   /* unreachable through SetImageProperty */
  value = GetImageProperty(image, "film-gamma", exception);
  if (value != (const char *) NULL) { o->film_gamma = StringToDouble(value, (char **) NULL); o->set |= MB200_CO_FILM_GAMMA; }
  value = GetImageProperty(image, "reference-black", exception);
  if (value != (const char *) NULL) { o->reference_black = StringToDouble(value, (char **) NULL); o->set |= MB200_CO_REFERENCE_BLACK; }
  value = GetImageProperty(image, "reference-white", exception);
  if (value != (const char *) NULL) { o->reference_white = StringToDouble(value, (char **) NULL); o->set |= MB200_CO_REFERENCE_WHITE; }
  /* the reference's table loops index past MaxMap for values outside the 10-bit scale */
  if ((o->set & MB200_CO_REFERENCE_BLACK) != 0 && !(o->reference_black >= 0.0 && o->reference_black <= 1024.0)) return MagickFalse;
  if ((o->set & MB200_CO_REFERENCE_WHITE) != 0 && !(o->reference_white >= 0.0 && o->reference_white <= 1024.0)) return MagickFalse;
  return MagickTrue;
}

/* GRAY, LinearGRAY or CMYK on either side: the pixel cache changes its channel layout.  The library runs from the current
   cache into a host buffer in the target layout (a failure there is a clean decline: nothing has changed yet); then
   SetImageColorspace re-lays the cache out, the buffer is copied into it, and `type` is set as the reference leaves it
   (GrayscaleType for the gray spaces, colorspace.c:898 / :955; ColorSeparation[Alpha]Type for CMYK, :837-838; otherwise
   what the pixel sync leaves, as after the reference's own pixel loops). */
static int b200_source_channels(Image *image, int from)
{
  const ColorspaceType saved = image->colorspace;
  int ch;
  if (from == MB200_CMYKColorspace) return b200_cmyk_channels(image);
  if (from == MB200_GRAYColorspace || from == MB200_LinearGRAYColorspace) return b200_channels(image);
  image->colorspace = sRGBColorspace;          /* the channel layout test is colourspace-agnostic for 3/4-channel images */
  ch = b200_channels(image);
  image->colorspace = saved;
  return ch == 3 || ch == 4 ? ch : 0;
}

static MagickBooleanType b200_transform_colorspace_layout(Image *image, const ColorspaceType colorspace, int from, int to,
                                                          const mb200_colorspace_options *copt, ExceptionInfo *exception)
{
  const int ch = b200_source_channels(image, from);
  const size_t n = image->columns * image->rows;
  int out_ch, rc = MB200_EINVAL;
  float *buf;
  const float *p;
  Quantum *q;
  MagickBooleanType ok = MagickFalse;
  if (ch == 0) return MagickFalse;
  out_ch = mb200_colorspace_channels(to, ch - mb200_colorspace_channels(from, 0));
  buf = (float *) AcquireQuantumMemory(n, (size_t) out_ch * sizeof(float));
  if (buf == (float *) NULL) return MagickFalse;
  {
    B200_ATTEMPT_BEGIN;
    p = b200_cache_pixels(image, ch, attempt);
    if (p != (const float *) NULL)
      rc = mb200_transform_colorspace_layout(p, ch, buf, out_ch, image->columns, image->rows, from, to,
                                             copt->set != 0 ? copt : (const mb200_colorspace_options *) NULL);
    B200_ATTEMPT_END;
  }
  if (rc == MB200_OK) {
    (void) DeleteImageProfile(image, "icc");                 /* colorspace.c:1763-1764 */
    (void) DeleteImageProfile(image, "icm");
    if (SetImageColorspace(image, colorspace, exception) != MagickFalse && (int) GetPixelChannels(image) == out_ch) {
      q = GetAuthenticPixels(image, 0, 0, image->columns, image->rows, exception);
      if (q != (Quantum *) NULL) {
        (void) memcpy(q, buf, n * (size_t) out_ch * sizeof(float));
        ok = SyncAuthenticPixels(image, exception);
      }
    }
    /* the pixel sync resets `type` (as the reference's own loops do); the reference then sets these two */
    if (colorspace == CMYKColorspace)
      image->type = image->alpha_trait == UndefinedPixelTrait ? ColorSeparationType : ColorSeparationAlphaType;
    else if (colorspace == GRAYColorspace || colorspace == LinearGRAYColorspace)
      image->type = GrayscaleType;
  }
  buf = (float *) RelinquishMagickMemory(buf);
  return ok;
}

MagickBooleanType B200AccelerateTransformImageColorspace(Image *image, const ColorspaceType colorspace,
                                                         ExceptionInfo *exception)
{
  const int from = map_colorspace(image->colorspace), to = map_colorspace(colorspace);
  ColorspaceType saved = image->colorspace;
  mb200_colorspace_options copt;
  Quantum *q;
  int ch;
  if (from < 0 || to < 0 || from == to || mb200_device_count() <= 0) return MagickFalse;
  if (b200_colorspace_options(image, &copt, exception) == MagickFalse) return MagickFalse;
  if (from == MB200_GRAYColorspace || from == MB200_LinearGRAYColorspace || from == MB200_CMYKColorspace ||
      to == MB200_GRAYColorspace || to == MB200_LinearGRAYColorspace || to == MB200_CMYKColorspace)
    return b200_transform_colorspace_layout(image, colorspace, from, to, &copt, exception);
  /* the channel layout test is colourspace-agnostic for 3/4-channel images */
  image->colorspace = sRGBColorspace;
  ch = b200_channels(image);
  image->colorspace = saved;
  if (ch != 3 && ch != 4) return MagickFalse;
  {
    MagickBooleanType ok = MagickFalse;
    B200_ATTEMPT_BEGIN;
    /* GetAuthenticPixels un-shares a copy-on-write cache (GetImagePixelCache, cache.c:1715) before it is written */
    q = GetAuthenticPixels(image, 0, 0, image->columns, image->rows, attempt);
    if (q != (Quantum *) NULL && b200_cache_pixels(image, ch, attempt) == (float *) q &&
        mb200_transform_colorspace_ex((float *) q, image->columns, image->rows, ch, from, to,
                                      copt.set != 0 ? &copt : (const mb200_colorspace_options *) NULL) == MB200_OK &&
        SyncAuthenticPixels(image, attempt) != MagickFalse)
      ok = MagickTrue;
    B200_ATTEMPT_END;
    if (ok == MagickFalse) return MagickFalse;    /* nothing was written back: the CPU path starts from the same pixels */
  }
  (void) DeleteImageProfile(image, "icc");                 /* colorspace.c:1763-1764 */
  (void) DeleteImageProfile(image, "icm");
  return SetImageColorspace(image, colorspace, exception);  /* colorspace.c:1051 */
}

/* ---- threshold.c point operators (in place, bit exact) ---------------------------------------------- */
static MagickBooleanType default_intensity(const Image *image)
{
  return ((image->intensity == UndefinedPixelIntensityMethod) ||
          (image->intensity == Rec709LumaPixelIntensityMethod)) ? MagickTrue : MagickFalse;
}

/* op: 0 BilevelImage, 1 BlackThresholdImage, 2 WhiteThresholdImage, 3 ClampImage */
static MagickBooleanType run_threshold(Image *image, int op, double threshold, const char *thresholds,
                                       ExceptionInfo *exception)
{
  Quantum *q;
  int ch, rc, cs;
  if (mb200_device_count() <= 0) return MagickFalse;
  /* With a channel mask the reference thresholds every selected channel on ITS OWN value (threshold.c:871, :1032,
     :2623); the kernel implements the default, intensity-driven form only.  `-channel RGB` on an opaque RGB image
     leaves every trait at its default, so the trait test of b200_channels() cannot see the mask. */
  if (op != 3 && image->channel_mask != AllChannels) return MagickFalse;
  if (op != 3 && default_intensity(image) == MagickFalse) return MagickFalse;
  if (image->colorspace == LinearGRAYColorspace) return MagickFalse;       /* intensity would need EncodePixelGamma */
  if ((op == 1 || op == 2) && thresholds == (const char *) NULL) return MagickFalse;
  ch = b200_channels(image);
  if (ch == 0) return MagickFalse;
  if ((op == 1 || op == 2) && (ch < 3 || image->colorspace == RGBColorspace)) return MagickFalse;  /* :949, pixel.c:2421 */
  if (op == 0 && image->colorspace != GRAYColorspace && image->colorspace != LinearGRAYColorspace)
    (void) SetImageColorspace(image, sRGBColorspace, exception);            /* threshold.c:827 */
  if (GetPixelChannels(image) != (size_t) ch) return MagickFalse;
  cs = image->colorspace == RGBColorspace ? MB200_RGBColorspace : MB200_sRGBColorspace;
  {
    MagickBooleanType ok = MagickFalse;
    B200_ATTEMPT_BEGIN;
    q = GetAuthenticPixels(image, 0, 0, image->columns, image->rows, attempt);
    rc = MB200_EINVAL;
    if (q != (Quantum *) NULL && b200_cache_pixels(image, ch, attempt) == (float *) q)
      switch (op) {
        case 0: rc = mb200_bilevel_image((float *) q, image->columns, image->rows, ch, threshold); break;
        case 1: rc = mb200_black_threshold_image((float *) q, image->columns, image->rows, ch, cs, thresholds); break;
        case 2: rc = mb200_white_threshold_image((float *) q, image->columns, image->rows, ch, cs, thresholds); break;
        default: rc = mb200_clamp_image((float *) q, image->columns, image->rows, ch); break;
      }
    /* on failure nothing was written back: the CPU path starts from the same pixels */
    if (rc == MB200_OK && SyncAuthenticPixels(image, attempt) != MagickFalse) ok = MagickTrue;
    B200_ATTEMPT_END;
    return ok;
  }
}

MagickBooleanType B200AccelerateBilevelImage(Image *image, const double threshold, ExceptionInfo *exception)
{ return run_threshold(image, 0, threshold, (const char *) NULL, exception); }
MagickBooleanType B200AccelerateBlackThresholdImage(Image *image, const char *thresholds, ExceptionInfo *exception)
{ return run_threshold(image, 1, 0.0, thresholds, exception); }
MagickBooleanType B200AccelerateWhiteThresholdImage(Image *image, const char *thresholds, ExceptionInfo *exception)
{ return run_threshold(image, 2, 0.0, thresholds, exception); }
MagickBooleanType B200AccelerateClampImage(Image *image, ExceptionInfo *exception)
{ return run_threshold(image, 3, 0.0, (const char *) NULL, exception); }

/* AdaptiveThresholdImage (threshold.c:182): edge / undefined virtual pixels; Copy-trait channels take the source sample,
   which the restore pass of run_same_size_masked puts back.  width or height 0 (a plain clone) and windows beyond the
   library's limit decline. */
typedef struct { size_t width, height; double bias; } adaptive_threshold_args;
static int op_adaptive_threshold(const float *s, float *d, size_t w, size_t h, int ch, const void *a)
{
  const adaptive_threshold_args *t = (const adaptive_threshold_args *) a;
  return mb200_adaptive_threshold_image(s, d, w, h, ch, t->width, t->height, t->bias, 0xfu);
}

Image *B200AccelerateAdaptiveThresholdImage(const Image *image, const size_t width, const size_t height, const double bias,
                                            ExceptionInfo *exception)
{
  adaptive_threshold_args a;
  if (width == 0 || height == 0) return (Image *) NULL;
  a.width = width; a.height = height; a.bias = bias;
  return run_same_size_masked(image, op_adaptive_threshold, &a, 3, exception);
}

/* In place on the Update channels of a single-stage operator (op 0 AutoThreshold, 1 RangeThreshold, 2 Perceptible). */
typedef struct { int op, method, per_channel; double x[4]; double threshold; } threshold_args;
static MagickBooleanType run_threshold_masked(Image *image, threshold_args *a)
{
  MagickBooleanType ok = MagickFalse;
  unsigned update_mask = 0;
  const int ch = b200_layout_traits(image, &update_mask, 1);     /* point operators: no virtual pixels */
  Quantum *q;
  int rc = MB200_EINVAL;
  if (ch == 0 || mb200_device_count() <= 0) return MagickFalse;
  {
    B200_ATTEMPT_BEGIN;
    q = GetAuthenticPixels(image, 0, 0, image->columns, image->rows, attempt);
    if (q != (Quantum *) NULL && b200_cache_pixels(image, ch, attempt) == (float *) q) {
      float *buf = (float *) q;
      const size_t w = image->columns, h = image->rows;
      switch (a->op) {
        case 0: rc = mb200_auto_threshold_image(buf, w, h, ch, a->method, &a->threshold); break;
        case 1:
          rc = mb200_range_threshold_image(buf, w, h, ch, a->x[0], a->x[1], a->x[2], a->x[3], a->per_channel, update_mask);
          break;
        default: rc = mb200_perceptible_image(buf, w, h, ch, a->x[0], update_mask); break;
      }
    }
    /* on failure nothing was written back: the CPU path starts from the same pixels */
    if (rc == MB200_OK && SyncAuthenticPixels(image, attempt) != MagickFalse) ok = MagickTrue;
    B200_ATTEMPT_END;
  }
  return ok;
}

/* AutoThresholdImage (threshold.c:660): the Rec709Luma intensity histogram of an sRGB-compatible or gray image, then
   BilevelImage under the default channel mask (its call stays inside threshold.o), the "auto-threshold:threshold"
   property and BilevelImage's sRGB tag.  The auto-threshold:verbose report, a channel mask (BilevelImage would then
   threshold each channel on its own value), other intensity methods and linear RGB / LinearGRAY images decline. */
MagickBooleanType B200AccelerateAutoThresholdImage(Image *image, const AutoThresholdMethod method, ExceptionInfo *exception)
{
  threshold_args a;
  char property[MagickPathExtent];
  if (GetImageArtifact(image, "auto-threshold:verbose") != (const char *) NULL) return MagickFalse;
  if (image->channel_mask != AllChannels || default_intensity(image) == MagickFalse) return MagickFalse;
  if (image->colorspace == RGBColorspace || image->colorspace == LinearGRAYColorspace) return MagickFalse;
  if (b200_layout_masked(image, (unsigned *) NULL) == 0) return MagickFalse;     /* every channel with its default traits */
  (void) memset(&a, 0, sizeof(a));
  a.op = 0;
  a.method = (method == KapurThresholdMethod) ? MB200_KapurThresholdMethod :
             (method == TriangleThresholdMethod) ? MB200_TriangleThresholdMethod : MB200_OTSUThresholdMethod;
  if (run_threshold_masked(image, &a) == MagickFalse) return MagickFalse;
  (void) FormatLocaleString(property, MagickPathExtent, "%g%%", a.threshold);
  (void) SetImageProperty(image, "auto-threshold:threshold", property, exception);
  if (IsGrayColorspace(image->colorspace) == MagickFalse)
    (void) SetImageColorspace(image, sRGBColorspace, exception);              /* threshold.c:827 */
  return MagickTrue;
}

/* RangeThresholdImage (threshold.c:2377): a gray image is first transformed to sRGB (:2407) through the wrapped
   TransformImageColorspace; the default channel mask thresholds on the intensity (Rec709Luma, not on a linear RGB
   image), a selection on each channel's own sample. */
MagickBooleanType B200AccelerateRangeThresholdImage(Image *image, const double low_black, const double low_white,
                                                    const double high_white, const double high_black,
                                                    ExceptionInfo *exception)
{
  threshold_args a;
  const int per_channel = image->channel_mask != AllChannels ? 1 : 0;
  if (mb200_device_count() <= 0) return MagickFalse;
  if (!per_channel && (default_intensity(image) == MagickFalse || image->colorspace == RGBColorspace)) return MagickFalse;
  {
    unsigned mask = 0;
    if (b200_layout_traits(image, &mask, 1) == 0) return MagickFalse;      /* before the transform */
  }
  if (IsGrayColorspace(image->colorspace) != MagickFalse &&
      TransformImageColorspace(image, sRGBColorspace, exception) == MagickFalse) return MagickFalse;
  (void) memset(&a, 0, sizeof(a));
  a.op = 1; a.per_channel = per_channel;
  a.x[0] = low_black; a.x[1] = low_white; a.x[2] = high_white; a.x[3] = high_black;
  return run_threshold_masked(image, &a);
}

/* PerceptibleImage (threshold.c:2092) on the Update channels; the PseudoClass colormap branch declines. */
MagickBooleanType B200AcceleratePerceptibleImage(Image *image, const double epsilon, ExceptionInfo *exception)
{
  threshold_args a;
  (void) exception;
  (void) memset(&a, 0, sizeof(a));
  a.op = 2; a.x[0] = epsilon;
  return run_threshold_masked(image, &a);
}

/* ---- SharpenImage / EdgeImage (effect.c:3991, :1520): inline kernel + ConvolveImage -------------------------- */
static int op_sharpen(const float *s, float *d, size_t w, size_t h, int ch, const void *a)
{ const blur_args *b = (const blur_args *) a; return mb200_sharpen_image(s, d, w, h, ch, b->radius, b->sigma); }
static int op_edge(const float *s, float *d, size_t w, size_t h, int ch, const void *a)
{ const blur_args *b = (const blur_args *) a; return mb200_edge_image(s, d, w, h, ch, b->radius); }

Image *B200AccelerateSharpenImage(const Image *image, const double radius, const double sigma, ExceptionInfo *exception)
{
  blur_args a;
  if (has_artifact(image, morphology_artifacts) != MagickFalse) return (Image *) NULL;
  a.radius = radius; a.sigma = sigma; a.gain = 0.0; a.threshold = 0.0;
  return run_same_size_masked(image, op_sharpen, &a, 1, exception);
}

Image *B200AccelerateEdgeImage(const Image *image, const double radius, ExceptionInfo *exception)
{
  blur_args a;
  if (has_artifact(image, morphology_artifacts) != MagickFalse) return (Image *) NULL;
  a.radius = radius; a.sigma = 0.0; a.gain = 0.0; a.threshold = 0.0;
  return run_same_size_masked(image, op_edge, &a, 1, exception);
}

/* ---- EqualizeImage (enhance.c:2040; the reference's hook is AccelerateEqualizeImage) and EmbossImage (effect.c:1600) ----- */
static MagickBooleanType equalize_eligible(const Image *image)
{
  /* the histogram is indexed by GetPixelIntensity (pixel.c:2356): only its default method on non-linear images is
     restated; linear RGB / gray would go through EncodePixelGamma */
  if (default_intensity(image) == MagickFalse) return MagickFalse;
  if (image->colorspace == RGBColorspace || image->colorspace == LinearGRAYColorspace) return MagickFalse;
  return MagickTrue;
}

MagickBooleanType B200AccelerateEqualizeImage(Image *image, ExceptionInfo *exception)
{
  const int ch = b200_channels(image);
  const int sync = (image->channel_mask & SyncChannels) != 0 ? 1 : 0;
  MagickBooleanType ok = MagickFalse;
  Quantum *q;
  (void) exception;
  if (ch == 0 || mb200_device_count() <= 0 || equalize_eligible(image) == MagickFalse) return MagickFalse;
  {
    B200_ATTEMPT_BEGIN;
    q = GetAuthenticPixels(image, 0, 0, image->columns, image->rows, attempt);
    if (q != (Quantum *) NULL && b200_cache_pixels(image, ch, attempt) == (float *) q &&
        mb200_equalize_image((float *) q, image->columns, image->rows, ch, sync) == MB200_OK &&
        SyncAuthenticPixels(image, attempt) != MagickFalse)
      ok = MagickTrue;
    B200_ATTEMPT_END;
  }
  return ok;
}

/* ---- in-place enhance operators (the reference's hooks AccelerateContrastImage, AccelerateModulateImage,
   AccelerateGrayscaleImage, AccelerateFunctionImage; accelerate-private.h:50-60) ----------------------------------------
   b200_channels[_masked] declines PseudoClass, CMYK, masks and the rest: the CPU path then serves them (and the colormap
   step of Contrast / Modulate). */
typedef struct {
  int op;                       /* 0 contrast, 1 modulate, 2 grayscale, 3 function */
  int sharpen, colorspace, illuminant, method;
  double brightness, saturation, hue;
  MagickFunction function;
  size_t n;
  const double *params;
} enhance_args;

static MagickBooleanType run_enhance(Image *image, int ch, unsigned update_mask, const enhance_args *a)
{
  MagickBooleanType ok = MagickFalse;
  Quantum *q;
  int rc = MB200_EINVAL;
  if (ch == 0 || mb200_device_count() <= 0) return MagickFalse;
  {
    B200_ATTEMPT_BEGIN;
    q = GetAuthenticPixels(image, 0, 0, image->columns, image->rows, attempt);
    if (q != (Quantum *) NULL && b200_cache_pixels(image, ch, attempt) == (float *) q)
      switch (a->op) {
        case 0: rc = mb200_contrast_image((float *) q, image->columns, image->rows, ch, a->sharpen); break;
        case 1:
          rc = mb200_modulate_image((float *) q, image->columns, image->rows, ch, a->brightness, a->saturation, a->hue,
                                    a->colorspace, a->illuminant);
          break;
        case 2: rc = mb200_grayscale_image((float *) q, image->columns, image->rows, ch, a->method, a->colorspace); break;
        default:
          rc = mb200_function_image((float *) q, image->columns, image->rows, ch, (int) a->function, a->n, a->params,
                                    update_mask);
          break;
      }
    /* on failure nothing was written back: the CPU path starts from the same pixels */
    if (rc == MB200_OK && SyncAuthenticPixels(image, attempt) != MagickFalse) ok = MagickTrue;
    B200_ATTEMPT_END;
  }
  return ok;
}

/* ContrastImage (enhance.c:1370) sets R, G and B whatever the channel mask says; a selection still declines here */
MagickBooleanType B200AccelerateContrastImage(Image *image, const MagickBooleanType sharpen, ExceptionInfo *exception)
{
  enhance_args a;
  (void) exception;
  (void) memset(&a, 0, sizeof(a));
  a.op = 0; a.sharpen = sharpen != MagickFalse ? 1 : 0;
  return run_enhance(image, b200_channels(image), 0u, &a);
}

/* ModulateImage's pixel loop (enhance.c:3800-3898) with the caller's parse: `colorspace` as ParseCommandOption gave it
   (UndefinedColorspace after an unparsable illuminant: HSL).  The LCH spaces' reference white is the "color:illuminant"
   artifact (:3694-3709), read here because the hook's signature does not carry it. */
MagickBooleanType B200AccelerateModulateImage(Image *image, const double percent_brightness, const double percent_hue,
                                              const double percent_saturation, const ColorspaceType colorspace,
                                              ExceptionInfo *exception)
{
  enhance_args a;
  const char *artifact = GetImageArtifact(image, "color:illuminant");
  (void) exception;
  (void) memset(&a, 0, sizeof(a));
  a.op = 1; a.brightness = percent_brightness; a.saturation = percent_saturation; a.hue = percent_hue;
  a.colorspace = (int) colorspace;
  a.illuminant = (int) D65Illuminant;
  if (artifact != (const char *) NULL) {
    const ssize_t type = ParseCommandOption(MagickIlluminantOptions, MagickFalse, artifact);
    a.illuminant = type < 0 ? (int) UndefinedIlluminant : (int) type;
  }
  return run_enhance(image, b200_channels(image), 0u, &a);
}

/* GrayscaleImage's pixel loop (enhance.c:2532-2639): the gray value into channel 0.  The caller does the rest of the hook
   branch (:2503-2511): intensity, type and SetImageColorspace. */
MagickBooleanType B200AccelerateGrayscaleImage(Image *image, const PixelIntensityMethod method, ExceptionInfo *exception)
{
  enhance_args a;
  (void) exception;
  (void) memset(&a, 0, sizeof(a));
  a.op = 2; a.method = (int) method; a.colorspace = (int) image->colorspace;
  return run_enhance(image, b200_channels(image), 0u, &a);
}

/* FunctionImage (statistic.c:1064) on the channels with the Update trait; more than MB200_MAX_FUNCTION_PARAMETERS
   parameters decline in the library */
MagickBooleanType B200AccelerateFunctionImage(Image *image, const MagickFunction function, const size_t number_parameters,
                                              const double *parameters, ExceptionInfo *exception)
{
  enhance_args a;
  unsigned update_mask = 0;
  const int ch = b200_channels_masked(image, &update_mask);
  (void) exception;
  (void) memset(&a, 0, sizeof(a));
  a.op = 3; a.function = function; a.n = number_parameters; a.params = parameters;
  return run_enhance(image, ch, update_mask, &a);
}

/* ---- level and stretch operators (enhance.c; AccelerateContrastStretchImage is accelerate-private.h:52) ------------------
   b200_channels_masked gives the Update channels and declines PseudoClass (the colormap step stays on the CPU path), CMYK
   and the rest.  The histogram operators index the histogram by GetPixelIntensity: equalize_eligible. */
typedef struct {
  int op;                       /* 0 level, 1 levelize, 2 minmax stretch, 3 gamma, 4 contrast stretch, 5 linear stretch */
  double a, b, gamma;
  float black[4], white[4];     /* contrast stretch: the bins per channel */
  double black_bin, white_bin;  /* linear stretch */
} level_args;

static MagickBooleanType run_level(Image *image, level_args *a)
{
  MagickBooleanType ok = MagickFalse;
  unsigned update_mask = 0;
  const int ch = b200_channels_masked(image, &update_mask);
  const int per_channel = image->channel_mask != AllChannels ? 1 : 0;
  Quantum *q;
  int rc = MB200_EINVAL;
  if (ch == 0 || mb200_device_count() <= 0) return MagickFalse;
  {
    B200_ATTEMPT_BEGIN;
    q = GetAuthenticPixels(image, 0, 0, image->columns, image->rows, attempt);
    if (q != (Quantum *) NULL && b200_cache_pixels(image, ch, attempt) == (float *) q) {
      float *buf = (float *) q;
      const size_t w = image->columns, h = image->rows;
      switch (a->op) {
        case 0: rc = mb200_level_image(buf, w, h, ch, a->a, a->b, a->gamma, update_mask); break;
        case 1: rc = mb200_levelize_image(buf, w, h, ch, a->a, a->b, a->gamma, update_mask); break;
        case 2: rc = mb200_minmax_stretch_image(buf, w, h, ch, a->a, a->b, a->gamma, per_channel, update_mask); break;
        case 3: rc = mb200_gamma_image(buf, w, h, ch, a->gamma, update_mask); break;
        case 4:
          rc = mb200_contrast_stretch_image(buf, w, h, ch, a->a, a->b, per_channel, update_mask, a->black, a->white);
          break;
        default:
          rc = mb200_linear_stretch_image(buf, w, h, ch, a->a, a->b, update_mask, &a->black_bin, &a->white_bin);
          break;
      }
    }
    /* on failure nothing was written back: the CPU path starts from the same pixels */
    if (rc == MB200_OK && SyncAuthenticPixels(image, attempt) != MagickFalse) ok = MagickTrue;
    B200_ATTEMPT_END;
  }
  return ok;
}

MagickBooleanType B200AccelerateLevelImage(Image *image, const double black_point, const double white_point,
                                           const double gamma, ExceptionInfo *exception)
{
  level_args a;
  (void) exception;
  (void) memset(&a, 0, sizeof(a));
  a.op = 0; a.a = black_point; a.b = white_point; a.gamma = gamma;
  return run_level(image, &a);
}

MagickBooleanType B200AccelerateLevelizeImage(Image *image, const double black_point, const double white_point,
                                              const double gamma, ExceptionInfo *exception)
{
  level_args a;
  (void) exception;
  (void) memset(&a, 0, sizeof(a));
  a.op = 1; a.a = black_point; a.b = white_point; a.gamma = gamma;
  return run_level(image, &a);
}

/* MinMaxStretchImage (histogram.c:927), AutoLevelImage's body: the per-channel loop runs in the library */
MagickBooleanType B200AccelerateMinMaxStretchImage(Image *image, const double black, const double white,
                                                   const double gamma, ExceptionInfo *exception)
{
  level_args a;
  (void) exception;
  (void) memset(&a, 0, sizeof(a));
  a.op = 2; a.a = black; a.b = white; a.gamma = gamma;
  return run_level(image, &a);
}

/* GammaImage (enhance.c:2322), with its image->gamma update (:2441-2442) */
MagickBooleanType B200AccelerateGammaImage(Image *image, const double gamma, ExceptionInfo *exception)
{
  level_args a;
  (void) exception;
  (void) memset(&a, 0, sizeof(a));
  a.op = 3; a.gamma = gamma;
  if (run_level(image, &a) == MagickFalse) return MagickFalse;
  if (gamma != 1.0 && image->gamma != 0.0) image->gamma *= gamma;
  return MagickTrue;
}

/* ContrastStretchImage (enhance.c:1544) with the reference's control plane: IdentifyImageType's gray test (:1589-1591; the
   pixel scan on the device), SetImageColorspace(GRAY), the stretch, then the property with the reference's own
   GetPixelIntensity and FormatLocaleString (:1810-1814). */
MagickBooleanType B200AccelerateContrastStretchImage(Image *image, const double black_point, const double white_point,
                                                     ExceptionInfo *exception)
{
  level_args a;
  Quantum black[MaxPixelChannels], white[MaxPixelChannels];
  char property[MagickPathExtent];
  unsigned mask = 0;
  int ch, i, gray = 0;
  if (mb200_device_count() <= 0) return MagickFalse;
  if (image->channel_mask == AllChannels && equalize_eligible(image) == MagickFalse) return MagickFalse;
  ch = b200_channels_masked(image, &mask);
  if (ch == 0) return MagickFalse;
  if (IsImageGray(image) != MagickFalse) gray = 1;                     /* IdentifyImageGray (attribute.c:1583-1584) */
  else if (IssRGBCompatibleColorspace(image->colorspace) != MagickFalse) {
    /* the cache itself (its HBM copy when attached): no GetVirtualPixels, which would pull a resident result back */
    const float *p = b200_cache_pixels(image, ch, exception);
    int type = 0;
    if (p == (const float *) NULL || mb200_identify_gray(p, image->columns, image->rows, ch, &type) != MB200_OK)
      return MagickFalse;
    gray = type != 0;
  }
  if (gray != 0) (void) SetImageColorspace(image, GRAYColorspace, exception);
  (void) memset(&a, 0, sizeof(a));
  a.op = 4; a.a = black_point; a.b = white_point;
  if (run_level(image, &a) == MagickFalse) return MagickFalse;
  (void) memset(black, 0, sizeof(black));
  (void) memset(white, 0, sizeof(white));
  for (i = 0; i < 4; i++) { black[i] = (Quantum) a.black[i]; white[i] = (Quantum) a.white[i]; }
  (void) FormatLocaleString(property, MagickPathExtent, "%gx%g%%", 100.0 * QuantumScale * GetPixelIntensity(image, black),
                            100.0 * QuantumScale * GetPixelIntensity(image, white));
  (void) SetImageProperty(image, "histogram:contrast-stretch", property, exception);
  return MagickTrue;
}

/* NormalizeImage (enhance.c:4130): its ContrastStretchImage call stays inside enhance.o, so it is wrapped itself */
MagickBooleanType B200AccelerateNormalizeImage(Image *image, ExceptionInfo *exception)
{
  const double black_point = 0.02 * image->columns * image->rows, white_point = 0.99 * image->columns * image->rows;
  return B200AccelerateContrastStretchImage(image, black_point, white_point, exception);
}

/* LinearStretchImage (enhance.c:3347): one intensity histogram, LevelImage, the property (:3421-3424) */
MagickBooleanType B200AccelerateLinearStretchImage(Image *image, const double black_point, const double white_point,
                                                   ExceptionInfo *exception)
{
  level_args a;
  char property[MagickPathExtent];
  if (equalize_eligible(image) == MagickFalse) return MagickFalse;
  (void) memset(&a, 0, sizeof(a));
  a.op = 5; a.a = black_point; a.b = white_point;
  if (run_level(image, &a) == MagickFalse) return MagickFalse;
  (void) FormatLocaleString(property, MagickPathExtent, "%gx%g%%", 100.0 * (ssize_t) a.black_bin / MaxMap,
                            100.0 * (ssize_t) a.white_bin / MaxMap);
  (void) SetImageProperty(image, "histogram:linear-stretch", property, exception);
  return MagickTrue;
}

static int op_emboss(const float *s, float *d, size_t w, size_t h, int ch, const void *a)
{ const blur_args *b = (const blur_args *) a; return mb200_emboss_image(s, d, w, h, ch, b->radius, b->sigma); }

Image *B200AccelerateEmbossImage(const Image *image, const double radius, const double sigma, ExceptionInfo *exception)
{
  blur_args a;
  if (has_artifact(image, morphology_artifacts) != MagickFalse) return (Image *) NULL;
  if (equalize_eligible(image) == MagickFalse || (image->channel_mask & SyncChannels) == 0) return (Image *) NULL;
  a.radius = radius; a.sigma = sigma; a.gain = 0.0; a.threshold = 0.0;
  return run_same_size(image, op_emboss, &a, exception);
}

/* ---- StatisticImage (statistic.c:2918), RotationalBlurImage (effect.c:3129), BilateralBlurImage (effect.c:821) -------------- */
typedef struct { int type; size_t width, height; double a, b, c; } stencil_args;
static int op_statistic(const float *s, float *d, size_t w, size_t h, int ch, const void *a)
{ const stencil_args *t = (const stencil_args *) a; return mb200_statistic_image(s, d, w, h, ch, t->type, t->width, t->height); }
static int op_rotational(const float *s, float *d, size_t w, size_t h, int ch, const void *a)
{ const stencil_args *t = (const stencil_args *) a; return mb200_rotational_blur_image(s, d, w, h, ch, t->a); }
static int op_bilateral(const float *s, float *d, size_t w, size_t h, int ch, const void *a)
{ const stencil_args *t = (const stencil_args *) a; return mb200_bilateral_blur_image(s, d, w, h, ch, t->width, t->height, t->a, t->b); }

Image *B200AccelerateStatisticImage(const Image *image, const StatisticType type, const size_t width, const size_t height,
                                    ExceptionInfo *exception)
{
  stencil_args a;
  switch (type) {
    case GradientStatistic: case MaximumStatistic: case MeanStatistic: case MedianStatistic: case MinimumStatistic:
    case ModeStatistic: case NonpeakStatistic:
    case RootMeanSquareStatistic: case StandardDeviationStatistic: case ContrastStatistic: break;
    default: return (Image *) NULL;
  }
  a.type = (int) type; a.width = width; a.height = height; a.a = a.b = a.c = 0.0;
  return run_same_size(image, op_statistic, &a, exception);
}

Image *B200AccelerateRotationalBlurImage(const Image *image, const double angle, ExceptionInfo *exception)
{
  stencil_args a;
  a.type = 0; a.width = a.height = 0; a.a = angle; a.b = a.c = 0.0;
  return run_same_size(image, op_rotational, &a, exception);
}

Image *B200AccelerateBilateralBlurImage(const Image *image, const size_t width, const size_t height,
                                        const double intensity_sigma, const double spatial_sigma, ExceptionInfo *exception)
{
  stencil_args a;
  if (equalize_eligible(image) == MagickFalse) return (Image *) NULL;        /* tonal weights use GetPixelIntensity */
  a.type = 0; a.width = width; a.height = height; a.a = intensity_sigma; a.b = spatial_sigma; a.c = 0.0;
  return run_same_size(image, op_bilateral, &a, exception);
}

/* AdaptiveBlurImage (effect.c:128) / AdaptiveSharpenImage (:447).  AutoLevelImage takes its all-channels branch only for the
   default mask (histogram.c:942) and EdgeImage / BlurImage read the convolve artifacts: anything else declines. */
static int op_adaptive_blur(const float *s, float *d, size_t w, size_t h, int ch, const void *a)
{ const blur_args *b = (const blur_args *) a; return mb200_adaptive_blur_image(s, d, w, h, ch, b->radius, b->sigma); }
static int op_adaptive_sharpen(const float *s, float *d, size_t w, size_t h, int ch, const void *a)
{ const blur_args *b = (const blur_args *) a; return mb200_adaptive_sharpen_image(s, d, w, h, ch, b->radius, b->sigma); }

static Image *adaptive(const Image *image, same_size_op op, const double radius, const double sigma, ExceptionInfo *exception)
{
  blur_args a;
  if (has_artifact(image, morphology_artifacts) != MagickFalse) return (Image *) NULL;
  if (equalize_eligible(image) == MagickFalse || image->channel_mask != AllChannels) return (Image *) NULL;
  a.radius = radius; a.sigma = sigma; a.gain = 0.0; a.threshold = 0.0;
  return run_same_size(image, op, &a, exception);
}

Image *B200AccelerateAdaptiveBlurImage(const Image *image, const double radius, const double sigma, ExceptionInfo *exception)
{ return adaptive(image, op_adaptive_blur, radius, sigma, exception); }
Image *B200AccelerateAdaptiveSharpenImage(const Image *image, const double radius, const double sigma, ExceptionInfo *exception)
{ return adaptive(image, op_adaptive_sharpen, radius, sigma, exception); }

/* SelectiveBlurImage (effect.c:3406): one stage, so channel selections are exact (unselected channels copy the centre) */
static int op_selective(const float *s, float *d, size_t w, size_t h, int ch, const void *a)
{ const stencil_args *t = (const stencil_args *) a; return mb200_selective_blur_image(s, d, w, h, ch, t->a, t->b, t->c); }

Image *B200AccelerateSelectiveBlurImage(const Image *image, const double radius, const double sigma, const double threshold,
                                        ExceptionInfo *exception)
{
  stencil_args a;
  if (equalize_eligible(image) == MagickFalse) return (Image *) NULL;        /* contrast uses GetPixelIntensity */
  a.type = 0; a.width = a.height = 0; a.a = radius; a.b = sigma; a.c = threshold;
  return run_same_size_masked(image, op_selective, &a, 1, exception);
}

/* ---- DespeckleImage (effect.c:1308), LocalContrastImage (effect.c:2013), WaveletDenoiseImage (visual-effects.c:3515) -----
   Despeckle skips Copy-trait channels (:1412) and LocalContrast updates only R, G, B with the Update trait (:2249-2260):
   both leave unselected channels as the source has them, so a -channel selection is served with the restore pass.
   WaveletDenoise tests only for an Undefined trait (visual-effects.c:3607-3614): it denoises R, G and B whatever the
   selection, and so does the GPU path. */
typedef struct { double a, b; } hook_args;
static int op_despeckle(const float *s, float *d, size_t w, size_t h, int ch, const void *a)
{ (void) a; return mb200_despeckle_image(s, d, w, h, ch); }
static int op_local_contrast(const float *s, float *d, size_t w, size_t h, int ch, const void *a)
{ const hook_args *t = (const hook_args *) a; return mb200_local_contrast_image(s, d, w, h, ch, t->a, t->b); }
static int op_wavelet_denoise(const float *s, float *d, size_t w, size_t h, int ch, const void *a)
{ const hook_args *t = (const hook_args *) a; return mb200_wavelet_denoise_image(s, d, w, h, ch, t->a, t->b); }

Image *B200AccelerateDespeckleImage(const Image *image, ExceptionInfo *exception)
{ return run_same_size_masked(image, op_despeckle, (const void *) NULL, 1, exception); }

Image *B200AccelerateLocalContrastImage(const Image *image, const double radius, const double strength,
                                        ExceptionInfo *exception)
{
  hook_args a;
  a.a = radius; a.b = strength;
  return run_same_size_masked(image, op_local_contrast, &a, 1, exception);
}

/* accelerate-private.h:48 declares AccelerateWaveletDenoiseImage(image, threshold, exception): the softness argument of
   WaveletDenoiseImage does not reach the hook, so a build that patched the #if OPENCL call site with it would denoise
   every image with softness 0.  This hook takes softness, so a call site passes the caller's value through. */
Image *B200AccelerateWaveletDenoiseImage(const Image *image, const double threshold, const double softness,
                                         ExceptionInfo *exception)
{
  hook_args a;
  a.a = threshold; a.b = softness;
  return run_same_size_masked(image, op_wavelet_denoise, &a, 2, exception);
}

/* ---- ld --wrap entry points ------------------------------------------------------------------------------ */
extern Image *__real_BlurImage(const Image *, const double, const double, ExceptionInfo *);
extern Image *__real_GaussianBlurImage(const Image *, const double, const double, ExceptionInfo *);
extern Image *__real_ConvolveImage(const Image *, const KernelInfo *, ExceptionInfo *);
extern Image *__real_UnsharpMaskImage(const Image *, const double, const double, const double, const double,
                                      ExceptionInfo *);
extern Image *__real_MorphologyImage(const Image *, const MorphologyMethod, const ssize_t, const KernelInfo *,
                                     ExceptionInfo *);
extern Image *__real_ResizeImage(const Image *, const size_t, const size_t, const FilterType, ExceptionInfo *);
extern MagickBooleanType __real_TransformImageColorspace(Image *, const ColorspaceType, ExceptionInfo *);
extern Image *__real_SampleImage(const Image *, const size_t, const size_t, ExceptionInfo *);
extern Image *__real_SharpenImage(const Image *, const double, const double, ExceptionInfo *);
extern Image *__real_EdgeImage(const Image *, const double, ExceptionInfo *);
extern MagickBooleanType __real_BilevelImage(Image *, const double, ExceptionInfo *);
extern MagickBooleanType __real_BlackThresholdImage(Image *, const char *, ExceptionInfo *);
extern MagickBooleanType __real_WhiteThresholdImage(Image *, const char *, ExceptionInfo *);
extern MagickBooleanType __real_ClampImage(Image *, ExceptionInfo *);
extern Image *__real_AdaptiveThresholdImage(const Image *, const size_t, const size_t, const double, ExceptionInfo *);
extern MagickBooleanType __real_AutoThresholdImage(Image *, const AutoThresholdMethod, ExceptionInfo *);
extern MagickBooleanType __real_RangeThresholdImage(Image *, const double, const double, const double, const double,
                                                    ExceptionInfo *);
extern MagickBooleanType __real_PerceptibleImage(Image *, const double, ExceptionInfo *);

static long b200_hits = 0, b200_fallbacks = 0;          /* updated with atomic adds: the entry points are re-entrant */
static int b200_enabled = -1;       /* -1: not yet read from the environment */
#define B200_COUNT(var) ((void) __atomic_fetch_add(&(var), 1L, __ATOMIC_RELAXED))
long B200ShimHits(void) { return __atomic_load_n(&b200_hits, __ATOMIC_RELAXED); }
long B200ShimFallbacks(void) { return __atomic_load_n(&b200_fallbacks, __ATOMIC_RELAXED); }
/* Runtime switch (also: environment MAGICK_B200_DISABLE=1), e.g. to A/B against the CPU path. */
void B200ShimEnable(int on) { b200_enabled = on ? 1 : 0; }
static int b200_on(void)
{
  if (b200_enabled < 0) {
    const char *e = getenv("MAGICK_B200_DISABLE");
    b200_enabled = (e != (const char *) NULL && *e != '\0' && *e != '0') ? 0 : 1;
  }
  return b200_enabled;
}
#define TRY(expr) do { if (b200_on()) { Image *r_ = (expr); if (r_ != (Image *) NULL) { B200_COUNT(b200_hits); return r_; } B200_COUNT(b200_fallbacks); } } while (0)

Image *__wrap_BlurImage(const Image *image, const double radius, const double sigma, ExceptionInfo *exception)
{
  TRY(B200AccelerateBlurImage(image, radius, sigma, exception));
  return __real_BlurImage(image, radius, sigma, exception);
}

Image *__wrap_GaussianBlurImage(const Image *image, const double radius, const double sigma,
                                ExceptionInfo *exception)
{
  TRY(B200AccelerateGaussianBlurImage(image, radius, sigma, exception));
  return __real_GaussianBlurImage(image, radius, sigma, exception);
}

Image *__wrap_ConvolveImage(const Image *image, const KernelInfo *kernel, ExceptionInfo *exception)
{
  TRY(B200AccelerateMorphologyImage(image, ConvolveMorphology, 1, kernel, exception));
  return __real_ConvolveImage(image, kernel, exception);
}

Image *__wrap_UnsharpMaskImage(const Image *image, const double radius, const double sigma, const double gain,
                               const double threshold, ExceptionInfo *exception)
{
  TRY(B200AccelerateUnsharpMaskImage(image, radius, sigma, gain, threshold, exception));
  return __real_UnsharpMaskImage(image, radius, sigma, gain, threshold, exception);
}

Image *__wrap_MorphologyImage(const Image *image, const MorphologyMethod method, const ssize_t iterations,
                              const KernelInfo *kernel, ExceptionInfo *exception)
{
  TRY(B200AccelerateMorphologyImage(image, method, iterations, kernel, exception));
  return __real_MorphologyImage(image, method, iterations, kernel, exception);
}

Image *__wrap_ResizeImage(const Image *image, const size_t columns, const size_t rows, const FilterType filter,
                          ExceptionInfo *exception)
{
  TRY(B200AccelerateResizeImage(image, columns, rows, filter, exception));
  return __real_ResizeImage(image, columns, rows, filter, exception);
}

MagickBooleanType __wrap_TransformImageColorspace(Image *image, const ColorspaceType colorspace,
                                                  ExceptionInfo *exception)
{
  if (b200_on()) {
    if (B200AccelerateTransformImageColorspace(image, colorspace, exception) != MagickFalse) {
      B200_COUNT(b200_hits);
      return MagickTrue;
    }
    B200_COUNT(b200_fallbacks);
  }
  return __real_TransformImageColorspace(image, colorspace, exception);
}

#define TRY_BOOL(expr) do { if (b200_on()) { if ((expr) != MagickFalse) { B200_COUNT(b200_hits); return MagickTrue; } B200_COUNT(b200_fallbacks); } } while (0)

MagickBooleanType __wrap_BilevelImage(Image *image, const double threshold, ExceptionInfo *exception)
{
  TRY_BOOL(B200AccelerateBilevelImage(image, threshold, exception));
  return __real_BilevelImage(image, threshold, exception);
}

MagickBooleanType __wrap_BlackThresholdImage(Image *image, const char *thresholds, ExceptionInfo *exception)
{
  TRY_BOOL(B200AccelerateBlackThresholdImage(image, thresholds, exception));
  return __real_BlackThresholdImage(image, thresholds, exception);
}

MagickBooleanType __wrap_WhiteThresholdImage(Image *image, const char *thresholds, ExceptionInfo *exception)
{
  TRY_BOOL(B200AccelerateWhiteThresholdImage(image, thresholds, exception));
  return __real_WhiteThresholdImage(image, thresholds, exception);
}

MagickBooleanType __wrap_ClampImage(Image *image, ExceptionInfo *exception)
{
  TRY_BOOL(B200AccelerateClampImage(image, exception));
  return __real_ClampImage(image, exception);
}

Image *__wrap_AdaptiveThresholdImage(const Image *image, const size_t width, const size_t height, const double bias,
                                     ExceptionInfo *exception)
{
  TRY(B200AccelerateAdaptiveThresholdImage(image, width, height, bias, exception));
  return __real_AdaptiveThresholdImage(image, width, height, bias, exception);
}

MagickBooleanType __wrap_AutoThresholdImage(Image *image, const AutoThresholdMethod method, ExceptionInfo *exception)
{
  TRY_BOOL(B200AccelerateAutoThresholdImage(image, method, exception));
  return __real_AutoThresholdImage(image, method, exception);
}

MagickBooleanType __wrap_RangeThresholdImage(Image *image, const double low_black, const double low_white,
                                             const double high_white, const double high_black, ExceptionInfo *exception)
{
  TRY_BOOL(B200AccelerateRangeThresholdImage(image, low_black, low_white, high_white, high_black, exception));
  return __real_RangeThresholdImage(image, low_black, low_white, high_white, high_black, exception);
}

MagickBooleanType __wrap_PerceptibleImage(Image *image, const double epsilon, ExceptionInfo *exception)
{
  TRY_BOOL(B200AcceleratePerceptibleImage(image, epsilon, exception));
  return __real_PerceptibleImage(image, epsilon, exception);
}

Image *__wrap_SharpenImage(const Image *image, const double radius, const double sigma, ExceptionInfo *exception)
{
  TRY(B200AccelerateSharpenImage(image, radius, sigma, exception));
  return __real_SharpenImage(image, radius, sigma, exception);
}

Image *__wrap_EdgeImage(const Image *image, const double radius, ExceptionInfo *exception)
{
  TRY(B200AccelerateEdgeImage(image, radius, exception));
  return __real_EdgeImage(image, radius, exception);
}

extern Image *__real_StatisticImage(const Image *, const StatisticType, const size_t, const size_t, ExceptionInfo *);
extern Image *__real_RotationalBlurImage(const Image *, const double, ExceptionInfo *);
extern Image *__real_BilateralBlurImage(const Image *, const size_t, const size_t, const double, const double, ExceptionInfo *);

Image *__wrap_StatisticImage(const Image *image, const StatisticType type, const size_t width, const size_t height,
                             ExceptionInfo *exception)
{
  TRY(B200AccelerateStatisticImage(image, type, width, height, exception));
  return __real_StatisticImage(image, type, width, height, exception);
}

Image *__wrap_RotationalBlurImage(const Image *image, const double angle, ExceptionInfo *exception)
{
  TRY(B200AccelerateRotationalBlurImage(image, angle, exception));
  return __real_RotationalBlurImage(image, angle, exception);
}

Image *__wrap_BilateralBlurImage(const Image *image, const size_t width, const size_t height, const double intensity_sigma,
                                 const double spatial_sigma, ExceptionInfo *exception)
{
  TRY(B200AccelerateBilateralBlurImage(image, width, height, intensity_sigma, spatial_sigma, exception));
  return __real_BilateralBlurImage(image, width, height, intensity_sigma, spatial_sigma, exception);
}

extern Image *__real_DespeckleImage(const Image *, ExceptionInfo *);
extern Image *__real_LocalContrastImage(const Image *, const double, const double, ExceptionInfo *);
extern Image *__real_WaveletDenoiseImage(const Image *, const double, const double, ExceptionInfo *);

Image *__wrap_DespeckleImage(const Image *image, ExceptionInfo *exception)
{
  TRY(B200AccelerateDespeckleImage(image, exception));
  return __real_DespeckleImage(image, exception);
}

Image *__wrap_LocalContrastImage(const Image *image, const double radius, const double strength, ExceptionInfo *exception)
{
  TRY(B200AccelerateLocalContrastImage(image, radius, strength, exception));
  return __real_LocalContrastImage(image, radius, strength, exception);
}

Image *__wrap_WaveletDenoiseImage(const Image *image, const double threshold, const double softness,
                                  ExceptionInfo *exception)
{
  TRY(B200AccelerateWaveletDenoiseImage(image, threshold, softness, exception));
  return __real_WaveletDenoiseImage(image, threshold, softness, exception);
}

extern Image *__real_AdaptiveBlurImage(const Image *, const double, const double, ExceptionInfo *);
extern Image *__real_AdaptiveSharpenImage(const Image *, const double, const double, ExceptionInfo *);
Image *__wrap_AdaptiveBlurImage(const Image *image, const double radius, const double sigma, ExceptionInfo *exception)
{
  TRY(B200AccelerateAdaptiveBlurImage(image, radius, sigma, exception));
  return __real_AdaptiveBlurImage(image, radius, sigma, exception);
}
Image *__wrap_AdaptiveSharpenImage(const Image *image, const double radius, const double sigma, ExceptionInfo *exception)
{
  TRY(B200AccelerateAdaptiveSharpenImage(image, radius, sigma, exception));
  return __real_AdaptiveSharpenImage(image, radius, sigma, exception);
}

extern Image *__real_SelectiveBlurImage(const Image *, const double, const double, const double, ExceptionInfo *);
Image *__wrap_SelectiveBlurImage(const Image *image, const double radius, const double sigma, const double threshold,
                                 ExceptionInfo *exception)
{
  TRY(B200AccelerateSelectiveBlurImage(image, radius, sigma, threshold, exception));
  return __real_SelectiveBlurImage(image, radius, sigma, threshold, exception);
}

extern Image *__real_EmbossImage(const Image *, const double, const double, ExceptionInfo *);
extern MagickBooleanType __real_EqualizeImage(Image *, ExceptionInfo *);

Image *__wrap_EmbossImage(const Image *image, const double radius, const double sigma, ExceptionInfo *exception)
{
  TRY(B200AccelerateEmbossImage(image, radius, sigma, exception));
  return __real_EmbossImage(image, radius, sigma, exception);
}

MagickBooleanType __wrap_EqualizeImage(Image *image, ExceptionInfo *exception)
{
  TRY_BOOL(B200AccelerateEqualizeImage(image, exception));
  return __real_EqualizeImage(image, exception);
}

extern MagickBooleanType __real_ContrastImage(Image *, const MagickBooleanType, ExceptionInfo *);
extern MagickBooleanType __real_ModulateImage(Image *, const char *, ExceptionInfo *);
extern MagickBooleanType __real_GrayscaleImage(Image *, const PixelIntensityMethod, ExceptionInfo *);
extern MagickBooleanType __real_FunctionImage(Image *, const MagickFunction, const size_t, const double *, ExceptionInfo *);

MagickBooleanType __wrap_ContrastImage(Image *image, const MagickBooleanType sharpen, ExceptionInfo *exception)
{
  TRY_BOOL(B200AccelerateContrastImage(image, sharpen, exception));
  return __real_ContrastImage(image, sharpen, exception);
}

/* ModulateImage's set-up (enhance.c:3677-3710): the re-tag, ParseGeometry and the two artifacts, as the reference does
   them before its hook */
MagickBooleanType __wrap_ModulateImage(Image *image, const char *modulate, ExceptionInfo *exception)
{
  if (b200_on() && modulate != (const char *) NULL) {
    ColorspaceType colorspace = UndefinedColorspace;
    double brightness = 100.0, saturation = 100.0, hue = 100.0;
    GeometryInfo geometry_info;
    MagickStatusType flags;
    const char *artifact;
    if (IssRGBCompatibleColorspace(image->colorspace) == MagickFalse)
      (void) SetImageColorspace(image, sRGBColorspace, exception);
    flags = ParseGeometry(modulate, &geometry_info);
    if ((flags & RhoValue) != 0) brightness = geometry_info.rho;
    if ((flags & SigmaValue) != 0) saturation = geometry_info.sigma;
    if ((flags & XiValue) != 0) hue = geometry_info.xi;
    artifact = GetImageArtifact(image, "modulate:colorspace");
    if (artifact != (const char *) NULL)
      colorspace = (ColorspaceType) ParseCommandOption(MagickColorspaceOptions, MagickFalse, artifact);
    artifact = GetImageArtifact(image, "color:illuminant");
    if (artifact != (const char *) NULL && ParseCommandOption(MagickIlluminantOptions, MagickFalse, artifact) < 0)
      colorspace = UndefinedColorspace;
    TRY_BOOL(B200AccelerateModulateImage(image, brightness, hue, saturation, colorspace, exception));
  }
  return __real_ModulateImage(image, modulate, exception);
}

/* GrayscaleImage's hook branch (enhance.c:2503-2511) */
MagickBooleanType __wrap_GrayscaleImage(Image *image, const PixelIntensityMethod method, ExceptionInfo *exception)
{
  if (b200_on()) {
    if (B200AccelerateGrayscaleImage(image, method, exception) != MagickFalse) {
      B200_COUNT(b200_hits);
      image->intensity = method;
      image->type = GrayscaleType;
      if ((method == Rec601LuminancePixelIntensityMethod) || (method == Rec709LuminancePixelIntensityMethod))
        return SetImageColorspace(image, LinearGRAYColorspace, exception);
      return SetImageColorspace(image, GRAYColorspace, exception);
    }
    B200_COUNT(b200_fallbacks);
  }
  return __real_GrayscaleImage(image, method, exception);
}

MagickBooleanType __wrap_FunctionImage(Image *image, const MagickFunction function, const size_t number_parameters,
                                       const double *parameters, ExceptionInfo *exception)
{
  TRY_BOOL(B200AccelerateFunctionImage(image, function, number_parameters, parameters, exception));
  return __real_FunctionImage(image, function, number_parameters, parameters, exception);
}

extern MagickBooleanType __real_ContrastStretchImage(Image *, const double, const double, ExceptionInfo *);
extern MagickBooleanType __real_NormalizeImage(Image *, ExceptionInfo *);
extern MagickBooleanType __real_LinearStretchImage(Image *, const double, const double, ExceptionInfo *);
extern MagickBooleanType __real_LevelImage(Image *, const double, const double, const double, ExceptionInfo *);
extern MagickBooleanType __real_LevelizeImage(Image *, const double, const double, const double, ExceptionInfo *);
extern MagickBooleanType __real_MinMaxStretchImage(Image *, const double, const double, const double, ExceptionInfo *);
extern MagickBooleanType __real_GammaImage(Image *, const double, ExceptionInfo *);

MagickBooleanType __wrap_ContrastStretchImage(Image *image, const double black_point, const double white_point,
                                              ExceptionInfo *exception)
{
  TRY_BOOL(B200AccelerateContrastStretchImage(image, black_point, white_point, exception));
  return __real_ContrastStretchImage(image, black_point, white_point, exception);
}

extern Image *__real_DistortImage(const Image *, const DistortMethod, const size_t, const double *, MagickBooleanType,
                                  ExceptionInfo *);
extern Image *__real_RotateImage(const Image *, const double, ExceptionInfo *);

Image *__wrap_DistortImage(const Image *image, const DistortMethod method, const size_t number_arguments,
                           const double *arguments, MagickBooleanType bestfit, ExceptionInfo *exception)
{
  TRY(B200AccelerateDistortImage(image, method, number_arguments, arguments, bestfit, exception));
  return __real_DistortImage(image, method, number_arguments, arguments, bestfit, exception);
}

Image *__wrap_RotateImage(const Image *image, const double degrees, ExceptionInfo *exception)
{
  TRY(B200AccelerateRotateImage(image, degrees, exception));
  return __real_RotateImage(image, degrees, exception);
}

/* ---- the orientation and crop operators (transform.c, shear.c) -------------------------------------------------------
   mb200_geometry_plan gives the output's size and page; the result is CloneImage(image, columns, rows) as the reference
   clones it, its pixels written by mb200_geometry_image, then the page and type the reference sets.  Calls between these
   operators inside transform.o (AutoOrientImage -> FlipImage, CropImageToTiles / ShaveImage -> CropImage) and from
   distort.o's RotateImage to shear.o's IntegralRotateImage are served by the wraps of their callers or cross objects.
   NULL == declined, with the caller's exception untouched: no device, a layout the library does not take (CMYK,
   PseudoClass, masks, meta channels), and the plan's declines (a crop outside the canvas or of zero area, a shave of
   half the image, IntegralRotateImage by 0). */
static Image *b200_run_geometry(const Image *image, int ch, const mb200_geometry_params *p);

static Image *b200_geometry(const Image *image, int op, const long *args)
{
  mb200_geometry_params plan;
  mb200_page page;
  int ch;
  if (mb200_device_count() <= 0) return (Image *) NULL;
  ch = b200_layout_masked(image, (unsigned *) NULL);
  if (ch == 0) return (Image *) NULL;
  page.width = image->page.width; page.height = image->page.height; page.x = (long) image->page.x;
  page.y = (long) image->page.y;
  if (mb200_geometry_plan(op, image->columns, image->rows, &page, args, &plan) != MB200_OK) return (Image *) NULL;
  return b200_run_geometry(image, ch, &plan);
}

/* A plan of mb200_geometry_plan (or mb200_trim_plan) on an image of `ch` channels: the result image, or NULL. */
static Image *b200_run_geometry(const Image *image, int ch, const mb200_geometry_params *p)
{
  const mb200_geometry_params plan = *p;
  Image *out = (Image *) NULL;
  {
    B200_ATTEMPT_BEGIN;
    const float *p = b200_cache_pixels(image, ch, attempt);
    if (p != (const float *) NULL) out = new_result(image, plan.columns, plan.rows, attempt);
    if (out != (Image *) NULL) {
      Quantum *q = GetAuthenticPixels(out, 0, 0, out->columns, out->rows, attempt);
      if (q == (Quantum *) NULL || b200_cache_pixels(out, ch, attempt) != (float *) q ||
          mb200_geometry_image(p, image->columns, image->rows, ch, (float *) q, &plan) != MB200_OK ||
          SyncAuthenticPixels(out, attempt) == MagickFalse)
        out = DestroyImage(out);
    }
    B200_ATTEMPT_END;
  }
  if (out != (Image *) NULL) {
    out->page.width = plan.page.width; out->page.height = plan.page.height;
    out->page.x = (ssize_t) plan.page.x; out->page.y = (ssize_t) plan.page.y;
    out->type = image->type;
  }
  return out;
}

static Image *b200_crop(const Image *image, const RectangleInfo *geometry)
{
  const long args[4] = { (long) geometry->width, (long) geometry->height, (long) geometry->x, (long) geometry->y };
  return b200_geometry(image, MB200_GeometryCrop, args);
}

/* AutoOrientImage (transform.c:103): the reference's dispatch; Undefined / TopLeft (a clone) decline. */
static Image *b200_auto_orient(const Image *image, const OrientationType orientation)
{
  long rotations = 0;
  int op;
  Image *out;
  switch (orientation) {
    case TopRightOrientation: op = MB200_GeometryFlop; break;
    case BottomRightOrientation: op = MB200_GeometryIntegralRotate; rotations = 2; break;   /* RotateImage(180) */
    case BottomLeftOrientation: op = MB200_GeometryFlip; break;
    case LeftTopOrientation: op = MB200_GeometryTranspose; break;
    case RightTopOrientation: op = MB200_GeometryIntegralRotate; rotations = 1; break;     /* RotateImage(90) */
    case RightBottomOrientation: op = MB200_GeometryTransverse; break;
    case LeftBottomOrientation: op = MB200_GeometryIntegralRotate; rotations = 3; break;   /* RotateImage(270) */
    default: return (Image *) NULL;
  }
  out = b200_geometry(image, op, &rotations);
  if (out != (Image *) NULL) out->orientation = TopLeftOrientation;
  return out;
}

/* CropImageToTiles (transform.c:791): the geometry parsed with the reference's own ParseGravityGeometry; the single
   region (with the `!` page fix-up) and the fixed-size WxH tiles as the same loop of served crops.  The `@` tiles and the
   final clone decline, and so does a tile loop any of whose crops declines. */
static Image *b200_crop_to_tiles(const Image *image, const char *crop_geometry)
{
  RectangleInfo geometry;
  MagickStatusType flags;
  ExceptionType severity;
  Image *list = (Image *) NULL;
  if (mb200_device_count() <= 0 || b200_layout_masked(image, (unsigned *) NULL) == 0 ||
      crop_geometry == (const char *) NULL) return (Image *) NULL;
  {
    B200_ATTEMPT_BEGIN;
    flags = ParseGravityGeometry(image, crop_geometry, &geometry, attempt);
    severity = attempt->severity;
    B200_ATTEMPT_END;
  }
  if (severity != UndefinedException || (flags & AreaValue) != 0) return (Image *) NULL;
  if ((geometry.width == 0 && geometry.height == 0) || (flags & XValue) != 0 || (flags & YValue) != 0) {
    list = b200_crop(image, &geometry);
    if (list != (Image *) NULL && (flags & AspectValue) != 0) {
      list->page.width = geometry.width;
      list->page.height = geometry.height;
      list->page.x -= geometry.x;
      list->page.y -= geometry.y;
    }
    return list;
  }
  if (image->columns > geometry.width || image->rows > geometry.height) {
    RectangleInfo page = image->page;
    size_t width, height;
    ssize_t x, y;
    if (page.width == 0) page.width = image->columns;
    if (page.height == 0) page.height = image->rows;
    width = geometry.width == 0 ? page.width : geometry.width;
    height = geometry.height == 0 ? page.height : geometry.height;
    for (y = 0; y < (ssize_t) page.height; y += (ssize_t) height)
      for (x = 0; x < (ssize_t) page.width; x += (ssize_t) width) {
        Image *next;
        geometry.width = width; geometry.height = height; geometry.x = x; geometry.y = y;
        next = b200_crop(image, &geometry);
        if (next == (Image *) NULL) {
          if (list != (Image *) NULL) list = DestroyImageList(list);
          return (Image *) NULL;
        }
        AppendImageToList(&list, next);
      }
    return list;
  }
  return (Image *) NULL;
}

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

Image *__wrap_FlipImage(const Image *image, ExceptionInfo *exception)
{
  TRY(b200_geometry(image, MB200_GeometryFlip, (const long *) NULL));
  return __real_FlipImage(image, exception);
}

Image *__wrap_FlopImage(const Image *image, ExceptionInfo *exception)
{
  TRY(b200_geometry(image, MB200_GeometryFlop, (const long *) NULL));
  return __real_FlopImage(image, exception);
}

Image *__wrap_TransposeImage(const Image *image, ExceptionInfo *exception)
{
  TRY(b200_geometry(image, MB200_GeometryTranspose, (const long *) NULL));
  return __real_TransposeImage(image, exception);
}

Image *__wrap_TransverseImage(const Image *image, ExceptionInfo *exception)
{
  TRY(b200_geometry(image, MB200_GeometryTransverse, (const long *) NULL));
  return __real_TransverseImage(image, exception);
}

Image *__wrap_IntegralRotateImage(const Image *image, size_t rotations, ExceptionInfo *exception)
{
  const long r = (long) (rotations % 4);
  TRY(b200_geometry(image, MB200_GeometryIntegralRotate, &r));
  return __real_IntegralRotateImage(image, rotations, exception);
}

Image *__wrap_CropImage(const Image *image, const RectangleInfo *geometry, ExceptionInfo *exception)
{
  TRY(b200_crop(image, geometry));
  return __real_CropImage(image, geometry, exception);
}

Image *__wrap_CropImageToTiles(const Image *image, const char *crop_geometry, ExceptionInfo *exception)
{
  TRY(b200_crop_to_tiles(image, crop_geometry));
  return __real_CropImageToTiles(image, crop_geometry, exception);
}

Image *__wrap_ShaveImage(const Image *image, const RectangleInfo *shave_info, ExceptionInfo *exception)
{
  const long args[2] = { (long) shave_info->width, (long) shave_info->height };
  TRY(b200_geometry(image, MB200_GeometryShave, args));
  return __real_ShaveImage(image, shave_info, exception);
}

Image *__wrap_RollImage(const Image *image, const ssize_t x_offset, const ssize_t y_offset, ExceptionInfo *exception)
{
  const long args[2] = { (long) x_offset, (long) y_offset };
  TRY(b200_geometry(image, MB200_GeometryRoll, args));
  return __real_RollImage(image, x_offset, y_offset, exception);
}

Image *__wrap_AutoOrientImage(const Image *image, const OrientationType orientation, ExceptionInfo *exception)
{
  TRY(b200_auto_orient(image, orientation));
  return __real_AutoOrientImage(image, orientation, exception);
}

/* ---- GetImageBoundingBox (attribute.c:391) and TrimImage (transform.c:2412) --------------------------------------------
   The box is mb200_bounding_box on the pixel cache, with the image's fuzz, "trim:edges" (split and compared with the
   reference's own StringToken / LocaleCompare) and colourspace.  TrimImage needs a wrap of its own: its call to CropImage
   stays inside transform.o (its call to GetImageBoundingBox crosses objects).  Declined, with the caller's exception
   untouched: no device, a layout the library does not take (CMYK, PseudoClass, masks, meta channels), and
   "trim:percent-background" (GetEdgeBoundingBox, another algorithm); TrimImage also declines an image with an 8bim
   profile (Update8BIMClipPath rewrites its clip path) and the crops mb200_trim_plan declines. */
static int b200_bounding_box(const Image *image, RectangleInfo *box, int *warning)
{
  mb200_trim_options options;
  mb200_page b;
  const char *edges;
  int ch, rc = MB200_EUNSUPPORTED;
  if (mb200_device_count() <= 0 || GetImageArtifact(image, "trim:percent-background") != (const char *) NULL) return 0;
  ch = b200_layout_masked(image, (unsigned *) NULL);
  if (ch == 0) return 0;
  options.fuzz = image->fuzz;
  options.colorspace = (int) image->colorspace;
  options.edges = MB200_TRIM_EDGES_UNSET;
  edges = GetImageArtifact(image, "trim:edges");
  if (edges != (const char *) NULL) {                                        /* attribute.c:442-455 */
    char *copy = AcquireString(edges), *r = copy, *q;
    options.edges = 0;
    while ((q = StringToken(",", &r)) != (char *) NULL) {
      if (LocaleCompare(q, "north") == 0) options.edges |= MB200_TrimEdgeNorth;
      if (LocaleCompare(q, "east") == 0) options.edges |= MB200_TrimEdgeEast;
      if (LocaleCompare(q, "south") == 0) options.edges |= MB200_TrimEdgeSouth;
      if (LocaleCompare(q, "west") == 0) options.edges |= MB200_TrimEdgeWest;
    }
    copy = DestroyString(copy);
  }
  {
    B200_ATTEMPT_BEGIN;
    const float *p = b200_cache_pixels(image, ch, attempt);
    if (p != (const float *) NULL) rc = mb200_bounding_box(p, image->columns, image->rows, ch, &options, &b, warning);
    B200_ATTEMPT_END;
  }
  if (rc != MB200_OK) return 0;
  box->width = b.width; box->height = b.height; box->x = (ssize_t) b.x; box->y = (ssize_t) b.y;
  return 1;
}

static void b200_box_warning(const Image *image, ExceptionInfo *exception)      /* attribute.c:553-555 */
{
  (void) ThrowMagickException(exception, GetMagickModule(), OptionWarning, "GeometryDoesNotContainImage", "`%s'",
                              image->filename);
}

extern RectangleInfo __real_GetImageBoundingBox(const Image *, ExceptionInfo *);
extern Image *__real_TrimImage(const Image *, ExceptionInfo *);

RectangleInfo __wrap_GetImageBoundingBox(const Image *image, ExceptionInfo *exception)
{
  if (b200_on()) {
    RectangleInfo box;
    int warning = 0;
    if (b200_bounding_box(image, &box, &warning)) {
      B200_COUNT(b200_hits);
      if (warning) b200_box_warning(image, exception);
      return box;
    }
    B200_COUNT(b200_fallbacks);
  }
  return __real_GetImageBoundingBox(image, exception);
}

Image *__wrap_TrimImage(const Image *image, ExceptionInfo *exception)
{
  if (b200_on()) {
    RectangleInfo box;
    int warning = 0;
    const int ch = b200_layout_masked(image, (unsigned *) NULL);
    if (ch != 0 && GetImageProfile(image, "8bim") == (const StringInfo *) NULL &&
        b200_bounding_box(image, &box, &warning)) {
      Image *out = (Image *) NULL;
      if (box.width == 0 || box.height == 0) {                               /* transform.c:2429-2444, no pixel read */
        B200_COUNT(b200_hits);
        if (warning) b200_box_warning(image, exception);
        out = CloneImage(image, 1, 1, MagickTrue, exception);
        if (out == (Image *) NULL) return out;
        out->background_color.alpha_trait = BlendPixelTrait;
        out->background_color.alpha = (MagickRealType) TransparentAlpha;
        (void) SetImageBackgroundColor(out, exception);
        out->page = image->page;
        out->page.x = -1;
        out->page.y = -1;
        return out;
      }
      {
        mb200_geometry_params plan;
        mb200_page page, b;
        size_t min_size[2];
        const char *artifact = GetImageArtifact(image, "trim:minSize");
        page.width = image->page.width; page.height = image->page.height;
        page.x = (long) image->page.x; page.y = (long) image->page.y;
        b.width = box.width; b.height = box.height; b.x = (long) box.x; b.y = (long) box.y;
        if (artifact != (const char *) NULL) {                               /* :2445-2448 */
          RectangleInfo size = box;
          (void) ParseAbsoluteGeometry(artifact, &size);
          min_size[0] = size.width; min_size[1] = size.height;
        }
        if (mb200_trim_plan(image->columns, image->rows, &page, &b, (int) image->gravity,
                            artifact != (const char *) NULL ? min_size : (const size_t *) NULL, &plan) == MB200_OK)
          out = b200_run_geometry(image, ch, &plan);
      }
      if (out != (Image *) NULL) {
        B200_COUNT(b200_hits);
        return out;
      }
    }
    B200_COUNT(b200_fallbacks);
  }
  return __real_TrimImage(image, exception);
}

MagickBooleanType __wrap_NormalizeImage(Image *image, ExceptionInfo *exception)
{
  TRY_BOOL(B200AccelerateNormalizeImage(image, exception));
  return __real_NormalizeImage(image, exception);
}

MagickBooleanType __wrap_LinearStretchImage(Image *image, const double black_point, const double white_point,
                                            ExceptionInfo *exception)
{
  TRY_BOOL(B200AccelerateLinearStretchImage(image, black_point, white_point, exception));
  return __real_LinearStretchImage(image, black_point, white_point, exception);
}

MagickBooleanType __wrap_LevelImage(Image *image, const double black_point, const double white_point, const double gamma,
                                    ExceptionInfo *exception)
{
  TRY_BOOL(B200AccelerateLevelImage(image, black_point, white_point, gamma, exception));
  return __real_LevelImage(image, black_point, white_point, gamma, exception);
}

MagickBooleanType __wrap_LevelizeImage(Image *image, const double black_point, const double white_point, const double gamma,
                                       ExceptionInfo *exception)
{
  TRY_BOOL(B200AccelerateLevelizeImage(image, black_point, white_point, gamma, exception));
  return __real_LevelizeImage(image, black_point, white_point, gamma, exception);
}

MagickBooleanType __wrap_MinMaxStretchImage(Image *image, const double black, const double white, const double gamma,
                                            ExceptionInfo *exception)
{
  TRY_BOOL(B200AccelerateMinMaxStretchImage(image, black, white, gamma, exception));
  return __real_MinMaxStretchImage(image, black, white, gamma, exception);
}

MagickBooleanType __wrap_GammaImage(Image *image, const double gamma, ExceptionInfo *exception)
{
  TRY_BOOL(B200AccelerateGammaImage(image, gamma, exception));
  return __real_GammaImage(image, gamma, exception);
}

extern Image *__real_ScaleImage(const Image *, const size_t, const size_t, ExceptionInfo *);
Image *__wrap_ScaleImage(const Image *image, const size_t columns, const size_t rows, ExceptionInfo *exception)
{
  TRY(B200AccelerateScaleImage(image, columns, rows, exception));
  return __real_ScaleImage(image, columns, rows, exception);
}

Image *__wrap_SampleImage(const Image *image, const size_t columns, const size_t rows, ExceptionInfo *exception)
{
  TRY(B200AccelerateSampleImage(image, columns, rows, exception));
  return __real_SampleImage(image, columns, rows, exception);
}

/* ---- ThumbnailImage (resize.c:4591) ------------------------------------------------------------------------------
   Its SampleImage / ResizeImage calls are made from inside resize.o, which --wrap does not redirect, so the pixel
   cascade (:4617-4645) is re-issued here through the wrapped entry points (each stage takes the GPU or declines
   to the CPU on its own).  The metadata half of the reference (page geometry, depth, profile stripping, the
   Thumb::* properties) is NOT restated: the real ThumbnailImage is called on the finished thumbnail with its
   own size -- a same-size call skips the resize block and only applies the metadata, which it derives from
   fields the cascade's CloneImage-based results inherit from the source (filenames, magick_columns/rows, blob,
   properties).  Only the page count refers to the source's image list and is set afterwards. */
extern Image *__real_ThumbnailImage(const Image *, const size_t, const size_t, ExceptionInfo *);

Image *__wrap_ThumbnailImage(const Image *image, const size_t columns, const size_t rows, ExceptionInfo *exception)
{
  Image *clone_image, *stage, *result;
  ssize_t x_factor, y_factor;
  if (!b200_on() || columns == 0 || rows == 0 || ((columns == image->columns) && (rows == image->rows)))
    return __real_ThumbnailImage(image, columns, rows, exception);
  x_factor = (ssize_t) image->columns / (ssize_t) columns;
  y_factor = (ssize_t) image->rows / (ssize_t) rows;
  clone_image = (Image *) NULL;                       /* result of the previous stage (NULL: still the source) */
  if ((x_factor > 4) && (y_factor > 4)) {
    stage = SampleImage(image, 4 * columns, 4 * rows, exception);
    if (stage != (Image *) NULL) clone_image = stage;
  }
  if ((x_factor > 2) && (y_factor > 2)) {
    stage = ResizeImage(clone_image != (Image *) NULL ? clone_image : image, 2 * columns, 2 * rows, BoxFilter, exception);
    if (stage != (Image *) NULL) {
      if (clone_image != (Image *) NULL) clone_image = DestroyImage(clone_image);
      clone_image = stage;
    }
  }
  stage = ResizeImage(clone_image != (Image *) NULL ? clone_image : image, columns, rows,
                      image->filter == UndefinedFilter ? LanczosSharpFilter : image->filter, exception);
  if (clone_image != (Image *) NULL) clone_image = DestroyImage(clone_image);
  if (stage == (Image *) NULL) return (Image *) NULL;
  result = __real_ThumbnailImage(stage, columns, rows, exception);     /* same size: metadata only */
  stage = DestroyImage(stage);
  if (result != (Image *) NULL)
    (void) FormatImageProperty(result, "Thumb::Document::Pages", "%.20g", (double) GetImageListLength(image));
  return result;
}

/* ---- MinifyImage (resize.c:3158) and ResampleImage (:3209): one-line callers of ResizeImage from inside resize.o,
   which --wrap does not redirect; re-issued here through the wrapped ResizeImage. */
extern Image *__real_MinifyImage(const Image *, ExceptionInfo *);
extern Image *__real_ResampleImage(const Image *, const double, const double, const FilterType, ExceptionInfo *);

Image *__wrap_MinifyImage(const Image *image, ExceptionInfo *exception)
{
  if (!b200_on() || image->columns < 2 || image->rows < 2) return __real_MinifyImage(image, exception);
  return ResizeImage(image, image->columns / 2, image->rows / 2, SplineFilter, exception);          /* :3170 */
}

Image *__wrap_ResampleImage(const Image *image, const double x_resolution, const double y_resolution,
                            const FilterType filter, ExceptionInfo *exception)
{
  Image *out;
  size_t width, height;
  if (!b200_on()) return __real_ResampleImage(image, x_resolution, y_resolution, filter, exception);
  width = (size_t) (x_resolution * image->columns / (image->resolution.x == 0.0 ? 72.0 : image->resolution.x) + 0.5);   /* :3230 */
  height = (size_t) (y_resolution * image->rows / (image->resolution.y == 0.0 ? 72.0 : image->resolution.y) + 0.5);
  out = ResizeImage(image, width, height, filter, exception);
  if (out != (Image *) NULL) { out->resolution.x = x_resolution; out->resolution.y = y_resolution; }
  return out;
}

/* ---- MotionBlurImage (effect.c:2347; the reference's own hook is AccelerateMotionBlurImage, :2401) ------------------ */
typedef struct { double radius, sigma, angle; } motion_args;
static int op_motion(const float *s, float *d, size_t w, size_t h, int ch, const void *a)
{ const motion_args *m = (const motion_args *) a; return mb200_motion_blur_image(s, d, w, h, ch, m->radius, m->sigma, m->angle); }

Image *B200AccelerateMotionBlurImage(const Image *image, const double radius, const double sigma, const double angle,
                                     ExceptionInfo *exception)
{
  motion_args a;
  a.radius = radius; a.sigma = sigma; a.angle = angle;
  return run_same_size(image, op_motion, &a, exception);
}

extern Image *__real_MotionBlurImage(const Image *, const double, const double, const double, ExceptionInfo *);
Image *__wrap_MotionBlurImage(const Image *image, const double radius, const double sigma, const double angle,
                              ExceptionInfo *exception)
{
  TRY(B200AccelerateMotionBlurImage(image, radius, sigma, angle, exception));
  return __real_MotionBlurImage(image, radius, sigma, angle, exception);
}

/* ---- pixel caches in pinned host memory --------------------------------------------------------------------------------
   OpenPixelCache takes a memory cache's pixels from AcquireAlignedMemory (cache.c:3757), and that function honours the
   public SetMagickAlignedMemoryMethods hook (memory.c:376, :1541).  B200ShimInstallPixelCachePool() installs an allocator
   that serves large blocks (pixel caches) from a recycling pool of CUDA-pinned host memory and attaches each block to
   libmagickb200's residency registry: the operators then move pixels at PCIe speed (55 GB/s instead of the 9 / 19 GB/s of
   pageable cudaMemcpy, tools/micro/staging.cu) straight from / to the cache, and every pixel cache keeps one HBM copy for
   its lifetime.  Pinning costs ~300 ms per GiB, which is why freed blocks are recycled instead of being unpinned.  Small
   blocks and everything allocated before the installation stay with posix_memalign / free.
   Enabled by calling the function, or by MAGICK_B200_PINNED_CACHE=1 in the environment (checked when the shim is loaded). */
#include <pthread.h>

#define B200_POOL_MIN_BYTES ((size_t) 1 << 20)
#define B200_POOL_MAX_BLOCKS 256
static struct { void *ptr; size_t capacity; int in_use; } b200_pool[B200_POOL_MAX_BLOCKS];
static size_t b200_pool_idle_bytes = 0, b200_pool_idle_limit = (size_t) 8 << 30;
static pthread_mutex_t b200_pool_mutex = PTHREAD_MUTEX_INITIALIZER;
static long b200_pool_reused = 0, b200_pool_pinned = 0;

static void *b200_acquire_aligned(const size_t size, const size_t alignment)
{
  void *memory = (void *) NULL;
  if (size >= B200_POOL_MIN_BYTES && mb200_device_count() > 0) {
    int i, best = -1, slot = -1;
    pthread_mutex_lock(&b200_pool_mutex);
    for (i = 0; i < B200_POOL_MAX_BLOCKS; i++) {
      if (b200_pool[i].ptr == (void *) NULL) { if (slot < 0) slot = i; continue; }
      if (b200_pool[i].in_use == 0 && b200_pool[i].capacity >= size && b200_pool[i].capacity <= size + size / 4 &&
          (best < 0 || b200_pool[i].capacity < b200_pool[best].capacity)) best = i;
    }
    if (best >= 0) {
      b200_pool[best].in_use = 1;
      b200_pool_idle_bytes -= b200_pool[best].capacity;
      b200_pool_reused++;
      memory = b200_pool[best].ptr;
    } else if (slot >= 0) {
      const size_t capacity = (size + ((size_t) 1 << 21) - 1) & ~(((size_t) 1 << 21) - 1);
      b200_pool[slot].in_use = 1;                 /* reserve the slot while the (slow) pinning runs unlocked */
      b200_pool[slot].ptr = (void *) &b200_pool;  /* placeholder: not a block anybody can hold */
      pthread_mutex_unlock(&b200_pool_mutex);
      if (mb200_malloc_host(&memory, capacity) != MB200_OK) memory = (void *) NULL;
      pthread_mutex_lock(&b200_pool_mutex);
      if (memory != (void *) NULL) { b200_pool[slot].ptr = memory; b200_pool[slot].capacity = capacity; b200_pool_pinned++; }
      else { b200_pool[slot].ptr = (void *) NULL; b200_pool[slot].in_use = 0; }
    }
    pthread_mutex_unlock(&b200_pool_mutex);
    if (memory != (void *) NULL) {
      (void) mb200_cache_attach(memory, size, 0);
      return memory;
    }
  }
  if (posix_memalign(&memory, alignment < sizeof(void *) ? sizeof(void *) : alignment, size) != 0) return (void *) NULL;
  return memory;
}

static void b200_relinquish_aligned(void *memory)
{
  int i, ours = 0;
  void *release = (void *) NULL;
  if (memory == (void *) NULL) return;
  pthread_mutex_lock(&b200_pool_mutex);
  for (i = 0; i < B200_POOL_MAX_BLOCKS; i++)
    if (b200_pool[i].ptr == memory && b200_pool[i].in_use != 0) {
      ours = 1;
      b200_pool[i].in_use = 0;
      if (b200_pool_idle_bytes + b200_pool[i].capacity > b200_pool_idle_limit) { release = memory; b200_pool[i].ptr = (void *) NULL; }
      else b200_pool_idle_bytes += b200_pool[i].capacity;
      break;
    }
  pthread_mutex_unlock(&b200_pool_mutex);
  if (ours == 0) { free(memory); return; }
  (void) mb200_cache_detach(memory);              /* the image is gone: drop its HBM copy */
  if (release != (void *) NULL) (void) mb200_free_host(release);
}

void B200ShimInstallPixelCachePool(void)
{
  SetMagickAlignedMemoryMethods(b200_acquire_aligned, b200_relinquish_aligned);
}
void B200ShimPixelCachePoolStats(long *pinned_blocks, long *reused_blocks)
{
  if (pinned_blocks) *pinned_blocks = b200_pool_pinned;
  if (reused_blocks) *reused_blocks = b200_pool_reused;
}

/* ---- lazy synchronisation (hook mode) -----------------------------------------------------------------------------------
   The reference keeps an OpenCL result in its cl_mem until somebody looks at the pixels: CopyOpenCLBuffer() is called at
   three places of cache.c -- GetImagePixelCache (:1710, before the host writes), GetVirtualPixelCacheNexus (:2771, before the
   host reads) and PersistPixelCache (:4079).  A build that adds B200PixelCacheHook(cache_info->pixels, for_write) at the
   same three places (INTEGRATION.md has the patch; oracle/Makefile generates such a cache.c for the hooked harness) gets the
   same behaviour here: call B200ShimSetLazySync(1) once and chained operators (-blur ... -resize ...) upload once and
   download once.  Without the hooks lazy mode must stay off: nothing would bring a result back to the host. */
void B200PixelCacheHook(void *pixels, int for_write)
{
  if (pixels == (void *) NULL) return;
  (void) mb200_cache_sync(pixels);
  if (for_write != 0) (void) mb200_cache_host_written(pixels);
}
void B200ShimSetLazySync(int on) { (void) mb200_cache_set_lazy(on); }

__attribute__((constructor)) static void b200_shim_init(void)
{
  const char *e = getenv("MAGICK_B200_PINNED_CACHE");
  if (e != (const char *) NULL && *e != '\0' && *e != '0') B200ShimInstallPixelCachePool();
  e = getenv("MAGICK_B200_LAZY_SYNC");          /* only for builds that carry the cache.c hooks */
  if (e != (const char *) NULL && *e != '\0' && *e != '0') B200ShimSetLazySync(1);
}
