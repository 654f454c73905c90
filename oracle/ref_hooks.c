/*
  oracle/ref_hooks.c -- TEST INFRASTRUCTURE ONLY.

  Drivers of the UNMODIFIED reference's DespeckleImage, LocalContrastImage and WaveletDenoiseImage on raw, tightly
  packed float buffers (Quantum == float, channels interleaved; 1 Gray, 2 Gray+Alpha, 3 RGB, 4 RGBA), like
  oracle/ref_harness.c does for the other operators.  Built by oracle/Makefile against the reference archive it
  compiles from source, into oracle/_ref/libmagickref_hooks.so.
*/
#include "MagickCore/studio.h"
#include "MagickCore/MagickCore.h"
#include <string.h>

static int g_init = 0;

static Image *make_image(const float *src, size_t w, size_t h, int ch, ExceptionInfo *ex)
{
  ImageInfo *info;
  Image *im;
  Quantum *q;

  if (!g_init) { MagickCoreGenesis("magickref_hooks", MagickFalse); g_init = 1; }
  info = AcquireImageInfo();
  im = AcquireImage(info, ex);
  info = DestroyImageInfo(info);
  if (im == (Image *) NULL) return im;
  if (SetImageExtent(im, w, h, ex) == MagickFalse) return DestroyImage(im);
  if (ch == 1 || ch == 2)
    (void) SetImageColorspace(im, GRAYColorspace, ex);
  if (ch == 2 || ch == 4)
    im->alpha_trait = BlendPixelTrait;
  (void) SetImageStorageClass(im, DirectClass, ex);
  /* re-derive the channel map after the alpha_trait change (pixel.c:6132) */
  (void) SetImageColorspace(im, im->colorspace, ex);
  if ((int) GetPixelChannels(im) != ch) return DestroyImage(im);
  q = GetAuthenticPixels(im, 0, 0, w, h, ex);
  if (q == (Quantum *) NULL) return DestroyImage(im);
  memcpy(q, src, w * h * (size_t) ch * sizeof(float));
  (void) SyncAuthenticPixels(im, ex);
  return im;
}

static int export_image(const Image *im, float *dst, size_t w, size_t h, int ch, ExceptionInfo *ex)
{
  const Quantum *p;
  if (im == (const Image *) NULL) return -1;
  if (im->columns != w || im->rows != h || (int) GetPixelChannels(im) != ch) return -2;
  p = GetVirtualPixels(im, 0, 0, w, h, ex);
  if (p == (const Quantum *) NULL) return -3;
  memcpy(dst, p, w * h * (size_t) ch * sizeof(float));
  return 0;
}

#define BEGIN ExceptionInfo *ex = AcquireExceptionInfo(); Image *im = NULL, *out = NULL; int rc = -1;
#define END   if (out) out = DestroyImage(out); if (im) im = DestroyImage(im); ex = DestroyExceptionInfo(ex); return rc;

__attribute__((visibility("default")))
int ref_despeckle(const float *src, float *dst, size_t w, size_t h, int ch)
{
  BEGIN
  im = make_image(src, w, h, ch, ex);
  if (im) { out = DespeckleImage(im, ex); rc = export_image(out, dst, w, h, ch, ex); }
  END
}

__attribute__((visibility("default")))
int ref_local_contrast(const float *src, float *dst, size_t w, size_t h, int ch, double radius, double strength)
{
  BEGIN
  im = make_image(src, w, h, ch, ex);
  if (im) { out = LocalContrastImage(im, radius, strength, ex); rc = export_image(out, dst, w, h, ch, ex); }
  END
}

/* channels: a ChannelType selection set with SetPixelChannelMask before the call (0: none, the default mask) */
__attribute__((visibility("default")))
int ref_wavelet_denoise(const float *src, float *dst, size_t w, size_t h, int ch, double threshold, double softness,
                        int channels)
{
  BEGIN
  im = make_image(src, w, h, ch, ex);
  if (im) {
    if (channels != 0) (void) SetPixelChannelMask(im, (ChannelType) channels);
    out = WaveletDenoiseImage(im, threshold, softness, ex);
    rc = export_image(out, dst, w, h, ch, ex);
  }
  END
}
