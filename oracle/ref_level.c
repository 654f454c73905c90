/*
  oracle/ref_level.c -- TEST INFRASTRUCTURE ONLY.

  Drivers of the UNMODIFIED reference's LevelImage, LevelizeImage, MinMaxStretchImage, AutoLevelImage,
  ContrastStretchImage, NormalizeImage, LinearStretchImage and GammaImage on raw, tightly packed float buffers, in place,
  each under SetPixelChannelMask(channel_mask) (a ChannelType; -1 leaves the default mask).  They use the image helpers of
  oracle/ref_harness.c (make_image, export_image, the BEGIN / END bracket), which are file-local there, so this
  translation unit includes it.  Built by oracle/Makefile against the reference archive it compiles
  from source, into oracle/_ref/libmagickref_level.so.
*/
#include "ref_harness.c"

enum { REF_LEVEL, REF_LEVELIZE, REF_MINMAX, REF_AUTO_LEVEL, REF_CONTRAST_STRETCH, REF_NORMALIZE, REF_LINEAR_STRETCH,
       REF_GAMMA };

/* Runs operator `op` with arguments a, b, g on the image; exports the resulting cache (whose channel count may differ:
   ContrastStretch's gray re-layout) into `buf` and returns its channel count.  `property` (>= 64 bytes, may be NULL)
   receives the operator's "histogram:*" property, `image_gamma` (may be NULL) image->gamma afterwards.  Negative on
   failure. */
__attribute__((visibility("default")))
int ref_level_op(float *buf, size_t w, size_t h, int ch, int op, double a, double b, double g, long channel_mask,
                 char *property, double *image_gamma)
{
  BEGIN
  im = make_image(buf, w, h, ch, -1, ex);
  if (im) {
    MagickBooleanType ok = MagickFalse;
    const char *name = NULL;
    if (channel_mask >= 0) (void) SetPixelChannelMask(im, (ChannelType) channel_mask);
    switch (op) {
      case REF_LEVEL: ok = LevelImage(im, a, b, g, ex); break;
      case REF_LEVELIZE: ok = LevelizeImage(im, a, b, g, ex); break;
      case REF_MINMAX: ok = MinMaxStretchImage(im, a, b, g, ex); break;
      case REF_AUTO_LEVEL: ok = AutoLevelImage(im, ex); break;
      case REF_CONTRAST_STRETCH: ok = ContrastStretchImage(im, a, b, ex); name = "histogram:contrast-stretch"; break;
      case REF_NORMALIZE: ok = NormalizeImage(im, ex); name = "histogram:contrast-stretch"; break;
      case REF_LINEAR_STRETCH: ok = LinearStretchImage(im, a, b, ex); name = "histogram:linear-stretch"; break;
      case REF_GAMMA: ok = GammaImage(im, g, ex); break;
      default: break;
    }
    if (ok != MagickFalse) {
      const int out_ch = (int) GetPixelChannels(im);
      rc = export_image(im, buf, w, h, out_ch, ex);
      if (rc == 0) rc = out_ch;
      if (property != NULL) {
        const char *value = name != NULL ? GetImageProperty(im, name, ex) : NULL;
        (void) CopyMagickString(property, value != NULL ? value : "", 64);
      }
      if (image_gamma != NULL) *image_gamma = im->gamma;
    }
  }
  END
}
