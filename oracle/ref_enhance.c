/*
  oracle/ref_enhance.c -- TEST INFRASTRUCTURE ONLY.

  Drivers of the UNMODIFIED reference's ContrastImage, ModulateImage, GrayscaleImage and FunctionImage on raw, tightly
  packed float buffers, in place.  They use the image helpers of oracle/ref_harness.c (make_image, export_image, the
  BEGIN / END bracket), which are file-local there, so this translation unit includes it.  Built by oracle/enhance.mk
  against the reference archive that oracle/Makefile compiles from source, into oracle/_ref/libmagickref_enhance.so.
*/
#include "ref_harness.c"

/* enhance.c:1370 ContrastImage, in place; `from` tags the image (ColorspaceType, -1: the default) */
__attribute__((visibility("default")))
int ref_contrast(float *buf, size_t w, size_t h, int ch, int from, int sharpen)
{
  BEGIN
  im = make_image(buf, w, h, ch, from, ex);
  if (im && ContrastImage(im, sharpen ? MagickTrue : MagickFalse, ex) != MagickFalse)
    rc = export_image(im, buf, w, h, ch, ex);
  END
}

/* enhance.c:3461 ModulateImage(modulate), in place, with "key=value;key=value" image artifacts ("modulate:colorspace",
   "color:illuminant") */
__attribute__((visibility("default")))
int ref_modulate(float *buf, size_t w, size_t h, int ch, int from, const char *modulate, const char *artifacts)
{
  BEGIN
  im = make_image(buf, w, h, ch, from, ex);
  if (im) {
    char *copy = AcquireString(artifacts != (const char *) NULL ? artifacts : ""), *p = copy;
    while (p != (char *) NULL && *p != '\0') {
      char *end = strchr(p, ';'), *eq;
      if (end != (char *) NULL) *end = '\0';
      eq = strchr(p, '=');
      if (eq != (char *) NULL) {
        *eq = '\0';
        (void) SetImageArtifact(im, p, eq + 1);
      }
      p = end != (char *) NULL ? end + 1 : (char *) NULL;
    }
    copy = DestroyString(copy);
    if (ModulateImage(im, modulate, ex) != MagickFalse)
      rc = export_image(im, buf, w, h, ch, ex);
  }
  END
}

/* enhance.c:2474 GrayscaleImage(method), in place: exports the re-laid-out GRAY / LinearGRAY cache and returns its
   channel count (1, or 2 with alpha); negative on failure */
__attribute__((visibility("default")))
int ref_grayscale(float *buf, size_t w, size_t h, int ch, int from, int method)
{
  BEGIN
  im = make_image(buf, w, h, ch, from, ex);
  if (im && GrayscaleImage(im, (PixelIntensityMethod) method, ex) != MagickFalse) {
    const int out_ch = (int) GetPixelChannels(im);
    rc = export_image(im, buf, w, h, out_ch, ex);
    if (rc == 0) rc = out_ch;
  }
  END
}

/* statistic.c:1064 FunctionImage, in place, under SetPixelChannelMask(channel_mask) (a ChannelType; -1: untouched) */
__attribute__((visibility("default")))
int ref_function(float *buf, size_t w, size_t h, int ch, int function, size_t n, const double *params, long channel_mask)
{
  BEGIN
  im = make_image(buf, w, h, ch, -1, ex);
  if (im) {
    if (channel_mask >= 0) (void) SetPixelChannelMask(im, (ChannelType) channel_mask);
    if (FunctionImage(im, (MagickFunction) function, n, params, ex) != MagickFalse)
      rc = export_image(im, buf, w, h, ch, ex);
  }
  END
}
