/*
  oracle/ref_layout.c -- TEST INFRASTRUCTURE ONLY.

  Driver of the UNMODIFIED reference's TransformImageColorspace for the colourspaces that change the channel layout
  (GRAY, LinearGRAY, CMYK) on raw, tightly packed float buffers.  It reuses export_image and the BEGIN / END bracket of
  oracle/ref_harness.c, which are file-local there, so this translation unit includes it; images tagged GRAY,
  LinearGRAY or CMYK are built by its own helper, because their channel map is the colourspace's.  Built by
  oracle/Makefile against the reference archive it compiles from source, into
  oracle/_ref/libmagickref_layout.so.
*/
#include "ref_harness.c"

/* An image of `ch` channels tagged `colorspace` (ColorspaceType): SetImageColorspace lays the cache out for the space
   (gray[, alpha]; C, M, Y, K[, alpha]), the alpha trait is added, and the storage class sync re-derives the map. */
static Image *make_layout_image(const float *src, size_t w, size_t h, int ch, int colorspace, ExceptionInfo *ex)
{
  const int base = colorspace == CMYKColorspace ? 4 :
                   (colorspace == GRAYColorspace || colorspace == LinearGRAYColorspace) ? 1 : 3;
  ImageInfo *info;
  Image *im;
  Quantum *q;
  if (base == 3) return make_image(src, w, h, ch, colorspace, ex);
  if (ch != base && ch != base + 1) return (Image *) NULL;
  ensure_init();
  info = AcquireImageInfo();
  im = AcquireImage(info, ex);
  info = DestroyImageInfo(info);
  if (im == (Image *) NULL) return im;
  if (SetImageExtent(im, w, h, ex) == MagickFalse) return DestroyImage(im);
  (void) SetImageColorspace(im, (ColorspaceType) colorspace, ex);
  if (ch == base + 1) im->alpha_trait = BlendPixelTrait;
  (void) SetImageStorageClass(im, DirectClass, ex);
  if ((int) GetPixelChannels(im) != ch) return DestroyImage(im);
  q = GetAuthenticPixels(im, 0, 0, w, h, ex);
  if (q == (Quantum *) NULL) return DestroyImage(im);
  memcpy(q, src, w * h * (size_t) ch * sizeof(float));
  (void) SyncAuthenticPixels(im, ex);
  return im;
}

/* colorspace.c:1751 TransformImageColorspace from `src` (ch channels, tagged `from`) to `to`, with "key=value;..."
   settings as ref_colorspace_defines takes them ("color:" keys as artifacts, the others as properties).  Exports the
   re-laid-out cache into `dst` and returns its channel count; *type receives image->type.  Negative on failure. */
__attribute__((visibility("default")))
int ref_colorspace_layout(const float *src, float *dst, size_t w, size_t h, int ch, int from, int to, const char *defines,
                          int *type)
{
  BEGIN
  im = make_layout_image(src, w, h, ch, from, ex);
  if (im) {
    char *copy = AcquireString(defines != (const char *) NULL ? defines : ""), *p = copy;
    while (p != (char *) NULL && *p != '\0') {
      char *end = strchr(p, ';'), *eq;
      if (end != (char *) NULL) *end = '\0';
      eq = strchr(p, '=');
      if (eq != (char *) NULL) {
        *eq = '\0';
        if (strncmp(p, "color:", 6) == 0) (void) SetImageArtifact(im, p, eq + 1);
        else (void) SetImageProperty(im, p, eq + 1, ex);
      }
      p = end != (char *) NULL ? end + 1 : (char *) NULL;
    }
    copy = DestroyString(copy);
    if (TransformImageColorspace(im, (ColorspaceType) to, ex) != MagickFalse && (int) im->colorspace == to) {
      const int out_ch = (int) GetPixelChannels(im);
      rc = export_image(im, dst, w, h, out_ch, ex);
      if (rc == 0) {
        rc = out_ch;
        if (type != (int *) NULL) *type = (int) im->type;
      }
    }
  }
  END
}
