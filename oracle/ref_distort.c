/*
  oracle/ref_distort.c -- TEST INFRASTRUCTURE ONLY.

  Driver of the UNMODIFIED reference's DistortImage and RotateImage on raw, tightly packed float buffers.  It uses the
  image helpers of oracle/ref_harness.c (make_image, the BEGIN / END bracket), which are file-local there, so this
  translation unit includes it.  Built by oracle/Makefile against the reference archive it compiles
  from source, into oracle/_ref/libmagickref_distort.so.
*/
#include "ref_harness.c"

static void set_color(PixelInfo *p, const double *rgba, int alpha_trait)
{
  p->red = rgba[0];
  p->green = rgba[1];
  p->blue = rgba[2];
  p->alpha = rgba[3];
  p->alpha_trait = alpha_trait ? BlendPixelTrait : UndefinedPixelTrait;
}

/* Sets every "key=value" line of `artifacts` (may be NULL) on the image. */
static void set_artifacts(Image *im, const char *artifacts)
{
  char buf[4096], *line, *save = NULL;
  if (artifacts == NULL) return;
  (void) strncpy(buf, artifacts, sizeof(buf) - 1);
  buf[sizeof(buf) - 1] = '\0';
  for (line = strtok_r(buf, "\n", &save); line != NULL; line = strtok_r(NULL, "\n", &save)) {
    char *eq = strchr(line, '=');
    if (eq == NULL) continue;
    *eq = '\0';
    (void) SetImageArtifact(im, line, eq + 1);
  }
}

/* method > 0: DistortImage(src, method, nargs, args, bestfit); method == 0: RotateImage(src, args[0]).  The source
   takes page (page_x, page_y), the filter, interpolate and virtual-pixel method, and background / matte colours
   (rgba, with an alpha trait when *_alpha is set); `artifacts` is "key=value" lines.  The result (room for cap floats)
   is exported into dst; geometry[0..3] receives its columns, rows, page.x and page.y.  Returns its channel count, or a
   negative number when the reference returned no image or the result does not fit. */
__attribute__((visibility("default")))
int ref_distort(const float *src, size_t w, size_t h, int ch, long page_x, long page_y, int method, const double *args,
                size_t nargs, int bestfit, int filter, int interpolate, int vp, const double *background, int bg_alpha,
                const double *matte, int matte_alpha, const char *artifacts, float *dst, size_t cap, long *geometry)
{
  BEGIN
  im = make_image(src, w, h, ch, -1, ex);
  if (im) {
    im->page.x = page_x;
    im->page.y = page_y;
    im->filter = (FilterType) filter;
    im->interpolate = (PixelInterpolateMethod) interpolate;
    set_color(&im->background_color, background, bg_alpha);
    set_color(&im->matte_color, matte, matte_alpha);
    set_artifacts(im, artifacts);
    if (method == 0)
      out = RotateImage(im, args[0], ex);
    else {
      (void) SetImageVirtualPixelMethod(im, (VirtualPixelMethod) vp, ex);
      out = DistortImage(im, (DistortMethod) method, nargs, args, bestfit ? MagickTrue : MagickFalse, ex);
    }
    if (out) {
      const int out_ch = (int) GetPixelChannels(out);
      geometry[0] = (long) out->columns;
      geometry[1] = (long) out->rows;
      geometry[2] = (long) out->page.x;
      geometry[3] = (long) out->page.y;
      if (out->columns * out->rows * (size_t) out_ch > cap)
        rc = -4;
      else {
        rc = export_image(out, dst, out->columns, out->rows, out_ch, ex);
        if (rc == 0) rc = out_ch;
      }
    }
  }
  END
}
