/*
  oracle/ref_geometry.c -- TEST INFRASTRUCTURE ONLY.

  Driver of the UNMODIFIED reference's orientation and crop operators (CropImage, ShaveImage, FlipImage, FlopImage,
  TransposeImage, TransverseImage, IntegralRotateImage, RollImage, AutoOrientImage) on raw, tightly packed float
  buffers.  It uses the image helpers of oracle/ref_harness.c (make_image, export_image, the BEGIN / END bracket), which
  are file-local there, so this translation unit includes it.  Built by oracle/Makefile against the reference archive
  it compiles from source, into oracle/_ref/libmagickref_geometry.so.
*/
#include "ref_harness.c"

/* CMYK (4 channels) or CMYKA (5): the colourspace's own channel map, then the samples. */
static Image *make_cmyk_image(const float *src, size_t w, size_t h, int ch, ExceptionInfo *ex)
{
  ImageInfo *info;
  Image *im;
  Quantum *q;
  ensure_init();
  info = AcquireImageInfo();
  im = AcquireImage(info, ex);
  info = DestroyImageInfo(info);
  if (im == (Image *) NULL) return im;
  if (SetImageExtent(im, w, h, ex) == MagickFalse) return DestroyImage(im);
  (void) SetImageColorspace(im, CMYKColorspace, ex);
  if (ch == 5) im->alpha_trait = BlendPixelTrait;
  (void) SetImageStorageClass(im, DirectClass, ex);
  (void) SetImageColorspace(im, CMYKColorspace, ex);
  if ((int) GetPixelChannels(im) != ch) return DestroyImage(im);
  q = GetAuthenticPixels(im, 0, 0, w, h, ex);
  if (q == (Quantum *) NULL) return DestroyImage(im);
  memcpy(q, src, w * h * (size_t) ch * sizeof(float));
  (void) SyncAuthenticPixels(im, ex);
  return im;
}

/* op (mb200_geometry_op): 0 CropImage(args: width, height, x, y), 1 ShaveImage(width, height), 2 FlipImage,
   3 FlopImage, 4 TransposeImage, 5 TransverseImage, 6 IntegralRotateImage(rotations), 7 RollImage(x, y); 8
   AutoOrientImage(orientation).  The source is CMYK(A) when `cmyk` is set (4 or 5 channels) and takes the page
   page[0..3] = width, height, x, y.  The result (room for cap floats) is exported into dst; geometry[0..5] receives its
   columns, rows, page.width, page.height, page.x and page.y, geometry[6] its orientation.  Returns its channel count,
   or a negative number when the reference returned no image or the result does not fit. */
__attribute__((visibility("default")))
int ref_geometry(const float *src, size_t w, size_t h, int ch, int cmyk, const long *page, int op, const long *args,
                 float *dst, size_t cap, long *geometry)
{
  BEGIN
  im = cmyk ? make_cmyk_image(src, w, h, ch, ex) : make_image(src, w, h, ch, -1, ex);
  if (im) {
    RectangleInfo r;
    im->page.width = (size_t) page[0];
    im->page.height = (size_t) page[1];
    im->page.x = page[2];
    im->page.y = page[3];
    switch (op) {
      case 0:
        r.width = (size_t) args[0]; r.height = (size_t) args[1]; r.x = args[2]; r.y = args[3];
        out = CropImage(im, &r, ex);
        break;
      case 1:
        r.width = (size_t) args[0]; r.height = (size_t) args[1]; r.x = 0; r.y = 0;
        out = ShaveImage(im, &r, ex);
        break;
      case 2: out = FlipImage(im, ex); break;
      case 3: out = FlopImage(im, ex); break;
      case 4: out = TransposeImage(im, ex); break;
      case 5: out = TransverseImage(im, ex); break;
      case 6: out = IntegralRotateImage(im, (size_t) args[0], ex); break;
      case 7: out = RollImage(im, (ssize_t) args[0], (ssize_t) args[1], ex); break;
      case 8: out = AutoOrientImage(im, (OrientationType) args[0], ex); break;
      default: break;
    }
    if (out) {
      const int out_ch = (int) GetPixelChannels(out);
      geometry[0] = (long) out->columns;
      geometry[1] = (long) out->rows;
      geometry[2] = (long) out->page.width;
      geometry[3] = (long) out->page.height;
      geometry[4] = (long) out->page.x;
      geometry[5] = (long) out->page.y;
      geometry[6] = (long) out->orientation;
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
