/*
  oracle/ref_trim.c -- TEST INFRASTRUCTURE ONLY.

  Driver of the UNMODIFIED reference's GetImageBoundingBox (attribute.c:391) and TrimImage (transform.c:2412) on raw,
  tightly packed float buffers.  It uses the image helpers of oracle/ref_geometry.c (make_cmyk_image) and
  oracle/ref_harness.c (make_image, export_image, the BEGIN / END bracket), which are file-local there, so this
  translation unit includes the former.  Built by oracle/Makefile into oracle/_ref/libmagickref_trim.so.
*/
#include "ref_geometry.c"

/* op 0: GetImageBoundingBox, op 1: TrimImage, on an image of `ch` channels (CMYK(A) when `cmyk` is set, otherwise
   tagged with `colorspace` when it is >= 0 and the image has 3 or more channels) with page[0..3] = width, height, x, y,
   image->fuzz = fuzz, image->gravity = gravity and the artifacts "trim:edges" = edges and "trim:minSize" = min_size
   (NULL: not set).  box[0..3] receives the bounding box (width, height, x, y; TrimImage computes its own, op 0 only) and
   *severity the exception's severity afterwards.  For TrimImage the result (room for cap floats) is exported into dst
   and geometry[0..5] receives its columns, rows, page.width, page.height, page.x and page.y; the return value is its
   channel count.  Op 0 returns 0.  A negative number: no image, or a result that does not fit.

   The reference runs with `threads` threads; the recorded results use one.  Its row loop (attribute.c:484-535) gives
   each row a copy of the shared bounds taken when the row starts, and the target[3] rule at :529-535 reads that copy's
   width; with several threads the rows start in schedule order, so when the bottom corners differ the box of an image
   of 512 rows or more depends on the OpenMP schedule.  The single-threaded order is the one result the library
   reproduces.  tools/devbench.py times the reference with every core. */
__attribute__((visibility("default")))
int ref_trim(const float *src, size_t w, size_t h, int ch, int cmyk, int colorspace, const long *page, double fuzz,
             const char *edges, const char *min_size, int gravity, int op, long *box, int *severity, float *dst,
             size_t cap, long *geometry, int threads)
{
  BEGIN
  ref_set_threads(threads);
  im = cmyk ? make_cmyk_image(src, w, h, ch, ex) : make_image(src, w, h, ch, colorspace, ex);
  if (im) {
    im->page.width = (size_t) page[0];
    im->page.height = (size_t) page[1];
    im->page.x = page[2];
    im->page.y = page[3];
    im->fuzz = fuzz;
    im->gravity = (GravityType) gravity;
    (void) strcpy(im->filename, "trim-case");
    if (edges) (void) SetImageArtifact(im, "trim:edges", edges);
    if (min_size) (void) SetImageArtifact(im, "trim:minSize", min_size);
    if (op == 0) {
      const RectangleInfo r = GetImageBoundingBox(im, ex);
      box[0] = (long) r.width;
      box[1] = (long) r.height;
      box[2] = (long) r.x;
      box[3] = (long) r.y;
      rc = 0;
    } else {
      out = TrimImage(im, ex);
      if (out) {
        const int out_ch = (int) GetPixelChannels(out);
        geometry[0] = (long) out->columns;
        geometry[1] = (long) out->rows;
        geometry[2] = (long) out->page.width;
        geometry[3] = (long) out->page.height;
        geometry[4] = (long) out->page.x;
        geometry[5] = (long) out->page.y;
        if (out->columns * out->rows * (size_t) out_ch > cap)
          rc = -4;
        else {
          rc = export_image(out, dst, out->columns, out->rows, out_ch, ex);
          if (rc == 0) rc = out_ch;
        }
      }
    }
    *severity = (int) ex->severity;
  }
  END
}
