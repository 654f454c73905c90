/*
  oracle/ref_direct.c -- TEST INFRASTRUCTURE ONLY.

  Driver of the UNMODIFIED reference's MorphologyImage with the directly applied methods, Distance (21) and Voronoi (22),
  on raw, tightly packed float buffers.  It uses the image helpers of oracle/ref_harness.c (make_image, export_image, the
  BEGIN / END bracket), which are file-local there, so this translation unit includes it.  Built by oracle/direct.mk
  against the reference archive that oracle/Makefile compiles from source, into oracle/_ref/libmagickref_direct.so.
*/
#include "ref_harness.c"

/* MorphologyImage(src, method, iterations, AcquireKernelInfo(kernel)).  The result is exported into `dst` (room for
   w*h*(ch+1) floats: Voronoi adds an alpha channel to an image without one); returns its channel count and stores its
   alpha_trait in *alpha_trait.  Negative on failure. */
__attribute__((visibility("default")))
int ref_morphology_direct(const float *src, float *dst, size_t w, size_t h, int ch, int method, long iterations,
                          const char *kernel, int *alpha_trait)
{
  BEGIN
  KernelInfo *k;
  im = make_image(src, w, h, ch, -1, ex);
  k = AcquireKernelInfo(kernel, ex);
  if (im && k) {
    out = MorphologyImage(im, (MorphologyMethod) method, (ssize_t) iterations, k, ex);
    if (out) {
      const int out_ch = (int) GetPixelChannels(out);
      rc = export_image(out, dst, w, h, out_ch, ex);
      if (rc == 0) rc = out_ch;
      if (alpha_trait != NULL) *alpha_trait = (int) out->alpha_trait;
    }
  }
  if (k) k = DestroyKernelInfo(k);
  END
}
