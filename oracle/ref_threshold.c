/*
  oracle/ref_threshold.c -- TEST INFRASTRUCTURE ONLY.

  Drivers of the UNMODIFIED reference's AdaptiveThresholdImage, AutoThresholdImage, RangeThresholdImage and
  PerceptibleImage on raw, tightly packed float buffers, each under SetPixelChannelMask(channel_mask) (a ChannelType; -1
  leaves the default mask).  They use the image helpers of oracle/ref_harness.c (make_image, export_image, the BEGIN /
  END bracket), which are file-local there, so this translation unit includes it.  Built by oracle/threshold.mk against
  the reference archive that oracle/Makefile compiles from source, into oracle/_ref/libmagickref_threshold.so.
*/
#include "ref_harness.c"

enum { REF_ADAPTIVE, REF_AUTO, REF_RANGE, REF_PERCEPTIBLE };

/* Runs operator `op` with arguments a[0..3] on the image in `buf` (w x h x ch); AdaptiveThreshold takes a[0] x a[1]
   windows and bias a[2], AutoThreshold method (int) a[0], RangeThreshold the four limits, Perceptible epsilon a[0].
   The result's cache (whose channel count may differ: RangeThreshold's sRGB transform of a gray image) is exported into
   `buf` (which must hold w x h x 4 floats) and its channel count returned; `property` (>= 64 bytes) receives the
   "auto-threshold:threshold" property.  Negative on failure. */
__attribute__((visibility("default")))
int ref_threshold_op(float *buf, size_t w, size_t h, int ch, int op, const double *a, long channel_mask, char *property)
{
  BEGIN
  im = make_image(buf, w, h, ch, -1, ex);
  if (im) {
    MagickBooleanType ok = MagickFalse;
    Image *result = im;
    if (channel_mask >= 0) (void) SetPixelChannelMask(im, (ChannelType) channel_mask);
    switch (op) {
      case REF_ADAPTIVE:
        out = AdaptiveThresholdImage(im, (size_t) a[0], (size_t) a[1], a[2], ex);
        ok = out != NULL ? MagickTrue : MagickFalse;
        result = out;
        break;
      case REF_AUTO: ok = AutoThresholdImage(im, (AutoThresholdMethod) (int) a[0], ex); break;
      case REF_RANGE: ok = RangeThresholdImage(im, a[0], a[1], a[2], a[3], ex); break;
      case REF_PERCEPTIBLE: ok = PerceptibleImage(im, a[0], ex); break;
      default: break;
    }
    if (ok != MagickFalse) {
      const int out_ch = (int) GetPixelChannels(result);
      rc = export_image(result, buf, w, h, out_ch, ex);
      if (rc == 0) rc = out_ch;
      if (property != NULL) {
        const char *value = GetImageProperty(result, "auto-threshold:threshold", ex);
        (void) CopyMagickString(property, value != NULL ? value : "", 64);
      }
    }
  }
  END
}
