/*
  oracle/enhance_oracle.c -- TEST INFRASTRUCTURE ONLY.  Never linked into, imported by or executed from the product.

  The plain-C oracle of the in-place enhance operators of ImageMagick 7.1.1-45 Q16-HDRI whose accelerate hooks have call
  sites (accelerate-private.h:50-60): ContrastImage, ModulateImage, GrayscaleImage and FunctionImage, restated in the
  reference's operation order.  They are built on the colour restatements of the main oracle -- rgb_to_hsb / hsb_to_rgb
  and the other hue legs, rgb_to_xyz / xyz_to_lab / xyz_to_luv and their inverses, the illuminant table,
  decode_pixel_gamma / encode_pixel_gamma -- which are file-local there, so this translation unit includes oracle.c
  itself rather than carrying a second copy of them.  Built by oracle/Makefile into oracle/libenhance_oracle.so with
  the main oracle's flags (no contraction, standard excess precision); pinned bit for bit against the reference compiled
  from source by tests/test_oracle_enhance_vs_ref.py.  Buffers as in oracle.h.

    int orc_contrast(float *buf, size_t w, size_t h, int ch, int sharpen);
    int orc_modulate(float *buf, size_t w, size_t h, int ch, double percent_brightness, double percent_saturation,
                     double percent_hue, int colorspace, int illuminant);
        `colorspace` the "modulate:colorspace" value (anything but HCL / HCLp / HSB / HSI / HSL / HSV / HWB / LCH / LCHab /
        LCHuv is HSL), `illuminant` an IlluminantType
    int orc_grayscale(float *buf, size_t w, size_t h, int ch, int method, int colorspace);
        returns the channel count of the re-laid-out GRAY cache (1, or 2 with alpha)
    int orc_function(float *buf, size_t w, size_t h, int ch, int function, size_t n_params, const double *params,
                     unsigned update_mask);
        on the channels of update_mask (bit c = channel c)
*/
#include "oracle.c"

/* ------------------------------------------------------------------------------------------
   In-place enhance operators (the reference's in-place accelerate hooks).  Gray images (1 or 2 channels) give the
   red, green and blue accessors the gray sample; SetPixelRed / Green / Blue then write the same slot, blue last.
   ClampToQuantum (HDRI) is a float cast.
   ------------------------------------------------------------------------------------------ */
static void get_rgb(const float *q, int ch, double *red, double *green, double *blue)
{
  *red = (double) q[0];
  *green = ch >= 3 ? (double) q[1] : (double) q[0];
  *blue = ch >= 3 ? (double) q[2] : (double) q[0];
}

static void set_rgb(float *q, int ch, double red, double green, double blue)
{
  if (ch >= 3) { q[0] = (float) red; q[1] = (float) green; q[2] = (float) blue; }
  else q[0] = (float) blue;
}

/* enhance.c:1370-1505 ContrastImage */
int orc_contrast(float *buf, size_t w, size_t h, int ch, int sharpen)
{
  const int sign = sharpen != 0 ? 1 : -1;
  long i, n = (long) (w * h);
  if (ch < 1 || ch > 4) return -1;
#pragma omp parallel for schedule(static)
  for (i = 0; i < n; i++) {
    float *q = buf + (size_t) i * ch;
    double red, green, blue, hue, saturation, brightness;
    get_rgb(q, ch, &red, &green, &blue);
    rgb_to_hsb(red, green, blue, &hue, &saturation, &brightness);
    brightness += 0.5 * sign * (0.5 * (sin((double) (PI_ * (brightness - 0.5))) + 1.0) - brightness);
    if (brightness > 1.0) brightness = 1.0;
    else if (brightness < 0.0) brightness = 0.0;
    hsb_to_rgb(hue, saturation, brightness, &red, &green, &blue);
    set_rgb(q, ch, red, green, blue);
  }
  return 0;
}

/* enhance.c:3594-3630 ModulateLCHab / ModulateLCHuv (reference white in cs_ill) */
static void modulate_lch(int uv, double percent_luma, double percent_chroma, double percent_hue, double *red,
                         double *green, double *blue)
{
  double X, Y, Z, luma, chroma, hue, C, H;
  rgb_to_xyz(*red, *green, *blue, &X, &Y, &Z);
  if (uv) {                                                           /* colorspace-private.h:1163-1176 */
    double u, v;
    xyz_to_luv(X, Y, Z, &luma, &u, &v);
    chroma = hypot(354.0 * u - 134.0, 262.0 * v - 140.0) / 255.0 + 0.5;
    hue = 180.0 * atan2(262.0 * v - 140.0, 354.0 * u - 134.0) / PI_ / 360.0;
  } else {                                                            /* :1104-1117 */
    double a, b;
    xyz_to_lab(X, Y, Z, &luma, &a, &b);
    chroma = hypot(a - 0.5, b - 0.5) / 1.0 + 0.5;
    hue = 180.0 * atan2(b - 0.5, a - 0.5) / PI_ / 360.0;
  }
  if (hue < 0.0) hue += 1.0;
  luma *= 0.01 * percent_luma;
  chroma *= 0.01 * percent_chroma;
  hue += fmod((percent_hue - 100.0), 200.0) / 200.0;
  C = 255.0 * (chroma - 0.5);                                         /* :580-653 */
  H = 360.0 * hue;
  if (uv) luv_to_xyz(100.0 * luma, C * cos(degrees_to_radians(H)), C * sin(degrees_to_radians(H)), &X, &Y, &Z);
  else lab_to_xyz(100.0 * luma, C * cos(degrees_to_radians(H)), C * sin(degrees_to_radians(H)), &X, &Y, &Z);
  xyz_to_rgb(X, Y, Z, red, green, blue);
}

/* enhance.c:3461-3910 ModulateImage with the geometry parsed (percentages), `colorspace` the "modulate:colorspace"
   artifact's value (anything but the nine spaces below is HSL) and `illuminant` an IlluminantType (color.h:40-54) */
int orc_modulate(float *buf, size_t w, size_t h, int ch, double percent_brightness, double percent_saturation,
                 double percent_hue, int colorspace, int illuminant)
{
  long i, n = (long) (w * h);
  if (ch < 1 || ch > 4 || illuminant < 0 || illuminant > 10) return -1;
  cs_ill[0] = illuminant_table[illuminant][0]; cs_ill[1] = illuminant_table[illuminant][1];
  cs_ill[2] = illuminant_table[illuminant][2];
#pragma omp parallel for schedule(static)
  for (i = 0; i < n; i++) {
    float *q = buf + (size_t) i * ch;
    double red, green, blue, x, y, z;
    get_rgb(q, ch, &red, &green, &blue);
    switch (colorspace) {                     /* :3461-3592: hue += shift, the other two scaled by 0.01 * percent */
      case ORC_CS_HCL: case ORC_CS_HCLP:
        rgb_to_hcl(red, green, blue, &x, &y, &z);
        x += fmod((percent_hue - 100.0), 200.0) / 200.0; y *= 0.01 * percent_saturation; z *= 0.01 * percent_brightness;
        hcl_to_rgb(x, y, z, colorspace == ORC_CS_HCLP, &red, &green, &blue);
        break;
      case ORC_CS_HSB:
        rgb_to_hsb(red, green, blue, &x, &y, &z);
        x += fmod((percent_hue - 100.0), 200.0) / 200.0; y *= 0.01 * percent_saturation; z *= 0.01 * percent_brightness;
        hsb_to_rgb(x, y, z, &red, &green, &blue);
        break;
      case ORC_CS_HSI:
        rgb_to_hsi(red, green, blue, &x, &y, &z);
        x += fmod((percent_hue - 100.0), 200.0) / 200.0; y *= 0.01 * percent_saturation; z *= 0.01 * percent_brightness;
        hsi_to_rgb(x, y, z, &red, &green, &blue);
        break;
      case ORC_CS_HSV:
        rgb_to_hsl_hsv(red, green, blue, 1, &x, &y, &z);
        x += fmod((percent_hue - 100.0), 200.0) / 200.0; y *= 0.01 * percent_saturation; z *= 0.01 * percent_brightness;
        hsl_hsv_to_rgb(x, y, z, 1, &red, &green, &blue);
        break;
      case ORC_CS_HWB:                        /* (hue, whiteness, blackness) */
        rgb_to_hwb(red, green, blue, &x, &y, &z);
        x += fmod((percent_hue - 100.0), 200.0) / 200.0; z *= 0.01 * percent_brightness; y *= 0.01 * percent_saturation;
        hwb_to_rgb(x, y, z, &red, &green, &blue);
        break;
      case ORC_CS_LCH: case ORC_CS_LCHAB:
        modulate_lch(0, percent_brightness, percent_saturation, percent_hue, &red, &green, &blue);
        break;
      case ORC_CS_LCHUV:
        modulate_lch(1, percent_brightness, percent_saturation, percent_hue, &red, &green, &blue);
        break;
      default:
        rgb_to_hsl_hsv(red, green, blue, 0, &x, &y, &z);
        x += fmod((percent_hue - 100.0), 200.0) / 200.0; y *= 0.01 * percent_saturation; z *= 0.01 * percent_brightness;
        hsl_hsv_to_rgb(x, y, z, 0, &red, &green, &blue);
        break;
    }
    set_rgb(q, ch, red, green, blue);
  }
  cs_ill[0] = illuminant_table[5][0]; cs_ill[1] = illuminant_table[5][1]; cs_ill[2] = illuminant_table[5][2];
  return 0;
}

/* enhance.c:2474-2650 GrayscaleImage (pixel.h:110-120 PixelIntensityMethod) on an image tagged `colorspace`, followed by
   SetImageColorspace(GRAY or LinearGRAY): the cache keeps the gray channel (and alpha), compacted in place.  Returns the
   channel count of the result. */
int orc_grayscale(float *buf, size_t w, size_t h, int ch, int method, int colorspace)
{
  const int out_ch = (ch == 2 || ch == 4) ? 2 : 1;
  size_t i, n = w * h;
  if (ch < 1 || ch > 4 || method < 0 || method > 9) return -1;
#pragma omp parallel for schedule(static)
  for (i = 0; i < n; i++) {
    float *q = buf + i * ch;
    double red, green, blue, intensity = 0.0;
    get_rgb(q, ch, &red, &green, &blue);
    switch (method) {
      case 1: intensity = (red + green + blue) / 3.0; break;
      case 2: intensity = ORC_MAX(ORC_MAX(red, green), blue); break;
      case 3: intensity = (ORC_MIN(ORC_MIN(red, green), blue) + ORC_MAX(ORC_MAX(red, green), blue)) / 2.0; break;
      case 4: intensity = (double) (((double) red * red + green * green + blue * blue) / 3.0); break;
      case 5:
        if (colorspace == ORC_CS_RGB) {
          red = encode_pixel_gamma(red); green = encode_pixel_gamma(green); blue = encode_pixel_gamma(blue);
        }
        intensity = 0.298839 * red + 0.586811 * green + 0.114350 * blue;
        break;
      case 6:
        if (colorspace == ORC_CS_SRGB) {
          red = decode_pixel_gamma(red); green = decode_pixel_gamma(green); blue = decode_pixel_gamma(blue);
        }
        intensity = 0.298839 * red + 0.586811 * green + 0.114350 * blue;
        break;
      case 8:
        if (colorspace == ORC_CS_SRGB) {
          red = decode_pixel_gamma(red); green = decode_pixel_gamma(green); blue = decode_pixel_gamma(blue);
        }
        intensity = 0.212656 * red + 0.715158 * green + 0.072186 * blue;
        break;
      case 9: intensity = (double) (sqrt((double) red * red + green * green + blue * blue) / sqrt(3.0)); break;
      default:                                  /* Rec709Luma and Undefined */
        if (colorspace == ORC_CS_RGB) {
          red = encode_pixel_gamma(red); green = encode_pixel_gamma(green); blue = encode_pixel_gamma(blue);
        }
        intensity = 0.212656 * red + 0.715158 * green + 0.072186 * blue;
        break;
    }
    q[0] = (float) intensity;
  }
  for (i = 0; i < n; i++) {                       /* the re-laid-out cache: gray, then alpha */
    const float gray = buf[i * ch], alpha = buf[i * ch + ch - 1];
    buf[i * out_ch] = gray;
    if (out_ch == 2) buf[i * out_ch + 1] = alpha;
  }
  return out_ch;
}

/* statistic.c:962-1170 FunctionImage (statistic.h:130-137 MagickFunction) on the channels whose bit is set in
   update_mask (bit c: channel c carries the Update trait) */
int orc_function(float *buf, size_t w, size_t h, int ch, int function, size_t n_params, const double *params,
                 unsigned update_mask)
{
  long i, n = (long) (w * h);
  if (ch < 1 || ch > 4 || function < 0 || function > 4) return -1;
#pragma omp parallel for schedule(static)
  for (i = 0; i < n; i++) {
    float *q = buf + (size_t) i * ch;
    int c;
    for (c = 0; c < ch; c++) {
      const double pixel = (double) q[c];
      double result = 0.0;
      size_t k;
      if (((update_mask >> c) & 1u) == 0) continue;
      switch (function) {
        case 3:                                   /* Polynomial */
          for (k = 0; k < n_params; k++) result = result * QS * pixel + params[k];
          result *= QR;
          break;
        case 4: {                                 /* Sinusoid */
          const double frequency = n_params >= 1 ? params[0] : 1.0, phase = n_params >= 2 ? params[1] : 0.0,
                       amplitude = n_params >= 3 ? params[2] : 0.5, bias = n_params >= 4 ? params[3] : 0.5;
          result = QR * (amplitude * sin((double) (2.0 * PI_ * (frequency * QS * pixel + phase / 360.0))) + bias);
          break;
        }
        case 1: {                                 /* Arcsin */
          const double width = n_params >= 1 ? params[0] : 1.0, center = n_params >= 2 ? params[1] : 0.5,
                       range = n_params >= 3 ? params[2] : 1.0, bias = n_params >= 4 ? params[3] : 0.5;
          result = 2.0 * precip(width) * (QS * pixel - center);
          if (result <= -1.0) result = bias - range / 2.0;
          else if (result >= 1.0) result = bias + range / 2.0;
          else result = (double) (range / PI_ * asin((double) result) + bias);
          result *= QR;
          break;
        }
        case 2: {                                 /* Arctan */
          const double slope = n_params >= 1 ? params[0] : 1.0, center = n_params >= 2 ? params[1] : 0.5,
                       range = n_params >= 3 ? params[2] : 1.0, bias = n_params >= 4 ? params[3] : 0.5;
          result = PI_ * slope * (QS * pixel - center);
          result = QR * (range / PI_ * atan((double) result) + bias);
          break;
        }
        default: break;                           /* Undefined: 0 */
      }
      q[c] = (float) result;
    }
  }
  return 0;
}
