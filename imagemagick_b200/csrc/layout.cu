// layout.cu -- TransformImageColorspace (MagickCore/colorspace.c:1751) to and from the colourspaces that change the
// channel layout of the pixel cache, out of place:
//   sRGB -> GRAY        :901-957    gray = 0.212656 R + 0.715158 G + 0.072186 B into channel 0; SetImageColorspace(GRAY)
//                                   then keeps gray (and alpha)
//   sRGB -> LinearGRAY  :843-900    the same sum of DecodePixelGamma of each channel
//   GRAY -> sRGB        :2224-2291  SetImageColorspace(sRGB) runs first and copies the gray sample into R, G and B
//                                   (pixel.c:6149-6153, cache.c:783-796); the loop writes the same sum into all three
//   LinearGRAY -> sRGB  :2171-2223  ... of EncodePixelGamma of each channel
//   sRGB -> CMYK        :778-842    SetImageColorspace(CMYK) runs first (K = 0), so ConvertRGBToCMYK sees a CMYK-tagged
//                                   pixel and takes its linear branch (colorspace-private.h:1600-1611)
//   CMYK -> sRGB        :2110-2170  ConvertCMYKToRGB (colorspace-private.h:131-139) on the CMYK layout; the cache then
//                                   drops K
// SetPixelViaPixelInfo clamps every channel with ClampToQuantum, a float cast in HDRI: alpha is carried over as it is.
// Every other pair goes through sRGB (:1770-1781): the in-place legs of colorspace.cu / hexcone.cu run on a
// stream-ordered temporary (source side) or on dst (target side); src is never written.
//
// The sums and the CMYK arithmetic are the reference's IEEE double operations in its order, unfused: bit exact.  The
// gamma steps are the colorspace_math.cuh curves with NaN / +inf settled like the reference's: <= 1 ULP.
// One thread per pixel.  RGBA / CMYK (16 bytes) move as float4 and gray + alpha (8 bytes) as float2 when both buffers
// are aligned for their widths; RGB, gray and CMYKA (20 bytes, never 16-byte aligned) move per channel.
#include "mb200_internal.h"
#include "colorspace_math.cuh"
#include "hexcone.cuh"

#include <cuda_runtime.h>

#include <cstdint>

namespace mb200 {
namespace {

enum Leg { kToGray, kToLinearGray, kFromGray, kFromLinearGray, kToCmyk, kFromCmyk };

__host__ __device__ constexpr int base_channels(int cs) {
  return cs == MB200_CMYKColorspace ? 4 : (cs == MB200_GRAYColorspace || cs == MB200_LinearGRAYColorspace) ? 1 : 3;
}
__host__ __device__ constexpr int leg_src(int leg) {
  return leg == kFromGray || leg == kFromLinearGray ? 1 : leg == kFromCmyk ? 4 : 3;
}
__host__ __device__ constexpr int leg_dst(int leg) {
  return leg == kToGray || leg == kToLinearGray ? 1 : leg == kToCmyk ? 4 : 3;
}
bool is_layout_space(int cs) {
  return cs == MB200_GRAYColorspace || cs == MB200_LinearGRAYColorspace || cs == MB200_CMYKColorspace;
}

template <int CH, bool VEC>
__device__ __forceinline__ void load_px(const float *p, float (&v)[5]) {
  if (VEC && CH == 4) {
    const float4 t = *reinterpret_cast<const float4 *>(p);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  } else if (VEC && CH == 2) {
    const float2 t = *reinterpret_cast<const float2 *>(p);
    v[0] = t.x; v[1] = t.y;
  } else {
#pragma unroll
    for (int c = 0; c < CH; ++c) v[c] = p[c];
  }
}
template <int CH, bool VEC>
__device__ __forceinline__ void store_px(float *q, const float (&v)[5]) {
  if (VEC && CH == 4) *reinterpret_cast<float4 *>(q) = make_float4(v[0], v[1], v[2], v[3]);
  else if (VEC && CH == 2) *reinterpret_cast<float2 *>(q) = make_float2(v[0], v[1]);
  else {
#pragma unroll
    for (int c = 0; c < CH; ++c) q[c] = v[c];
  }
}

// 0.212656*R + 0.715158*G + 0.072186*B, left to right (colorspace.c:888, :945, :2213, :2280)
__device__ __forceinline__ double gray_sum(double r, double g, double b) {
  return ad(ad(ml(0.212656, r), ml(0.715158, g)), ml(0.072186, b));
}

template <int LEG, bool ALPHA, bool VEC>
__global__ void __launch_bounds__(256) layout_kernel(const float *__restrict__ src, float *__restrict__ dst, size_t npixels) {
  constexpr int SRC_CH = leg_src(LEG) + (ALPHA ? 1 : 0), DST_CH = leg_dst(LEG) + (ALPHA ? 1 : 0);
  const size_t i = static_cast<size_t>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= npixels) return;
  float in[5], out[5];
  load_px<SRC_CH, VEC>(src + i * SRC_CH, in);
  if (LEG == kToGray || LEG == kToLinearGray) {
    double r = in[0], g = in[1], b = in[2];
    if (LEG == kToLinearGray) { r = decode_pixel_gamma<true>(r); g = decode_pixel_gamma<true>(g); b = decode_pixel_gamma<true>(b); }
    out[0] = static_cast<float>(gray_sum(r, g, b));
  } else if (LEG == kFromGray || LEG == kFromLinearGray) {
    const double v = LEG == kFromLinearGray ? encode_pixel_gamma<true>(static_cast<double>(in[0])) : static_cast<double>(in[0]);
    out[0] = out[1] = out[2] = static_cast<float>(gray_sum(v, v, v));
  } else if (LEG == kToCmyk) {                                             // colorspace-private.h:1589-1633
    const double red = ml(QS, in[0]), green = ml(QS, in[1]), blue = ml(QS, in[2]);
    if (tiny(red) && tiny(green) && tiny(blue)) {                          // black: only K changes
      out[0] = in[0]; out[1] = in[1]; out[2] = in[2]; out[3] = static_cast<float>(QR);
    } else {
      const double cyan = sb(1.0, red), magenta = sb(1.0, green), yellow = sb(1.0, blue);
      double black = cyan;
      if (magenta < black) black = magenta;
      if (yellow < black) black = yellow;
      const double k = reciprocal(sb(1.0, black));
      out[0] = static_cast<float>(ml(QR, ml(k, sb(cyan, black))));
      out[1] = static_cast<float>(ml(QR, ml(k, sb(magenta, black))));
      out[2] = static_cast<float>(ml(QR, ml(k, sb(yellow, black))));
      out[3] = static_cast<float>(ml(QR, black));
    }
  } else {                                                                 // kFromCmyk, colorspace-private.h:131-139
    const double black = in[3], white = sb(QR, black);
#pragma unroll
    for (int c = 0; c < 3; ++c) out[c] = static_cast<float>(sb(QR, ad(ml(ml(QS, in[c]), white), black)));
  }
  if (ALPHA) out[DST_CH - 1] = in[SRC_CH - 1];
  store_px<DST_CH, VEC>(dst + i * DST_CH, out);
}

bool aligned_for(const void *p, int channels) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  return channels == 4 ? (a & 15) == 0 : channels == 2 ? (a & 7) == 0 : true;
}

template <int LEG, bool ALPHA>
void launch_leg_as(const float *src, float *dst, size_t npixels, cudaStream_t s) {
  constexpr int SRC_CH = leg_src(LEG) + (ALPHA ? 1 : 0), DST_CH = leg_dst(LEG) + (ALPHA ? 1 : 0);
  const unsigned blocks = static_cast<unsigned>((npixels + 255) / 256);
  if (aligned_for(src, SRC_CH) && aligned_for(dst, DST_CH)) layout_kernel<LEG, ALPHA, true><<<blocks, 256, 0, s>>>(src, dst, npixels);
  else layout_kernel<LEG, ALPHA, false><<<blocks, 256, 0, s>>>(src, dst, npixels);
}

template <int LEG>
int launch_leg(const float *src, float *dst, size_t npixels, bool alpha, cudaStream_t s) {
  if (alpha) launch_leg_as<LEG, true>(src, dst, npixels, s);
  else launch_leg_as<LEG, false>(src, dst, npixels, s);
  count_launch();
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? MB200_OK : cuda_fail(e, "colorspace layout launch");
}

// The layout leg between `cs` and sRGB (forward: sRGB -> cs).
int run_layout_leg(int cs, bool forward, const float *src, float *dst, size_t npixels, bool alpha, cudaStream_t s) {
  if (cs == MB200_CMYKColorspace)
    return forward ? launch_leg<kToCmyk>(src, dst, npixels, alpha, s) : launch_leg<kFromCmyk>(src, dst, npixels, alpha, s);
  if (cs == MB200_GRAYColorspace)
    return forward ? launch_leg<kToGray>(src, dst, npixels, alpha, s) : launch_leg<kFromGray>(src, dst, npixels, alpha, s);
  return forward ? launch_leg<kToLinearGray>(src, dst, npixels, alpha, s)
                 : launch_leg<kFromLinearGray>(src, dst, npixels, alpha, s);
}

struct PoolBuffer {            // stream-ordered temporary from the library's pool, freed (stream-ordered) on scope exit
  float *ptr = nullptr;
  cudaStream_t s;
  explicit PoolBuffer(cudaStream_t stream) : s(stream) {}
  int alloc(size_t bytes) {
    const cudaError_t e = cudaMallocAsync(reinterpret_cast<void **>(&ptr), bytes, temp_pool(), s);
    if (e != cudaSuccess) { ptr = nullptr; return cuda_fail(e, "colorspace layout: temporary"); }
    return MB200_OK;
  }
  ~PoolBuffer() { if (ptr) cudaFreeAsync(ptr, s); }
  PoolBuffer(const PoolBuffer &) = delete;
  PoolBuffer &operator=(const PoolBuffer &) = delete;
};

}  // namespace

int colorspace_layout_check(const void *src, int src_channels, const void *dst, int dst_channels, size_t width,
                            size_t height, int from, int to, const mb200_colorspace_options *options) {
  if (!src || !dst || src == dst || width == 0 || height == 0) return fail(MB200_EINVAL, "colorspace layout: bad arguments");
  const int alpha = src_channels - base_channels(from);
  if ((alpha != 0 && alpha != 1) || dst_channels != base_channels(to) + alpha)
    return fail(MB200_EINVAL, "colorspace layout: %d -> %d channels do not fit colourspaces %d -> %d", src_channels,
                dst_channels, from, to);
  if (!(is_layout_space(from) || colorspace_served(from)) || !(is_layout_space(to) || colorspace_served(to)))
    return fail(MB200_EUNSUPPORTED, "colorspace %d -> %d not implemented", from, to);
  if (options && (options->set & MB200_CO_ILLUMINANT) && (options->illuminant < 0 || options->illuminant > 10))
    return fail(MB200_EINVAL, "colorspace: illuminant %d", options->illuminant);
  if (width * height > 0xffffffffull * 256) return fail(MB200_EINVAL, "colorspace: image too large");
  return MB200_OK;
}

int launch_colorspace_layout(const float *src, int src_channels, float *dst, int dst_channels, size_t npixels, int from,
                             int to, const mb200_colorspace_options *options, void *stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const bool alpha = src_channels != base_channels(from);
  const int rgb_channels = 3 + (alpha ? 1 : 0);
  const size_t rgb_bytes = npixels * rgb_channels * sizeof(float);
  cudaError_t e;
  if (from == to) {
    e = cudaMemcpyAsync(dst, src, npixels * src_channels * sizeof(float), cudaMemcpyDeviceToDevice, s);
    return e == cudaSuccess ? MB200_OK : cuda_fail(e, "colorspace layout: copy");
  }
  const bool from_layout = is_layout_space(from), to_layout = is_layout_space(to);
  if (from_layout && to == MB200_sRGBColorspace) return run_layout_leg(from, false, src, dst, npixels, alpha, s);
  if (from == MB200_sRGBColorspace && to_layout) return run_layout_leg(to, true, src, dst, npixels, alpha, s);
  // `work` holds the image in sRGB between the two legs: dst itself when the target is a 3/4-channel space whose
  // in-place leg can run there (3 channels, or RGBA on a 16-byte boundary), a temporary otherwise
  const bool work_is_dst = !to_layout && (rgb_channels == 3 || aligned_for(dst, 4));
  PoolBuffer tmp(s);
  float *work = dst;
  int rc = MB200_OK;
  if (!work_is_dst) {
    rc = tmp.alloc(rgb_bytes);
    if (rc) return rc;
    work = tmp.ptr;
  }
  if (from_layout) {
    rc = run_layout_leg(from, false, src, work, npixels, alpha, s);
    if (rc == MB200_OK && !to_layout && to != MB200_sRGBColorspace)
      rc = launch_colorspace(work, npixels, rgb_channels, MB200_sRGBColorspace, to, options, s);
  } else {
    e = cudaMemcpyAsync(work, src, rgb_bytes, cudaMemcpyDeviceToDevice, s);
    rc = e == cudaSuccess ? MB200_OK : cuda_fail(e, "colorspace layout: copy");
    // a non-layout target: both in-place legs, exactly as the in-place entry points run them
    if (rc == MB200_OK) rc = launch_colorspace(work, npixels, rgb_channels, from, to_layout ? MB200_sRGBColorspace : to, options, s);
  }
  if (rc == MB200_OK && to_layout) rc = run_layout_leg(to, true, work, dst, npixels, alpha, s);
  if (rc == MB200_OK && !to_layout && work != dst) {
    e = cudaMemcpyAsync(dst, work, rgb_bytes, cudaMemcpyDeviceToDevice, s);
    if (e != cudaSuccess) rc = cuda_fail(e, "colorspace layout: copy");
  }
  return rc;
}

}  // namespace mb200
