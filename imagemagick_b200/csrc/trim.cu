// trim.cu -- GetImageBoundingBox's scan (MagickCore/attribute.c:457-551): the per-row summaries the serial bounding-box
// rule reduces to (mb200_bounding_box_from_rows in geometry_plan.cpp applies that rule).
//
// One read-only pass.  Every CTA loads the four corner pixels (the targets, :457-480) itself, so nothing travels to the
// host before the scan, and finds which targets are bitwise equal: those share one comparison, so the common "all
// corners are the background" case costs one IsFuzzyEquivalencePixelInfo per pixel instead of four.  The comparison is
// fuzzy.cuh's, in double; this file is compiled with -fmad=false.
//
// Row y's summary is four 32-bit words, all 0 when nothing in the row mismatches (so the buffer starts from a memset):
//   [0] columns - the first x that mismatches target 0    [1] 1 + the last x that mismatches target 1
//   [2] 1 when any x mismatches target 2                  [3] columns - the first x that mismatches target 3
// Each is a maximum, reduced per warp (__reduce_max_sync) and then merged with one atomicMax per warp and word, issued
// only when the warp found a mismatch.  Offsets are 64-bit and both loops grid-stride.
#include "fuzzy.cuh"
#include "mb200_internal.h"

#include <cuda_runtime.h>

namespace mb200 {
namespace {

constexpr int kThreads = 256;
constexpr int kUnroll = 4;               // pixels each thread has in flight

struct Scan {
  const float *src;
  unsigned *rows;
  long long w, h;
  double fuzz_sq;
  int cls;
};

template <int CH>
struct Raw {
  float v[CH];
};

template <int CH, bool VEC>
__device__ __forceinline__ Raw<CH> load(const float *row, long long x) {
  Raw<CH> r;
  if constexpr (VEC) {
    const float4 q = __ldg(reinterpret_cast<const float4 *>(row) + x);
    r.v[0] = q.x;
    r.v[1] = q.y;
    r.v[2] = q.z;
    r.v[3] = q.w;
  } else {
#pragma unroll
    for (int c = 0; c < CH; ++c) r.v[c] = __ldg(row + x * CH + c);
  }
  return r;
}

// GetPixelInfoPixel for the six layouts: gray, gray + alpha, RGB, RGBA (CMYK false) and CMYK, CMYKA (CMYK true).
template <int CH, bool CMYK>
__device__ __forceinline__ FuzzyPixel info(const Raw<CH> &r) {
  FuzzyPixel p;
  p.red = r.v[0];
  p.green = CH >= 3 ? r.v[CH >= 3 ? 1 : 0] : r.v[0];
  p.blue = CH >= 3 ? r.v[CH >= 3 ? 2 : 0] : r.v[0];
  p.black = CMYK ? r.v[CMYK ? 3 : 0] : 0.0;
  p.alpha = CH == 2 || (CH == 4 && !CMYK) || CH == 5 ? r.v[CH - 1] : 65535.0;
  return p;
}

template <int CH>
__device__ __forceinline__ bool same_bits(const Raw<CH> &a, const Raw<CH> &b) {
  bool eq = true;
#pragma unroll
  for (int c = 0; c < CH; ++c) eq &= __float_as_uint(a.v[c]) == __float_as_uint(b.v[c]);
  return eq;
}

template <int CH, bool CMYK, bool VEC>
__global__ void __launch_bounds__(kThreads) bounding_box_rows(const __grid_constant__ Scan s) {
  constexpr bool kAlpha = CH == 2 || (CH == 4 && !CMYK) || CH == 5;
  const long long w = s.w, h = s.h;
  // the targets: [0] top-left, [1] top-right, [2] bottom-left, [3] bottom-right; alias[k] is the first target with
  // target k's bits, whose mismatch target k reuses
  const Raw<CH> r0 = load<CH, VEC>(s.src, 0), r1 = load<CH, VEC>(s.src, w - 1);
  const float *last = s.src + (h - 1) * w * CH;
  const Raw<CH> r2 = load<CH, VEC>(last, 0), r3 = load<CH, VEC>(last, w - 1);
  const FuzzyPixel t0 = info<CH, CMYK>(r0), t1 = info<CH, CMYK>(r1), t2 = info<CH, CMYK>(r2), t3 = info<CH, CMYK>(r3);
  const int a1 = same_bits(r1, r0) ? 0 : 1;
  const int a2 = same_bits(r2, r0) ? 0 : same_bits(r2, r1) ? 1 : 2;
  const int a3 = same_bits(r3, r0) ? 0 : same_bits(r3, r1) ? 1 : same_bits(r3, r2) ? 2 : 3;
  const double fuzz_sq = s.fuzz_sq;
  const int cls = s.cls;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long y = blockIdx.y; y < h; y += gridDim.y) {
    const float *row = s.src + y * w * CH;
    unsigned f0 = 0, f1 = 0, f2 = 0, f3 = 0;
    for (long long x0 = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; x0 < w; x0 += stride * kUnroll) {
      Raw<CH> v[kUnroll];
#pragma unroll
      for (int u = 0; u < kUnroll; ++u)
        if (x0 + u * stride < w) v[u] = load<CH, VEC>(row, x0 + u * stride);
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        const long long x = x0 + u * stride;
        if (x >= w) break;
        const FuzzyPixel p = info<CH, CMYK>(v[u]);
        const bool m0 = !fuzzy_equivalent(p, t0, fuzz_sq, kAlpha, cls);
        const bool m1 = a1 == 0 ? m0 : !fuzzy_equivalent(p, t1, fuzz_sq, kAlpha, cls);
        const bool m2 = a2 == 0 ? m0 : a2 == 1 ? m1 : !fuzzy_equivalent(p, t2, fuzz_sq, kAlpha, cls);
        const bool m3 = a3 == 0 ? m0 : a3 == 1 ? m1 : a3 == 2 ? m2 : !fuzzy_equivalent(p, t3, fuzz_sq, kAlpha, cls);
        const unsigned from_end = static_cast<unsigned>(w - x);
        if (m0) f0 = max(f0, from_end);
        if (m1) f1 = max(f1, static_cast<unsigned>(x + 1));
        if (m2) f2 = 1;
        if (m3) f3 = max(f3, from_end);
      }
    }
    f0 = __reduce_max_sync(0xffffffffu, f0);
    f1 = __reduce_max_sync(0xffffffffu, f1);
    f2 = __reduce_max_sync(0xffffffffu, f2);
    f3 = __reduce_max_sync(0xffffffffu, f3);
    if ((threadIdx.x & 31) == 0 && (f0 | f1 | f2 | f3)) {
      unsigned *out = s.rows + 4 * y;
      if (f0) atomicMax(out + 0, f0);
      if (f1) atomicMax(out + 1, f1);
      if (f2) atomicMax(out + 2, f2);
      if (f3) atomicMax(out + 3, f3);
    }
  }
}

template <int CH, bool CMYK, bool VEC>
cudaError_t launch(const Scan &s, cudaStream_t stream) {
  const long long per_cta = static_cast<long long>(kThreads) * kUnroll;
  const dim3 grid(static_cast<unsigned>(min((s.w + per_cta - 1) / per_cta, 1024LL)), static_cast<unsigned>(min(s.h, 65535LL)));
  bounding_box_rows<CH, CMYK, VEC><<<grid, kThreads, 0, stream>>>(s);
  return cudaGetLastError();
}

}  // namespace

int bounding_box_check(size_t width, size_t height, int channels, const mb200_trim_options *options) {
  if (!options || width == 0 || height == 0 || channels < 1 || channels > 5 || options->edges < MB200_TRIM_EDGES_UNSET ||
      options->edges > 15)
    return fail(MB200_EINVAL, "bounding box: bad arguments");
  const bool cmyk = options->colorspace == MB200_CMYKColorspace;
  if (cmyk ? channels < 4 : channels == 5)
    return fail(MB200_EINVAL, "bounding box: CMYK images have 4 or 5 channels, 5 channels are CMYKA");
  if (width > 0xffffffffull) return fail(MB200_EUNSUPPORTED, "bounding box: images wider than 2^32 - 1 are not supported");
  return MB200_OK;
}

int launch_bounding_box(const float *src, size_t width, size_t height, int channels, const mb200_trim_options *options,
                        unsigned *d_rows, void *stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaError_t e = cudaMemsetAsync(d_rows, 0, height * 4 * sizeof(unsigned), st);
  if (e != cudaSuccess) return cuda_fail(e, "bounding box: clear");
  Scan s;
  s.src = src;
  s.rows = d_rows;
  s.w = static_cast<long long>(width);
  s.h = static_cast<long long>(height);
  s.fuzz_sq = fuzzy_fuzz_sq(options->fuzz);
  const int cs = options->colorspace;
  s.cls = cs == MB200_CMYKColorspace ? kFuzzyCMYK
          : (cs == MB200_HCLColorspace || cs == MB200_HCLpColorspace || cs == MB200_HSBColorspace ||
             cs == MB200_HSIColorspace || cs == MB200_HSLColorspace || cs == MB200_HSVColorspace) ? kFuzzyHue
                                                                                                   : kFuzzyPlain;
  const bool cmyk = s.cls == kFuzzyCMYK;
  switch (channels) {
    case 1: e = launch<1, false, false>(s, st); break;
    case 2: e = launch<2, false, false>(s, st); break;
    case 3: e = launch<3, false, false>(s, st); break;
    case 4:
      if (cmyk) e = launch<4, true, false>(s, st);
      else if (reinterpret_cast<uintptr_t>(src) % 16 == 0) e = launch<4, false, true>(s, st);
      else e = launch<4, false, false>(s, st);
      break;
    default: e = launch<5, true, false>(s, st); break;
  }
  if (e != cudaSuccess) return cuda_fail(e, "bounding box launch");
  count_family(kBoundingBox);
  count_launch();
  return MB200_OK;
}

}  // namespace mb200
