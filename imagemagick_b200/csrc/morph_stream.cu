// morph_stream.cu -- ErodeMorphology / DilateMorphology for the structuring elements the reference's
// own generators produce (Disk, Square, Diamond, Octagon, Plus; morphology.c:1560-1700), streamed
// through registers.
//
// Semantics are MorphologyPrimitive's (MagickCore/morphology.c:2980-3036): erode = min over the kernel
// cells >= 0.5 starting from the centre value, dilate = max over the cells > 0.5 of the reflected kernel
// starting from 0.0; edge-clamped source; the result is one of the input floats (bit exact).
//
// Every row v of these kernels is one run of cells centred on the origin column, half-width hw[v].
// A warp owns 32 - 2R adjacent pixel columns (R = max hw; R halo lanes either side) and walks down a
// strip of rows.  Per input row a lane
//   1. takes its pixel from a K-deep register ring of prefetched loads (one coalesced 512-B request per warp),
//   2. builds the nested run extrema H[j] = op(p[x-j..x+j]) with 2 SHFL + 1 FMNMX3 per level and component,
//   3. folds H[hw[v]] into the K rotating output accumulators (the row is kernel row v of output r+oy-v),
//   4. emits the accumulator that just received its last kernel row.
// hw[] is a template parameter: the accumulator index and the level index are both compile-time, so the
// whole neighbourhood costs R + K min/max per component and no shared memory -- against one shared-memory
// read per active cell (29 for Disk:3) in the generic kernel.  Shapes outside the instantiated table, the
// `changed` count and other channel counts use morph2d.cu.
#include "mb200_internal.h"

#include <cuda_runtime.h>

#include <cmath>
#include <limits>

namespace mb200 {
namespace {

// CODE packs hw[v] + 1 in 4 bits per kernel row (0 = empty row), row 0 in the low nibble.
__host__ __device__ constexpr int shape_hw(unsigned long long code, int v) { return static_cast<int>((code >> (4 * v)) & 15ull) - 1; }
__host__ __device__ constexpr int shape_radius(unsigned long long code, int k) {
  int r = 0;
  for (int v = 0; v < k; ++v) r = shape_hw(code, v) > r ? shape_hw(code, v) : r;
  return r;
}

template <int CH> struct Px { float v[CH]; };

template <int CH>
__device__ __forceinline__ Px<CH> load_px(const float *p) {
  Px<CH> r;
  if constexpr (CH == 4) {
    const float4 t = __ldg(reinterpret_cast<const float4 *>(p));
    r.v[0] = t.x; r.v[1] = t.y; r.v[2] = t.z; r.v[3] = t.w;
  } else {
#pragma unroll
    for (int c = 0; c < CH; ++c) r.v[c] = __ldg(p + c);
  }
  return r;
}

template <int CH>
__device__ __forceinline__ void store_px(float *p, const Px<CH> &r) {
  if constexpr (CH == 4) {
    *reinterpret_cast<float4 *>(p) = make_float4(r.v[0], r.v[1], r.v[2], r.v[3]);
  } else {
#pragma unroll
    for (int c = 0; c < CH; ++c) p[c] = r.v[c];
  }
}

template <bool DILATE>
__device__ __forceinline__ float op2(float a, float b) { return DILATE ? fmaxf(a, b) : fminf(a, b); }
template <bool DILATE>
__device__ __forceinline__ float op3(float a, float b, float c) { return DILATE ? fmaxf(a, fmaxf(b, c)) : fminf(a, fminf(b, c)); }

struct StreamArgs {
  const float *src;
  float *dst;
  int width, height;
  int oy;         // window row of the origin
  int strip;      // output rows per CTA
};

template <int CH, bool DILATE, int K, unsigned long long CODE>
__global__ void __launch_bounds__(128) minmax_stream_kernel(const StreamArgs a) {
  constexpr int R = shape_radius(CODE, K);
  constexpr int USE = 32 - 2 * R;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int group = blockIdx.x * 4 + warp;
  const int x = group * USE + lane - R;
  if (group * USE >= a.width) return;                           // whole warp outside the image
  const int xc = min(max(x, 0), a.width - 1);
  const bool writer = lane >= R && lane < 32 - R && x < a.width;
  const int y0 = blockIdx.y * a.strip;
  const int nout = min(a.strip, a.height - y0);
  const int hmax = a.height - 1;
  const size_t pitch = static_cast<size_t>(a.width) * CH;
  const float *col = a.src + static_cast<size_t>(xc) * CH;
  float *outp = a.dst + static_cast<size_t>(y0) * pitch + static_cast<size_t>(max(x, 0)) * CH;
  const float init = DILATE ? 0.0f : __int_as_float(0x7f800000);
  // Erode keeps a NaN centre (the reference's `sample < pixel` never replaces it, morphology.c:2911), which the min
  // fold drops: bit q of centre_nan records that accumulator q's centre sample -- the lane's own sample at kernel row
  // oy, slot (s + cbase) mod K -- has a NaN component, and its output then takes the centre's NaN components.
  const int cbase = K - 1 - a.oy;                                // 0 <= oy < K
  unsigned centre_nan = 0;

  Px<CH> acc[K], pre[K];
#pragma unroll
  for (int q = 0; q < K; ++q)
#pragma unroll
    for (int c = 0; c < CH; ++c) acc[q].v[c] = init;
  int r = y0 - a.oy;                                             // source row of step 0
#pragma unroll
  for (int s = 0; s < K; ++s) pre[s] = load_px<CH>(col + static_cast<size_t>(min(max(r + s, 0), hmax)) * pitch);
  r += K;

  const int total = a.strip + K - 1;                             // steps (strip + K - 1 is a multiple of K)
  int j = -(K - 1);                                              // output row (relative to y0) finished by the step
#pragma unroll 1
  for (int mb = 0; mb < total; mb += K) {
#pragma unroll
    for (int s = 0; s < K; ++s) {
      const Px<CH> p = pre[s];
      pre[s] = load_px<CH>(col + static_cast<size_t>(min(max(r, 0), hmax)) * pitch);
      ++r;
      if constexpr (!DILATE) {
        unsigned nan = 0;
#pragma unroll
        for (int c = 0; c < CH; ++c) nan |= (__float_as_uint(p.v[c]) & 0x7fffffffu) > 0x7f800000u;
        const int cs = s + cbase >= K ? s + cbase - K : s + cbase;
        centre_nan |= nan << cs;
      }
      Px<CH> h[R + 1];
      h[0] = p;
#pragma unroll
      for (int lv = 1; lv <= R; ++lv) {
#pragma unroll
        for (int c = 0; c < CH; ++c) {
          const float lo = __shfl_sync(0xffffffffu, p.v[c], (lane - lv) & 31);
          const float hi = __shfl_sync(0xffffffffu, p.v[c], (lane + lv) & 31);
          h[lv].v[c] = op3<DILATE>(h[lv - 1].v[c], lo, hi);
        }
      }
#pragma unroll
      for (int v = 0; v < K; ++v) {
        const int hwv = shape_hw(CODE, v);
        if (hwv >= 0) {
          const int slot = (s + K - 1 - v) % K;
#pragma unroll
          for (int c = 0; c < CH; ++c) acc[slot].v[c] = op2<DILATE>(acc[slot].v[c], h[hwv].v[c]);
        }
      }
      const int done = s % K;
      if (writer && static_cast<unsigned>(j) < static_cast<unsigned>(nout)) {
        if constexpr (!DILATE) {
          if ((centre_nan >> done) & 1u) {             // rare: reload the centre (this output's own source pixel)
            const Px<CH> ctr = load_px<CH>(col + static_cast<size_t>(y0 + j) * pitch);
#pragma unroll
            for (int c = 0; c < CH; ++c)
              if (ctr.v[c] != ctr.v[c]) acc[done].v[c] = ctr.v[c];
          }
        }
        store_px<CH>(outp, acc[done]);
      }
      if constexpr (!DILATE) centre_nan &= ~(1u << done);
#pragma unroll
      for (int c = 0; c < CH; ++c) acc[done].v[c] = init;
      if (j >= 0) outp += pitch;
      ++j;
    }
  }
}

using Launcher = cudaError_t (*)(const StreamArgs &, dim3, cudaStream_t);

template <int CH, bool DILATE, int K, unsigned long long CODE>
cudaError_t launch_shape(const StreamArgs &a, dim3 grid, cudaStream_t s) {
  minmax_stream_kernel<CH, DILATE, K, CODE><<<grid, 128, 0, s>>>(a);
  return cudaGetLastError();
}

struct ShapeEntry {
  int k;
  unsigned long long code;
  Launcher fn[2][2];    // [channels == 4][dilate]
};

#define MB200_SHAPE(K, CODE)                                                                         \
  ShapeEntry{K, CODE, {{launch_shape<1, false, K, CODE>, launch_shape<1, true, K, CODE>},             \
                       {launch_shape<4, false, K, CODE>, launch_shape<4, true, K, CODE>}}}

// hw+1 per row, row 0 in the low nibble (the shapes are vertically symmetric, so the order is moot)
const ShapeEntry kShapes[] = {
    MB200_SHAPE(3, 0x121ull),            // Disk:1, Diamond:1, Octagon:1, Plus:1
    MB200_SHAPE(3, 0x222ull),            // Square:1, Disk:1.5
    MB200_SHAPE(5, 0x12321ull),          // Disk:2, Diamond:2
    MB200_SHAPE(5, 0x23332ull),          // Disk:2.5, Octagon:2
    MB200_SHAPE(5, 0x33333ull),          // Square:2
    MB200_SHAPE(5, 0x11311ull),          // Plus:2
    MB200_SHAPE(7, 0x1334331ull),        // Disk:3
    MB200_SHAPE(7, 0x2344432ull),        // Disk:3.5, Octagon:3
    MB200_SHAPE(7, 0x4444444ull),        // Square:3
    MB200_SHAPE(7, 0x1234321ull),        // Diamond:3
    MB200_SHAPE(7, 0x1114111ull),        // Plus:3
    MB200_SHAPE(9, 0x134454431ull),      // Disk:4
    MB200_SHAPE(9, 0x345555543ull),      // Disk:4.5, Octagon:4
    MB200_SHAPE(9, 0x555555555ull),      // Square:4
    MB200_SHAPE(9, 0x123454321ull),      // Diamond:4
    MB200_SHAPE(9, 0x111151111ull),      // Plus:4
    MB200_SHAPE(11, 0x14555655541ull),   // Disk:5
    MB200_SHAPE(11, 0x12345654321ull),   // Diamond:5
    MB200_SHAPE(11, 0x34566666543ull),   // Octagon:5
};

}  // namespace

// kernel_window_order: the primitive's window-order cells (already reflected for dilate); NaN and
// below-threshold cells are inactive.  Returns MB200_EUNSUPPORTED when the shape is not in the table.
int launch_morph_stream(const float *src, float *dst, size_t width, size_t height, int channels, int method,
                        const double *kernel_window_order, int kw, int kh, int ox, int oy, void *stream) {
  if (method != MB200_ErodeMorphology && method != MB200_DilateMorphology) return MB200_EUNSUPPORTED;
  if (channels != 1 && channels != 4) return MB200_EUNSUPPORTED;
  if (kh > 15 || kw > 31 || width > 0x3fffffffull || height > 0x3fffffffull) return MB200_EUNSUPPORTED;
  if (channels == 4 && ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) != 0) return MB200_EUNSUPPORTED;
  const bool dilate = method == MB200_DilateMorphology;
  unsigned long long code = 0;
  for (int v = 0; v < kh; ++v) {
    int first = -1, last = -1, count = 0;
    for (int u = 0; u < kw; ++u) {
      const double k = kernel_window_order[v * kw + u];
      if (k != k) continue;
      if (!(dilate ? (k > 0.5) : (k >= 0.5))) continue;
      if (first < 0) first = u;
      last = u;
      ++count;
    }
    int hw = -1;
    if (count != 0) {
      if (count != last - first + 1 || first + last != 2 * ox) return MB200_EUNSUPPORTED;   // one run centred on ox
      hw = (last - first) / 2;
    }
    if (!dilate && v == oy && hw < 0) hw = 0;     // erode starts from the centre value (morphology.c:2911)
    if (hw > 14) return MB200_EUNSUPPORTED;
    code |= static_cast<unsigned long long>(hw + 1) << (4 * v);
  }
  const ShapeEntry *entry = nullptr;
  for (const ShapeEntry &e : kShapes)
    if (e.k == kh && e.code == code) entry = &e;
  if (entry == nullptr) return MB200_EUNSUPPORTED;
  StreamArgs a{};
  a.src = src; a.dst = dst;
  a.width = static_cast<int>(width); a.height = static_cast<int>(height);
  a.oy = oy;
  int rot = 64 / kh;                               // strip + K - 1 is a whole number of K-step blocks
  if (rot < 2) rot = 2;
  a.strip = rot * kh + 1;
  const int radius = shape_radius(code, kh);
  const int use = 32 - 2 * radius;
  const int groups = (a.width + use - 1) / use;
  dim3 grid((groups + 3) / 4, (a.height + a.strip - 1) / a.strip);
  if (grid.y > 65535) return MB200_EUNSUPPORTED;
  const cudaError_t e = entry->fn[channels == 4 ? 1 : 0][dilate ? 1 : 0](a, grid, static_cast<cudaStream_t>(stream));
  count_launch();
  count_family(kMorphStream);
  if (e != cudaSuccess) return cuda_fail(e, "morph_stream launch");
  return MB200_OK;
}

}  // namespace mb200
