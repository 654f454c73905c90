// morph2d.cu -- the general neighbourhood loop: 2-D convolution (GaussianBlurImage,
// ConvolveImage with arbitrary KernelInfo), ErodeMorphology and DilateMorphology.
//
// Semantics: MorphologyPrimitive's row loop, MagickCore/morphology.c:2811-3220
//   Convolve :2897-2979 (reflected kernel, NaN cells skipped, alpha blending),
//   Erode :2980-3006 (kernel as is, cells >= 0.5, min starting from the centre value),
//   Dilate :3007-3036 (reflected, cells > 0.5, max starting from 0.0),
//   result = ClampToQuantum(PerceptibleReciprocal(gamma)*pixel) :3197, changed :3199.
// Erode/Dilate only select input values, so they are computed in float and are
// bit-exact by construction.
//
// Mapping: a 32x8-pixel output tile per CTA, source tile + halo staged (edge-clamped)
// in shared memory with coalesced loads; taps are read from a small global table
// with warp-uniform (broadcast) loads; the active-cell list is compacted on the host so
// NaN cells cost nothing.  Convolution accumulates in FP64.
#include "mb200_internal.h"

#include <cuda_runtime.h>

namespace mb200 {
namespace {

constexpr double kQuantumScale = 1.0 / 65535.0;
constexpr double kEpsilon = 1.0e-12;
constexpr int kTileW = 32, kTileH = 8;

struct Cell { short du, dv; float pad; double k; };   // window offset (u,v) and tap (window order)

struct Morph2dArgs {
  const float *src;
  float *dst;
  int width, height, channels;
  int ox, oy;            // window top-left = (x - ox, y - oy)
  int kw, kh;
  int ncells;
  const Cell *cells;     // device
  double bias;
  double gamma_scale;    // column-path kh/count factor (morphology.c:2775), else 1
  int method;
  unsigned long long *changed;
};

__device__ __forceinline__ double precise_reciprocal_gamma(double gamma) {
  if (fabs(gamma) >= kEpsilon) return 1.0 / gamma;
  return gamma < 0.0 ? -1.0 / kEpsilon : 1.0 / kEpsilon;
}

template <int CH>
__global__ void __launch_bounds__(kTileW *kTileH) morph2d_kernel(const Morph2dArgs a) {
  extern __shared__ __align__(16) float tile[];
  const int tw = kTileW + a.kw - 1, th = kTileH + a.kh - 1;
  const int bx = blockIdx.x * kTileW, by = blockIdx.y * kTileH;
  const int tid = threadIdx.y * kTileW + threadIdx.x;
  const int wmax = a.width - 1, hmax = a.height - 1;
  // stage (tw x th) pixels, clamped
  const int n = tw * th * CH;
  for (int idx = tid; idx < n; idx += kTileW * kTileH) {
    const int p = idx / CH, c = idx - p * CH;
    const int ty = p / tw, tx = p - ty * tw;
    const int sx = min(max(bx - a.ox + tx, 0), wmax);
    const int sy = min(max(by - a.oy + ty, 0), hmax);
    tile[idx] = __ldg(a.src + (static_cast<size_t>(sy) * a.width + sx) * CH + c);
  }
  __syncthreads();
  const int x = bx + threadIdx.x, y = by + threadIdx.y;
  if (x >= a.width || y >= a.height) return;
  const float *win = tile + (threadIdx.y * tw + threadIdx.x) * CH;   // window top-left
  const float *centre = win + (a.oy * tw + a.ox) * CH;
  float *out = a.dst + (static_cast<size_t>(y) * a.width + x) * CH;
  constexpr bool kHasAlpha = (CH == 2 || CH == 4);
  unsigned nchanged = 0;

  if (a.method == MB200_ConvolveMorphology) {
    double pix[CH];
    double gamma = 0.0;
#pragma unroll
    for (int c = 0; c < CH; ++c) pix[c] = 0.0;
    for (int i = 0; i < a.ncells; ++i) {
      const Cell cell = a.cells[i];
      const float *p = win + (cell.dv * tw + cell.du) * CH;
      if (kHasAlpha) {
        // premultiplied form of :2962-2977: sum K*(A*p), gamma' = sum K*A (QS folded at the end)
        const double al = static_cast<double>(p[CH - 1]);
        const double ka = cell.k * al;
        gamma += ka;
#pragma unroll
        for (int c = 0; c < CH - 1; ++c) pix[c] = fma(ka, static_cast<double>(p[c]), pix[c]);
        pix[CH - 1] = fma(cell.k, al, pix[CH - 1]);
      } else {
#pragma unroll
        for (int c = 0; c < CH; ++c) pix[c] = fma(cell.k, static_cast<double>(p[c]), pix[c]);
      }
    }
    if (kHasAlpha) {
      const double r = precise_reciprocal_gamma(kQuantumScale * gamma) * a.gamma_scale;
#pragma unroll
      for (int c = 0; c < CH - 1; ++c) {
        const double pixel = fma(kQuantumScale, pix[c], a.bias);
        out[c] = static_cast<float>(r * pixel);
        nchanged += fabs(pixel - static_cast<double>(centre[c])) >= kEpsilon;
      }
      const double pixel = a.bias + pix[CH - 1];
      out[CH - 1] = static_cast<float>(a.gamma_scale * pixel);
      nchanged += fabs(pixel - static_cast<double>(centre[CH - 1])) >= kEpsilon;
    } else {
#pragma unroll
      for (int c = 0; c < CH; ++c) {
        const double pixel = a.bias + pix[c];
        out[c] = static_cast<float>(a.gamma_scale * pixel);
        nchanged += fabs(pixel - static_cast<double>(centre[c])) >= kEpsilon;
      }
    }
  } else if (a.method == MB200_HitAndMissMorphology || a.method == MB200_ThinningMorphology ||
             a.method == MB200_ThickenMorphology) {
    // morphology.c:3037-3083: least foreground sample (cells > 0.7) minus greatest background sample (cells < 0.3), never
    // negative; Thinning / Thicken subtract it from / add it to the centre.  The host keeps foreground and background
    // cells only (k = 1 / 0).  Selections of floats, one double subtraction / addition, one rounding: bit exact.
    float lo[CH], hi[CH];
#pragma unroll
    for (int c = 0; c < CH; ++c) { lo[c] = 65535.0f; hi[c] = 0.0f; }
    for (int i = 0; i < a.ncells; ++i) {
      const Cell cell = a.cells[i];
      const float *p = win + (cell.dv * tw + cell.du) * CH;
      const bool fg = cell.k > 0.5;
#pragma unroll
      for (int c = 0; c < CH; ++c) {
        const float v = p[c];
        if (fg) { if (v < lo[c]) lo[c] = v; }
        else { if (v > hi[c]) hi[c] = v; }
      }
    }
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      double m = __dsub_rn(static_cast<double>(lo[c]), static_cast<double>(hi[c]));
      if (m < 0.0) m = 0.0;
      const double centre_v = static_cast<double>(centre[c]);
      double pixel = m;
      if (a.method == MB200_ThinningMorphology) pixel = __dsub_rn(centre_v, m);
      else if (a.method == MB200_ThickenMorphology) pixel = __dadd_rn(centre_v, m);
      out[c] = static_cast<float>(pixel);
      nchanged += fabs(__dsub_rn(pixel, centre_v)) >= kEpsilon;
    }
  } else if (a.method == MB200_ErodeIntensityMorphology || a.method == MB200_DilateIntensityMorphology) {
    // :3084-3137: the whole pixel of least / greatest intensity (pixel.c:2356, Rec709 luma of an sRGB / gray image,
    // three products summed left to right without contraction), first one in scan order; when no cell qualifies the
    // reference stores 0 (Erode) or the centre (Dilate) and counts the change.  Copied pixels are not counted (:3186).
    const bool erode = a.method == MB200_ErodeIntensityMorphology;
    double best = erode ? 65535.0 : 0.0;
    const float *pick = nullptr;
    for (int i = 0; i < a.ncells; ++i) {
      const Cell cell = a.cells[i];
      const float *p = win + (cell.dv * tw + cell.du) * CH;
      double intensity = static_cast<double>(p[0]);         // one channel: the gray value itself (pixel.c:2366)
      if (CH >= 2) {                                        // gray + alpha evaluates the same expression on (g, g, g)
        const double green = static_cast<double>(p[CH >= 3 ? 1 : 0]), blue = static_cast<double>(p[CH >= 3 ? 2 : 0]);
        intensity = __dadd_rn(__dadd_rn(__dmul_rn(0.212656, intensity), __dmul_rn(0.715158, green)), __dmul_rn(0.072186, blue));
      }
      if (erode ? intensity < best : intensity > best) { best = intensity; pick = p; }
    }
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      if (pick != nullptr) out[c] = pick[c];
      else {
        const float v = erode ? 0.0f : centre[c];
        out[c] = v;
        nchanged += fabs(static_cast<double>(v) - static_cast<double>(centre[c])) >= kEpsilon;
      }
    }
  } else if (a.method == MB200_IterativeDistanceMorphology) {
    // :3138-3181: min over the cells of sample + k (reflected kernel), starting from the centre
    double pix[CH];
#pragma unroll
    for (int c = 0; c < CH; ++c) pix[c] = static_cast<double>(centre[c]);
    for (int i = 0; i < a.ncells; ++i) {
      const Cell cell = a.cells[i];
      const float *p = win + (cell.dv * tw + cell.du) * CH;
#pragma unroll
      for (int c = 0; c < CH; ++c) {
        const double v = __dadd_rn(static_cast<double>(p[c]), cell.k);
        if (v < pix[c]) pix[c] = v;
      }
    }
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      out[c] = static_cast<float>(pix[c]);
      nchanged += fabs(__dsub_rn(pix[c], static_cast<double>(centre[c]))) >= kEpsilon;
    }
  } else {
    const bool dilate = a.method == MB200_DilateMorphology;
    float pix[CH];
#pragma unroll
    for (int c = 0; c < CH; ++c) pix[c] = dilate ? 0.0f : centre[c];
    for (int i = 0; i < a.ncells; ++i) {
      const Cell cell = a.cells[i];
      const float *p = win + (cell.dv * tw + cell.du) * CH;
#pragma unroll
      for (int c = 0; c < CH; ++c) {
        const float v = p[c];
        if (dilate) { if (v > pix[c]) pix[c] = v; }
        else { if (v < pix[c]) pix[c] = v; }
      }
    }
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      out[c] = pix[c];
      nchanged += fabs(static_cast<double>(pix[c]) - static_cast<double>(centre[c])) >= kEpsilon;
    }
  }
  if (a.changed != nullptr && nchanged != 0) atomicAdd(a.changed, static_cast<unsigned long long>(nchanged));
}

// Erode / dilate, tight version: CTA = 32x8 threads, each thread produces 4 output rows (y, y+8,
// y+16, y+24) of one column, so every active-cell offset (one broadcast LDS) is amortised over four
// LDS.128 + min/max groups.  fminf/fmaxf compile to FMNMX(3); a NaN sample never replaces the value, and
// erode keeps a NaN centre (the reference's `sample < pixel` never replaces it, morphology.c:2911) by
// selecting it at the output stage.  RGBA stages and stores whole float4 pixels: 16-byte aligned buffers only.
constexpr int kMmTile = 32, kMmRows = 4;
constexpr int kMmPitch = 64;          // fixed shared-memory pitch in pixels (kernel width <= 33)

template <int CH, bool DILATE>
__global__ void __launch_bounds__(256, 4) minmax2d_kernel(const Morph2dArgs a) {
  extern __shared__ __align__(16) float tile[];
  __shared__ int s_off[1024];
  const int tw = kMmTile + a.kw - 1, th = kMmTile + a.kh - 1;
  const int bx = blockIdx.x * kMmTile, by = blockIdx.y * kMmTile;
  const int tid = threadIdx.y * 32 + threadIdx.x;
  const int wmax = a.width - 1, hmax = a.height - 1;
  const int ncells = min(a.ncells, 1024);
  for (int i = tid; i < ncells; i += 256) s_off[i] = (a.cells[i].dv * kMmPitch + a.cells[i].du) * CH;
  // stage th rows x tw pixels: 64 threads per row, 4 rows per pass
  for (int ty = tid >> 6; ty < th; ty += 4) {
    const int tx = tid & 63;
    if (tx < tw) {
      const int sx = min(max(bx - a.ox + tx, 0), wmax);
      const int sy = min(max(by - a.oy + ty, 0), hmax);
      const float *g = a.src + (static_cast<size_t>(sy) * a.width + sx) * CH;
      float *d = tile + static_cast<size_t>(ty * kMmPitch + tx) * CH;
      if (CH == 4) *reinterpret_cast<float4 *>(d) = __ldg(reinterpret_cast<const float4 *>(g));
      else {
#pragma unroll
        for (int c = 0; c < CH; ++c) d[c] = __ldg(g + c);
      }
    }
  }
  __syncthreads();
  const int x = bx + threadIdx.x;
  const float *base = tile + (threadIdx.y * kMmPitch + threadIdx.x) * CH;   // window top-left of row 0
  constexpr int kRowStride = 8 * kMmPitch * CH;                             // rows handled: ty, ty+8, ...
  const int coff = (a.oy * kMmPitch + a.ox) * CH;
  float acc[kMmRows][CH], ctr[kMmRows][CH];
#pragma unroll
  for (int r = 0; r < kMmRows; ++r)
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      ctr[r][c] = base[r * kRowStride + coff + c];
      acc[r][c] = DILATE ? 0.0f : ctr[r][c];
    }
  auto fold = [&](const float *p) {
#pragma unroll
    for (int r = 0; r < kMmRows; ++r) {
      float v[CH];
      if (CH == 4) { const float4 t = *reinterpret_cast<const float4 *>(p + r * kRowStride); v[0] = t.x; v[1] = t.y; v[2] = t.z; v[CH - 1] = t.w; }
      else {
#pragma unroll
        for (int c = 0; c < CH; ++c) v[c] = p[r * kRowStride + c];
      }
#pragma unroll
      for (int c = 0; c < CH; ++c) acc[r][c] = DILATE ? fmaxf(acc[r][c], v[c]) : fminf(acc[r][c], v[c]);
    }
  };
  int i = 0;
  for (; i + 1 < ncells; i += 2) {          // two cells per trip: lets the compiler form 3-input min/max
    const float *p0 = base + s_off[i], *p1 = base + s_off[i + 1];
#pragma unroll
    for (int r = 0; r < kMmRows; ++r) {
      float v0[CH], v1[CH];
      if (CH == 4) {
        const float4 t0 = *reinterpret_cast<const float4 *>(p0 + r * kRowStride);
        const float4 t1 = *reinterpret_cast<const float4 *>(p1 + r * kRowStride);
        v0[0] = t0.x; v0[1] = t0.y; v0[2] = t0.z; v0[CH - 1] = t0.w;
        v1[0] = t1.x; v1[1] = t1.y; v1[2] = t1.z; v1[CH - 1] = t1.w;
      } else {
#pragma unroll
        for (int c = 0; c < CH; ++c) { v0[c] = p0[r * kRowStride + c]; v1[c] = p1[r * kRowStride + c]; }
      }
#pragma unroll
      for (int c = 0; c < CH; ++c)
        acc[r][c] = DILATE ? fmaxf(fmaxf(acc[r][c], v0[c]), v1[c]) : fminf(fminf(acc[r][c], v0[c]), v1[c]);
    }
  }
  if (i < ncells) fold(base + s_off[i]);
  unsigned nchanged = 0;
  if (x < a.width) {
#pragma unroll
    for (int r = 0; r < kMmRows; ++r) {
      const int y = by + threadIdx.y + 8 * r;
      if (y < a.height) {
        if (!DILATE) {
#pragma unroll
          for (int c = 0; c < CH; ++c)
            if (ctr[r][c] != ctr[r][c]) acc[r][c] = ctr[r][c];
        }
        float *o = a.dst + (static_cast<size_t>(y) * a.width + x) * CH;
        if (CH == 4) *reinterpret_cast<float4 *>(o) = make_float4(acc[r][0], acc[r][1], acc[r][2], acc[r][CH - 1]);
        else {
#pragma unroll
          for (int c = 0; c < CH; ++c) o[c] = acc[r][c];
        }
        if (a.changed != nullptr) {
#pragma unroll
          for (int c = 0; c < CH; ++c)
            nchanged += fabs(static_cast<double>(acc[r][c]) - static_cast<double>(ctr[r][c])) >= kEpsilon;
        }
      }
    }
  }
  if (a.changed != nullptr && nchanged != 0) atomicAdd(a.changed, static_cast<unsigned long long>(nchanged));
}

// ---- dense 2-D convolution, register tiled (SharpenImage 11x11, EdgeImage, EmbossImage, DoG / LoG, user kernels) -------------
// The generic kernel above spends, per kernel cell and output pixel, one tap load, one LDS.128 and four F2F conversions
// for four FMAs: it sits on the conversion (XU) and shared-memory pipes, not on FP64.  Here
//  * the source tile is converted to double and alpha-premultiplied ONCE while it is staged (v_c = A*p_c, v_alpha = A;
//    plain p_c without alpha), so the inner loop has no conversions;
//  * a thread owns R vertically adjacent outputs of one column: walking down a source column it loads each staged sample
//    once (2 x LDS.128, lanes = consecutive pixels: conflict free) and feeds up to R x CH FMAs, the taps K[v][u] coming
//    from shared memory as broadcast loads;
//  * accumulation in FP64 (column-major over the window instead of the reference's row-major order: the usual <= 1 ULP
//    argument of DESIGN.md section 4 applies), output stage as in morph2d_kernel (morphology.c:2962-2977, :3197).
// Cells must all be finite (NaN = "not in the neighbourhood" kernels keep the compacted-cell kernel).
// CTA = 32 x 8 threads, output tile 32 x (8*R); dynamic shared memory: taps + (8R+kh-1) x (32+kw-1) x CH doubles.
template <int CH, int R>
__global__ void __launch_bounds__(256) conv2d_dense_kernel(const Morph2dArgs a, const double *__restrict__ taps_window_order) {
  extern __shared__ __align__(16) double dsm[];
  constexpr bool kHasAlpha = (CH == 2 || CH == 4);
  const int tw = 32 + a.kw - 1, th = 8 * R + a.kh - 1;
  const int npix = tw * th;
  double *taps = dsm;                                        // kw*kh, window order
  double *tile = dsm + ((a.kw * a.kh + 1) & ~1);             // 16-byte aligned
  // RGBA: two planes of double2 -- (c0, c1) and (c2, alpha) -- so that consecutive lanes (= consecutive pixels) read
  // consecutive 16-byte words: conflict-free LDS.128 (one 32-byte pixel record per lane is a 2-way conflict: ncu showed
  // 41 % of the wavefronts conflicting and 6 short-scoreboard stalls per instruction).  Other layouts: pixel-interleaved.
  double *plane1 = tile + static_cast<size_t>(npix) * 2;
  const int tid = threadIdx.y * 32 + threadIdx.x;
  const int bx = blockIdx.x * 32, by = blockIdx.y * (8 * R);
  const int wmax = a.width - 1, hmax = a.height - 1;
  for (int i = tid; i < a.kw * a.kh; i += 256) taps[i] = taps_window_order[i];
  for (int p = tid; p < npix; p += 256) {
    const int ty = p / tw, tx = p - ty * tw;
    const int sx = min(max(bx - a.ox + tx, 0), wmax), sy = min(max(by - a.oy + ty, 0), hmax);
    const float *g = a.src + (static_cast<size_t>(sy) * a.width + sx) * CH;
    double v[CH];
    if (CH == 4) {
      const float4 t = __ldg(reinterpret_cast<const float4 *>(g));
      v[0] = t.x; v[1] = t.y; v[2] = t.z; v[CH - 1] = t.w;
    } else {
#pragma unroll
      for (int c = 0; c < CH; ++c) v[c] = __ldg(g + c);
    }
    if (kHasAlpha) {
#pragma unroll
      for (int c = 0; c < CH - 1; ++c) v[c] *= v[CH - 1];
    }
    if (CH == 4) {
      reinterpret_cast<double2 *>(tile)[p] = make_double2(v[0], v[1]);
      reinterpret_cast<double2 *>(plane1)[p] = make_double2(v[2], v[CH - 1]);
    } else if (CH == 2) {
      reinterpret_cast<double2 *>(tile)[p] = make_double2(v[0], v[CH - 1]);
    } else {
#pragma unroll
      for (int c = 0; c < CH; ++c) tile[static_cast<size_t>(p) * CH + c] = v[c];
    }
  }
  __syncthreads();
  double acc[R][CH];
#pragma unroll
  for (int r = 0; r < R; ++r)
#pragma unroll
    for (int c = 0; c < CH; ++c) acc[r][c] = 0.0;
  const int y0 = threadIdx.y * R;                              // first of this thread's R output rows (tile coordinates)
  const int span = R + a.kh - 1;                               // source rows that touch them
  for (int u = 0; u < a.kw; ++u) {
    const int p0 = y0 * tw + threadIdx.x + u;                  // first sample of this source column
    const double *kcol = taps + u;
    // k[r] = K[yy - r][u]: the tap the sample of source row yy has for output r; one new tap per row, the rest shifts
    double k[R];
#pragma unroll
    for (int r = 0; r < R; ++r) k[r] = 0.0;
    for (int yy = 0; yy < span; ++yy) {
#pragma unroll
      for (int r = R - 1; r > 0; --r) k[r] = k[r - 1];
      k[0] = yy < a.kh ? kcol[yy * a.kw] : 0.0;
      const int p = p0 + yy * tw;
      double v[CH];
      if (CH == 4) {
        const double2 lo = reinterpret_cast<const double2 *>(tile)[p], hi = reinterpret_cast<const double2 *>(plane1)[p];
        v[0] = lo.x; v[1] = lo.y; v[2] = hi.x; v[CH - 1] = hi.y;
      } else if (CH == 2) {
        const double2 lo = reinterpret_cast<const double2 *>(tile)[p];
        v[0] = lo.x; v[CH - 1] = lo.y;
      } else {
#pragma unroll
        for (int c = 0; c < CH; ++c) v[c] = tile[static_cast<size_t>(p) * CH + c];
      }
      // rows outside an output's window carry k = 0 but must not contribute 0 * (inf | NaN): predicate on the row range
#pragma unroll
      for (int r = 0; r < R; ++r) {
        if (yy >= r && yy - r < a.kh) {
#pragma unroll
          for (int c = 0; c < CH; ++c) acc[r][c] = fma(k[r], v[c], acc[r][c]);
        }
      }
    }
  }
  const int x = bx + threadIdx.x;
  unsigned nchanged = 0;
  if (x < a.width) {
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int y = by + y0 + r;
      if (y >= a.height) break;
      float *out = a.dst + (static_cast<size_t>(y) * a.width + x) * CH;
      const float *centre = a.src + (static_cast<size_t>(y) * a.width + x) * CH;
      float o[CH];
      if (kHasAlpha) {
        const double g = precise_reciprocal_gamma(kQuantumScale * acc[r][CH - 1]) * a.gamma_scale;
#pragma unroll
        for (int c = 0; c < CH - 1; ++c) {
          const double pixel = fma(kQuantumScale, acc[r][c], a.bias);
          o[c] = static_cast<float>(g * pixel);
          if (a.changed != nullptr) nchanged += fabs(pixel - static_cast<double>(__ldg(centre + c))) >= kEpsilon;
        }
        const double pixel = a.bias + acc[r][CH - 1];
        o[CH - 1] = static_cast<float>(a.gamma_scale * pixel);
        if (a.changed != nullptr) nchanged += fabs(pixel - static_cast<double>(__ldg(centre + CH - 1))) >= kEpsilon;
      } else {
#pragma unroll
        for (int c = 0; c < CH; ++c) {
          const double pixel = a.bias + acc[r][c];
          o[c] = static_cast<float>(a.gamma_scale * pixel);
          if (a.changed != nullptr) nchanged += fabs(pixel - static_cast<double>(__ldg(centre + c))) >= kEpsilon;
        }
      }
      if (CH == 4) *reinterpret_cast<float4 *>(out) = make_float4(o[0], o[1], o[2], o[CH - 1]);
      else {
#pragma unroll
        for (int c = 0; c < CH; ++c) out[c] = o[c];
      }
    }
  }
  if (a.changed != nullptr && nchanged != 0) atomicAdd(a.changed, static_cast<unsigned long long>(nchanged));
}

}  // namespace

int launch_morph2d(const float *src, float *dst, size_t width, size_t height, int channels, int method,
                   const double *kernel_window_order, int kw, int kh, int ox, int oy, double bias,
                   double gamma_scale, unsigned long long *d_changed, void *stream) {
  if (width == 0 || height == 0 || channels < 1 || channels > 4 || kw < 1 || kh < 1)
    return fail(MB200_EINVAL, "morph2d: bad geometry");
  if (width > 0x3fffffffull || height > 0x3fffffffull) return fail(MB200_EINVAL, "morph2d: image too large");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // compact the active cells (NaN = not in the neighbourhood; erode/dilate thresholds)
  const int total = kw * kh;
  Cell *host = static_cast<Cell *>(malloc(sizeof(Cell) * static_cast<size_t>(total)));
  if (!host) return fail(MB200_ENOMEM, "morph2d: host alloc");
  int n = 0;
  for (int v = 0; v < kh; ++v)
    for (int u = 0; u < kw; ++u) {
      const double k = kernel_window_order[v * kw + u];
      if (k != k) continue;
      if (method == MB200_ErodeMorphology && !(k >= 0.5)) continue;
      if (method == MB200_DilateMorphology && !(k > 0.5)) continue;
      if ((method == MB200_ErodeIntensityMorphology || method == MB200_DilateIntensityMorphology) && !(k >= 0.5)) continue;
      double kept = k;
      if (method == MB200_HitAndMissMorphology || method == MB200_ThinningMorphology || method == MB200_ThickenMorphology) {
        if (k > 0.7) kept = 1.0;             // foreground
        else if (k < 0.3) kept = 0.0;        // background
        else continue;                       // don't care
      }
      host[n].du = static_cast<short>(u); host[n].dv = static_cast<short>(v); host[n].pad = 0.f; host[n].k = kept;
      ++n;
    }
  const bool aligned = ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0;
  if (method == MB200_ConvolveMorphology && n == total && aligned) {
    // every cell is part of the neighbourhood: register-tiled dense kernel (R = 8 or 4 output rows per thread while the
    // staged tile of doubles leaves room for two CTAs per SM, else 2 while it fits at all).  The conv2d_rows option
    // forces an R whose tile fits.
    free(host);
    auto tile_bytes = [&](int R) {
      return (static_cast<size_t>((total + 1) & ~1) + static_cast<size_t>(32 + kw - 1) * (8 * R + kh - 1) * channels) * sizeof(double);
    };
    const int forced = tuning_knobs().conv2d_rows;
    int R = tile_bytes(8) <= 110 * 1024 ? 8 : tile_bytes(4) <= 110 * 1024 ? 4 : (tile_bytes(2) <= 200 * 1024 ? 2 : 0);
    if (forced != 0 && tile_bytes(forced) <= 200 * 1024) R = forced;
    if (R != 0) {
      double *d_taps = nullptr;
      cudaError_t e = cudaMallocAsync(reinterpret_cast<void **>(&d_taps), sizeof(double) * static_cast<size_t>(total), temp_pool(), s);
      if (e != cudaSuccess) return cuda_fail(e, "conv2d: tap table alloc");
      e = cudaMemcpyAsync(d_taps, kernel_window_order, sizeof(double) * static_cast<size_t>(total), cudaMemcpyHostToDevice, s);
      if (e != cudaSuccess) { cudaFreeAsync(d_taps, s); return cuda_fail(e, "conv2d: tap upload"); }
      Morph2dArgs a{};
      a.src = src; a.dst = dst;
      a.width = static_cast<int>(width); a.height = static_cast<int>(height); a.channels = channels;
      a.ox = ox; a.oy = oy; a.kw = kw; a.kh = kh; a.ncells = n;
      a.bias = bias; a.gamma_scale = gamma_scale; a.method = method; a.changed = d_changed;
      const size_t smem = tile_bytes(R);
      dim3 grid((a.width + 31) / 32, (a.height + 8 * R - 1) / (8 * R)), block(32, 8);
#define MB200_DENSE(CH, RR)                                                                                         \
      do {                                                                                                          \
        cudaFuncSetAttribute(conv2d_dense_kernel<CH, RR>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024); \
        conv2d_dense_kernel<CH, RR><<<grid, block, smem, s>>>(a, d_taps);                                           \
      } while (0)
      switch (channels * 10 + R) {
        case 18: MB200_DENSE(1, 8); break;
        case 14: MB200_DENSE(1, 4); break;
        case 12: MB200_DENSE(1, 2); break;
        case 28: MB200_DENSE(2, 8); break;
        case 24: MB200_DENSE(2, 4); break;
        case 22: MB200_DENSE(2, 2); break;
        case 38: MB200_DENSE(3, 8); break;
        case 34: MB200_DENSE(3, 4); break;
        case 32: MB200_DENSE(3, 2); break;
        case 48: MB200_DENSE(4, 8); break;
        case 44: MB200_DENSE(4, 4); break;
        default: MB200_DENSE(4, 2); break;
      }
#undef MB200_DENSE
      count_launch();
      count_family(R == 8 ? kConv2dDenseR8 : R == 4 ? kConv2dDenseR4 : kConv2dDenseR2);
      e = cudaGetLastError();
      cudaFreeAsync(d_taps, s);
      if (e != cudaSuccess) return cuda_fail(e, "conv2d launch");
      return MB200_OK;
    }
    host = static_cast<Cell *>(malloc(sizeof(Cell) * static_cast<size_t>(total)));      // too large: the compacted-cell kernel
    if (!host) return fail(MB200_ENOMEM, "morph2d: host alloc");
    n = 0;
    for (int v = 0; v < kh; ++v)
      for (int u = 0; u < kw; ++u) {
        host[n].du = static_cast<short>(u); host[n].dv = static_cast<short>(v); host[n].pad = 0.f;
        host[n].k = kernel_window_order[v * kw + u];
        ++n;
      }
  }
  void *d_cells = nullptr;
  cudaError_t e = cudaMallocAsync(&d_cells, sizeof(Cell) * static_cast<size_t>(total), temp_pool(), s);   // stream-ordered: re-entrant
  if (e != cudaSuccess) { free(host); return cuda_fail(e, "morph2d: tap table alloc"); }
  e = cudaMemcpyAsync(d_cells, host, sizeof(Cell) * static_cast<size_t>(n), cudaMemcpyHostToDevice, s);
  free(host);   // pageable source: the copy has been staged when the call returns
  if (e != cudaSuccess) { cudaFreeAsync(d_cells, s); return cuda_fail(e, "morph2d: tap upload"); }

  Morph2dArgs a{};
  a.src = src; a.dst = dst;
  a.width = static_cast<int>(width); a.height = static_cast<int>(height); a.channels = channels;
  a.ox = ox; a.oy = oy; a.kw = kw; a.kh = kh; a.ncells = n;
  a.cells = static_cast<const Cell *>(d_cells);
  a.bias = bias; a.gamma_scale = gamma_scale; a.method = method; a.changed = d_changed;
  if ((method == MB200_ErodeMorphology || method == MB200_DilateMorphology) && n <= 1024 && kw <= kMmPitch - kMmTile + 1 &&
      (channels != 4 || aligned)) {         // RGBA moves float4 pixels: unaligned buffers take morph2d_kernel below
    const int th = kMmTile + kh - 1;
    const size_t msmem = static_cast<size_t>(kMmPitch) * th * channels * sizeof(float);
    if (msmem <= 160 * 1024) {
      dim3 mgrid((a.width + kMmTile - 1) / kMmTile, (a.height + kMmTile - 1) / kMmTile), mblock(32, 8);
      const bool dil = method == MB200_DilateMorphology;
#define MB200_MM(CH)                                                                                   \
      do {                                                                                             \
        if (dil) {                                                                                     \
          cudaFuncSetAttribute(minmax2d_kernel<CH, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);  \
          minmax2d_kernel<CH, true><<<mgrid, mblock, msmem, s>>>(a);                            \
        } else {                                                                                       \
          cudaFuncSetAttribute(minmax2d_kernel<CH, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024); \
          minmax2d_kernel<CH, false><<<mgrid, mblock, msmem, s>>>(a);                           \
        }                                                                                              \
      } while (0)
      switch (channels) {
        case 1: MB200_MM(1); break;
        case 2: MB200_MM(2); break;
        case 3: MB200_MM(3); break;
        default: MB200_MM(4); break;
      }
#undef MB200_MM
      count_launch();
      count_family(kMinmax2d);
      e = cudaGetLastError();
      cudaFreeAsync(d_cells, s);
      if (e != cudaSuccess) return cuda_fail(e, "minmax2d launch");
      return MB200_OK;
    }
  }
  const size_t smem = static_cast<size_t>(kTileW + kw - 1) * (kTileH + kh - 1) * channels * sizeof(float);
  if (smem > 200 * 1024) { cudaFreeAsync(d_cells, s); return fail(MB200_EUNSUPPORTED, "morph2d: %dx%d kernel needs %zu bytes of shared memory", kw, kh, smem); }
  dim3 grid((a.width + kTileW - 1) / kTileW, (a.height + kTileH - 1) / kTileH), block(kTileW, kTileH);
#define MB200_LAUNCH(CH)                                                                         \
  do {                                                                                           \
    cudaFuncSetAttribute(morph2d_kernel<CH>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024); \
    morph2d_kernel<CH><<<grid, block, smem, s>>>(a);                                             \
  } while (0)
  switch (channels) {
    case 1: MB200_LAUNCH(1); break;
    case 2: MB200_LAUNCH(2); break;
    case 3: MB200_LAUNCH(3); break;
    default: MB200_LAUNCH(4); break;
  }
#undef MB200_LAUNCH
  count_launch();
  count_family(kMorph2d);
  e = cudaGetLastError();
  cudaFreeAsync(d_cells, s);
  if (e != cudaSuccess) return cuda_fail(e, "morph2d launch");
  return MB200_OK;
}

}  // namespace mb200
