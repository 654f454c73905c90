// hooks.cu -- the last three image-returning accelerate hooks (accelerate-private.h:36-48):
//   DespeckleImage       MagickCore/effect.c:1308-1480 (Hull :1211-1306)
//   LocalContrastImage   MagickCore/effect.c:2013-2275
//   WaveletDenoiseImage  MagickCore/visual-effects.c:3515-3782 (HatTransform :3478-3513)
// All three are bit exact: every operation is the reference's IEEE operation in the reference's order (__fadd_rn /
// __fmul_rn / __dadd_rn ... so nothing is contracted).  DESIGN §5.7 gives launch counts and bytes / FMAs per pixel.
// 8192^2 RGBA on one H100 80GB HBM3 at a 400 W power limit: Despeckle 20.2 ms (12.7 % of the 3.35 TB/s data-sheet HBM
// bandwidth), LocalContrast 10x12.5 12.2 ms (23.6 % of the probed FP64 FMA rate), WaveletDenoise 10 % 11.7 ms (41 % of
// HBM).
#include "launch.cuh"

#include <cuda_runtime.h>

#include <cmath>

namespace mb200 {
namespace {

// ------------------------------------------------------------------------------------------------------ DespeckleImage
// The reference runs 16 Hulls per channel over a zero-bordered plane, each Hull two full-plane sweeps.  One launch here
// runs the four Hulls of one direction (X[k], Y[k]) = 8 sweeps on a 32x32 tile held in shared memory with an 8-pixel halo:
// every sweep reads neighbours one step along the direction, so after 8 sweeps the tile's interior is exact.  Cells
// outside the image are the reference's zero border and stay 0; cells whose neighbour lies outside the halo region are
// not updated (they are outside the exact region by then).  All channels of a pixel go through the same launch.
constexpr int kDsTile = 32, kDsHalo = 8, kDsRegion = kDsTile + 2 * kDsHalo, kDsCells = kDsRegion * kDsRegion;
constexpr int kDsThreads = 256, kDsPerThread = (kDsCells + kDsThreads - 1) / kDsThreads;

template <int CH>
__global__ void __launch_bounds__(kDsThreads, 2) despeckle_kernel(const float *__restrict__ src, float *__restrict__ dst,
                                                               int w, int h, int dx, int dy) {
  __shared__ float plane[CH][kDsCells];
  const int x0 = static_cast<int>(blockIdx.x) * kDsTile - kDsHalo, y0 = static_cast<int>(blockIdx.y) * kDsTile - kDsHalo;
  const int tid = static_cast<int>(threadIdx.x);
  // coalesced load of the region: consecutive threads take consecutive floats of a region row
  for (int e = tid; e < kDsCells * CH; e += kDsThreads) {
    const int ly = e / (kDsRegion * CH), r = e - ly * kDsRegion * CH, lx = r / CH, c = r - lx * CH;
    const int gx = x0 + lx, gy = y0 + ly;
    float v = 0.0f;
    if (gx >= 0 && gx < w && gy >= 0 && gy < h) v = src[(static_cast<size_t>(gy) * w + gx) * CH + c];
    plane[c][ly * kDsRegion + lx] = v;
  }
  // this thread's cells: which are in the image, and whether both neighbours along the direction are in the region
  unsigned live = 0;                                          // bit j: cell j of this thread is updated
#pragma unroll
  for (int j = 0; j < kDsPerThread; ++j) {
    const int cell = tid + j * kDsThreads, lx = cell % kDsRegion, ly = cell / kDsRegion;
    const int gx = x0 + lx, gy = y0 + ly;
    const bool updated = cell < kDsCells && gx >= 0 && gx < w && gy >= 0 && gy < h && lx - dx >= 0 &&
                         lx - dx < kDsRegion && lx + dx >= 0 && lx + dx < kDsRegion && ly - dy >= 0 && ly + dy < kDsRegion;
    live |= static_cast<unsigned>(updated) << j;
  }
  __syncthreads();
  float next[kDsPerThread][CH];
  // Hull(x_offset, y_offset, polarity): the four calls of effect.c:1438-1441
#pragma unroll 1
  for (int hull = 0; hull < 4; ++hull) {
    const int sign = (hull == 1 || hull == 2) ? -1 : 1, polarity = hull < 2 ? 1 : -1;
    const int off = sign * (dy * kDsRegion + dx);
    // f -> g: v + 257 where r = f[i + off] >= v + 514 (polarity > 0), mirrored for polarity < 0 (:1248-1265)
#pragma unroll
    for (int j = 0; j < kDsPerThread; ++j) {
      const int cell = tid + j * kDsThreads;
#pragma unroll
      for (int c = 0; c < CH; ++c) {
        if (!(live >> j & 1u)) continue;
        const float p = plane[c][cell], r = plane[c][cell + off];
        double v = static_cast<double>(p);
        if (polarity > 0) { if (static_cast<double>(r) >= __dadd_rn(v, 514.0)) v = __dadd_rn(v, 257.0); }
        else if (static_cast<double>(r) <= __dsub_rn(v, 514.0)) v = __dsub_rn(v, 257.0);
        next[j][c] = __double2float_rn(v);
      }
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < kDsPerThread; ++j)
#pragma unroll
      for (int c = 0; c < CH; ++c)
        if (live >> j & 1u) plane[c][tid + j * kDsThreads] = next[j][c];
    __syncthreads();
    // g -> f: s = g[i - off] beyond v +/- 514 AND r = g[i + off] strictly beyond v (:1285-1304)
#pragma unroll
    for (int j = 0; j < kDsPerThread; ++j) {
      const int cell = tid + j * kDsThreads;
#pragma unroll
      for (int c = 0; c < CH; ++c) {
        if (!(live >> j & 1u)) continue;
        const float q = plane[c][cell], s = plane[c][cell - off], r = plane[c][cell + off];
        double v = static_cast<double>(q);
        if (polarity > 0) {
          if (static_cast<double>(s) >= __dadd_rn(v, 514.0) && static_cast<double>(r) > v) v = __dadd_rn(v, 257.0);
        } else if (static_cast<double>(s) <= __dsub_rn(v, 514.0) && static_cast<double>(r) < v) {
          v = __dsub_rn(v, 257.0);
        }
        next[j][c] = __double2float_rn(v);
      }
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < kDsPerThread; ++j)
#pragma unroll
      for (int c = 0; c < CH; ++c)
        if (live >> j & 1u) plane[c][tid + j * kDsThreads] = next[j][c];
    __syncthreads();
  }
  // the tile's interior
  for (int e = tid; e < kDsTile * kDsTile * CH; e += kDsThreads) {
    const int ty = e / (kDsTile * CH), r = e - ty * kDsTile * CH, tx = r / CH, c = r - tx * CH;
    const int gx = x0 + kDsHalo + tx, gy = y0 + kDsHalo + ty;
    if (gx < w && gy < h) dst[(static_cast<size_t>(gy) * w + gx) * CH + c] = plane[c][(ty + kDsHalo) * kDsRegion + tx + kDsHalo];
  }
}

// ------------------------------------------------------------------------------------------------- LocalContrastImage
// (float) GetPixelLuma (pixel-accessor.h:304): unfused double products and sums; gray images alias R, G and B to the one
// sample (pixel.c:6149-6155).
template <int CH>
__device__ __forceinline__ double pixel_luma(const float *p) {
  const double r = static_cast<double>(p[0]);
  const double g = CH >= 3 ? static_cast<double>(p[CH >= 3 ? 1 : 0]) : r, b = CH >= 3 ? static_cast<double>(p[CH >= 3 ? 2 : 0]) : r;
  return __dadd_rn(__dadd_rn(__dmul_rn(0.212656, r), __dmul_rn(0.715158, g)), __dmul_rn(0.072186, b));
}

template <int CH>
__global__ void luma_kernel(const float *__restrict__ src, float *__restrict__ luma, size_t n) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) luma[i] = __double2float_rn(pixel_luma<CH>(src + i * CH));
}

// Both passes sum the reference's taps k = 0 .. 2*width-2 of the line in tap order: weight k+1 for k < width, then
// 2*width+1-k (width+1 down to 3; the reference's second loop starts at i = width+1 and never reaches the last two taps
// of a symmetric triangle).  weight * sample is exact in double (weight < 2^29), so an FMA into the running sum equals
// the reference's separate multiply and add.  The line segment a block needs is staged in shared memory as double,
// CHUNK taps at a time.
constexpr int kLcChunk = 64;
constexpr int kLcVRows = 64, kLcVThreadsY = 8;           // vertical pass: 32 columns x 64 rows per block
constexpr int kLcHOut = 4, kLcHThreads = 256;            // horizontal pass: 1024 outputs of one row per block

__device__ __forceinline__ double lc_weight(int k, int width) {
  return static_cast<double>(k < width ? k + 1 : 2 * width + 1 - k);
}

// Vertical pass (:2107-2173): edge-clamped rows (the default virtual pixels), sum / totalWeight rounded to float.  The
// intermediate is unpadded: the horizontal pass reads the reference's mirrored padding through mirror indices.
__global__ void __launch_bounds__(32 * kLcVThreadsY) local_contrast_v_kernel(const float *__restrict__ luma,
                                                                              float *__restrict__ inter, int w, int h,
                                                                              int width, double total) {
  __shared__ double tile[kLcVRows + kLcChunk][32];
  const int tx = static_cast<int>(threadIdx.x), ty = static_cast<int>(threadIdx.y);
  const int x = static_cast<int>(blockIdx.x) * 32 + tx, y0 = static_cast<int>(blockIdx.y) * kLcVRows;
  const int xs = x < w ? x : w - 1;
  const int ntaps = width > 0 ? 2 * width - 1 : 0;
  double sum[kLcVRows / kLcVThreadsY];
#pragma unroll
  for (int j = 0; j < kLcVRows / kLcVThreadsY; ++j) sum[j] = 0.0;
  for (int kb = 0; kb < ntaps; kb += kLcChunk) {
    const int nk = ntaps - kb < kLcChunk ? ntaps - kb : kLcChunk;
    __syncthreads();
    for (int r = ty; r < kLcVRows + nk - 1; r += kLcVThreadsY) {
      int yy = y0 + kb - width + r;
      yy = yy < 0 ? 0 : (yy >= h ? h - 1 : yy);
      tile[r][tx] = static_cast<double>(luma[static_cast<size_t>(yy) * w + xs]);
    }
    __syncthreads();
    for (int k = 0; k < nk; ++k) {
      const double wt = lc_weight(kb + k, width);
#pragma unroll
      for (int j = 0; j < kLcVRows / kLcVThreadsY; ++j) sum[j] = fma(wt, tile[ty + j * kLcVThreadsY + k][tx], sum[j]);
    }
  }
  if (x >= w) return;
#pragma unroll
  for (int j = 0; j < kLcVRows / kLcVThreadsY; ++j) {
    const int y = y0 + ty + j * kLcVThreadsY;
    if (y < h) inter[static_cast<size_t>(y) * w + x] = __double2float_rn(__ddiv_rn(sum[j], total));
  }
}

// Horizontal pass (:2186-2266) with the apply step: the padded column j of the reference's intermediate holds column
// -j (j < 0) or 2*(w-1)-j (j > w-1), which the vertical pass wrote for width <= w-1.  sum / totalWeight stays double;
// mult = (src + (src - blur) * strength/100) / src scales R, G, B (ClampToQuantum is a bare cast in HDRI: a luma of 0
// gives NaN as in the reference); alpha is copied.
template <int CH>
__global__ void __launch_bounds__(kLcHThreads) local_contrast_h_kernel(const float *__restrict__ src,
                                                                      const float *__restrict__ luma,
                                                                      const float *__restrict__ inter,
                                                                      float *__restrict__ dst, int w, int width,
                                                                      double total, double strength100) {
  constexpr int kOut = kLcHThreads * kLcHOut;
  __shared__ double seg[kOut + kLcChunk];
  const int tid = static_cast<int>(threadIdx.x), y = static_cast<int>(blockIdx.y);
  const int x0 = static_cast<int>(blockIdx.x) * kOut;
  const float *row = inter + static_cast<size_t>(y) * w;
  const int ntaps = width > 0 ? 2 * width - 1 : 0;
  double sum[kLcHOut];
#pragma unroll
  for (int j = 0; j < kLcHOut; ++j) sum[j] = 0.0;
  for (int kb = 0; kb < ntaps; kb += kLcChunk) {
    const int nk = ntaps - kb < kLcChunk ? ntaps - kb : kLcChunk;
    __syncthreads();
    for (int t = tid; t < kOut + nk - 1; t += kLcHThreads) {
      int j = x0 + kb - width + t;
      j = j < 0 ? -j : (j > w - 1 ? 2 * (w - 1) - j : j);
      j = j < 0 ? 0 : (j > w - 1 ? w - 1 : j);            // only for slots no output of this block reads
      seg[t] = static_cast<double>(row[j]);
    }
    __syncthreads();
    for (int k = 0; k < nk; ++k) {
      const double wt = lc_weight(kb + k, width);
#pragma unroll
      for (int j = 0; j < kLcHOut; ++j) sum[j] = fma(wt, seg[tid + j * kLcHThreads + k], sum[j]);
    }
  }
#pragma unroll
  for (int j = 0; j < kLcHOut; ++j) {
    const int x = x0 + tid + j * kLcHThreads;
    if (x >= w) continue;
    const size_t i = static_cast<size_t>(y) * w + x;
    const double srcval = static_cast<double>(luma[i]);
    double mult = __dmul_rn(__dsub_rn(srcval, __ddiv_rn(sum[j], total)), strength100);
    mult = __ddiv_rn(__dadd_rn(srcval, mult), srcval);
    const float *p = src + i * CH;
    float *q = dst + i * CH;
    q[0] = __double2float_rn(__dmul_rn(static_cast<double>(p[0]), mult));
    if (CH >= 3) {
      q[CH >= 3 ? 1 : 0] = __double2float_rn(__dmul_rn(static_cast<double>(p[CH >= 3 ? 1 : 0]), mult));
      q[CH >= 3 ? 2 : 0] = __double2float_rn(__dmul_rn(static_cast<double>(p[CH >= 3 ? 2 : 0]), mult));
    }
    if (CH == 2 || CH == 4) q[CH - 1] = p[CH - 1];
  }
}

// ---------------------------------------------------------------------------------------------- WaveletDenoiseImage
// HatTransform (:3478-3513) at index i of a line of n samples, step s (n >= 2s): each end reflects about its end sample;
// at the right end the reflected index starts at n-2 and walks back.  Float arithmetic evaluated as written.
template <typename At>
__device__ __forceinline__ float hat(const At &at, int i, int n, int s) {
  const float p = at(i);
  if (i < s) return __fmul_rn(0.25f, __fadd_rn(__fadd_rn(__fadd_rn(p, p), at(s - i)), at(s + i)));
  if (i < n - s) return __fmul_rn(0.25f, __fadd_rn(__fadd_rn(__fmul_rn(2.0f, p), at(i - s)), at(i + s)));
  return __fmul_rn(0.25f, __fadd_rn(__fadd_rn(__fadd_rn(p, p), at(i - s)), at(n - 2 - (i - (n - s)))));
}

// One level for one colour channel (blockIdx.z) in one launch: the row hat and the column hat of the high-pass input
// (the channel of `src` at level 0, else the previous level's low-pass plane `in`), evaluated per output from the
// nine input samples it depends on, so the row-filtered plane never goes to memory.  The threshold / accumulate step
// follows: detail = high - low, thresholded against +/- magnitude (:3706-3719), is plane 0 at level 0 and is added to
// it afterwards.  The last level writes (double) plane 0 + (double) low-pass, cast to float (:3754-3756), into dst
// (and copies alpha).
struct WaveletLevel {
  int level, scale;
  double magnitude;
  float adjust, softness;      // (float) (magnitude - softness*magnitude), (float) softness
};

__global__ void __launch_bounds__(256) wavelet_level_kernel(const float *__restrict__ src, float *__restrict__ dst, int ch,
                                                            const float *__restrict__ in, float *__restrict__ out,
                                                            float *__restrict__ acc, int w, int h, WaveletLevel lv) {
  const int x = static_cast<int>(blockIdx.x * blockDim.x + threadIdx.x), y = static_cast<int>(blockIdx.y * blockDim.y + threadIdx.y);
  if (x >= w || y >= h) return;
  const int c = static_cast<int>(blockIdx.z);
  const size_t n = static_cast<size_t>(w) * h, plane = static_cast<size_t>(c) * n;
  const int s = lv.scale;
  float low;
  if (lv.level == 0) {
    const auto row_hat = [&](int r) {
      const float *line = src + static_cast<size_t>(r) * w * ch + c;
      return hat([&](int i) { return line[static_cast<size_t>(i) * ch]; }, x, w, s);
    };
    low = hat(row_hat, y, h, s);
  } else {
    const auto row_hat = [&](int r) {
      const float *line = in + plane + static_cast<size_t>(r) * w;
      return hat([&](int i) { return line[i]; }, x, w, s);
    };
    low = hat(row_hat, y, h, s);
  }
  const size_t i = static_cast<size_t>(y) * w + x;
  const float high = lv.level == 0 ? src[i * ch + c] : in[plane + i];
  float detail = __fsub_rn(high, low);
  if (static_cast<double>(detail) < -lv.magnitude) detail = __fadd_rn(detail, lv.adjust);
  else if (static_cast<double>(detail) > lv.magnitude) detail = __fsub_rn(detail, lv.adjust);
  else detail = __fmul_rn(detail, lv.softness);
  const float a = lv.level == 0 ? detail : __fadd_rn(acc[plane + i], detail);
  if (lv.level < 4) {
    acc[plane + i] = a;
    out[plane + i] = low;
    return;
  }
  dst[i * ch + c] = __double2float_rn(__dadd_rn(static_cast<double>(a), static_cast<double>(low)));
  if (c == 0 && (ch == 2 || ch == 4)) dst[i * ch + ch - 1] = src[i * ch + ch - 1];
}

int check_hook_image(const float *src, float *dst, size_t w, size_t h, int channels, const char *what) {
  if (!src || !dst || w == 0 || h == 0 || channels < 1 || channels > 4) return fail(MB200_EINVAL, "%s: bad arguments", what);
  if (w > 0x3fffffffull || h > 0x3fffffffull || w * h > (1ull << 40)) return fail(MB200_EUNSUPPORTED, "%s: image too large", what);
  return MB200_OK;
}

}  // namespace

int launch_despeckle(const float *src, float *dst, float *tmp, size_t w, size_t h, int channels, void *stream) {
  int rc = check_hook_image(src, dst, w, h, channels, "despeckle");
  if (rc) return rc;
  if ((h + kDsTile - 1) / kDsTile > 65535) return fail(MB200_EUNSUPPORTED, "despeckle: more than %d rows", 65535 * kDsTile);
  static const int X[4] = {0, 1, 1, -1}, Y[4] = {1, 0, 1, 1};
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const dim3 grid(static_cast<unsigned>((w + kDsTile - 1) / kDsTile), static_cast<unsigned>((h + kDsTile - 1) / kDsTile));
  const int iw = static_cast<int>(w), ih = static_cast<int>(h);
  // src -> tmp -> dst -> tmp -> dst: a launch never reads the buffer it writes (tiles read their neighbours' pixels)
  const float *in[4] = {src, tmp, dst, tmp};
  float *out[4] = {tmp, dst, tmp, dst};
  return with_channels(channels, "despeckle", [&](auto ch) -> int {
    for (int k = 0; k < 4; ++k) {
      despeckle_kernel<ch()><<<grid, kDsThreads, 0, s>>>(in[k], out[k], iw, ih, X[k], Y[k]);
      const int rc = launch_status("despeckle launch");
      if (rc) return rc;
    }
    return MB200_OK;
  });
}

long local_contrast_width(size_t w, size_t h, double radius) {
  // effect.c:2067-2068: (ssize_t) scanLineSize*0.002*fabs(radius)
  const double width = static_cast<double>(static_cast<long>(w > h ? w : h)) * 0.002 * std::fabs(radius);
  if (!(width < 1.0e15)) return -1;                        // NaN / inf / absurd radius
  return static_cast<long>(width);
}

int local_contrast_supported(size_t w, size_t h, double radius) {
  const long width = local_contrast_width(w, h, radius);
  if (width < 0) return fail(MB200_EUNSUPPORTED, "local contrast: radius %g", radius);
  // the mirror of :2166-2170 fills width <= columns - 1 padding columns on the left; a wider kernel reads unwritten memory
  if (width > 0 && width > static_cast<long>(w) - 1)
    return fail(MB200_EUNSUPPORTED, "local contrast: kernel width %ld exceeds columns - 1 = %zu", width, w - 1);
  if (width + 1 >= (1L << 29)) return fail(MB200_EUNSUPPORTED, "local contrast: kernel width %ld", width);
  return MB200_OK;
}

int launch_local_contrast(const float *src, float *dst, float *luma, float *inter, size_t w, size_t h, int channels,
                          double radius, double strength, void *stream) {
  int rc = check_hook_image(src, dst, w, h, channels, "local contrast");
  if (!rc) rc = local_contrast_supported(w, h, radius);
  if (rc) return rc;
  if ((h + kLcVRows - 1) / kLcVRows > 65535 || h > 65535)
    return fail(MB200_EUNSUPPORTED, "local contrast: more than 65535 rows");
  const int width = static_cast<int>(local_contrast_width(w, h, radius));
  const double total = static_cast<double>(static_cast<float>(static_cast<long>(width + 1) * (width + 1)));   // :2094
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t n = w * h;
  const unsigned lblocks = static_cast<unsigned>((n + 255) / 256);
  const int iw = static_cast<int>(w), ih = static_cast<int>(h);
  const dim3 vgrid(static_cast<unsigned>((w + 31) / 32), static_cast<unsigned>((h + kLcVRows - 1) / kLcVRows));
  const dim3 hgrid(static_cast<unsigned>((w + kLcHThreads * kLcHOut - 1) / (kLcHThreads * kLcHOut)), static_cast<unsigned>(h));
  const double strength100 = strength / 100.0;
  return with_channels(channels, "local contrast", [&](auto ch) {
    luma_kernel<ch()><<<lblocks, 256, 0, s>>>(src, luma, n);
    local_contrast_v_kernel<<<vgrid, dim3(32, kLcVThreadsY), 0, s>>>(luma, inter, iw, ih, width, total);
    local_contrast_h_kernel<ch()><<<hgrid, kLcHThreads, 0, s>>>(src, luma, inter, dst, iw, width, total, strength100);
    return launch_status("local contrast launch", 3);
  });
}

int wavelet_denoise_supported(size_t w, size_t h) {
  // HatTransform's first loop reads index 2*scale-1: the level-4 hat (scale 16) needs 32 samples per line
  if (w < 32 || h < 32) return fail(MB200_EUNSUPPORTED, "wavelet denoise: %zux%zu is below 32x32", w, h);
  return MB200_OK;
}

int launch_wavelet_denoise(const float *src, float *dst, float *planes, size_t w, size_t h, int channels, double threshold,
                           double softness, void *stream) {
  int rc = check_hook_image(src, dst, w, h, channels, "wavelet denoise");
  if (!rc) rc = wavelet_denoise_supported(w, h);
  if (rc) return rc;
  if ((h + 7) / 8 > 65535) return fail(MB200_EUNSUPPORTED, "wavelet denoise: more than %d rows", 65535 * 8);
  static const float noise_levels[5] = {0.8002f, 0.2735f, 0.1202f, 0.0585f, 0.0291f};       // :3541-3543
  const int colours = channels >= 3 ? 3 : 1;
  const size_t n = w * h, set = static_cast<size_t>(colours) * n;
  // planes: [acc | low A | low B], `colours` planes each; the low-pass planes alternate between levels
  float *acc = planes, *low[2] = {planes + set, planes + 2 * set};
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const dim3 grid(static_cast<unsigned>((w + 31) / 32), static_cast<unsigned>((h + 7) / 8), static_cast<unsigned>(colours));
  const int iw = static_cast<int>(w), ih = static_cast<int>(h);
  for (int level = 0; level < 5; ++level) {
    WaveletLevel lv;
    lv.level = level;
    lv.scale = 1 << level;
    lv.magnitude = threshold * static_cast<double>(noise_levels[level]);
    lv.adjust = static_cast<float>(lv.magnitude - softness * lv.magnitude);
    lv.softness = static_cast<float>(softness);
    wavelet_level_kernel<<<grid, dim3(32, 8), 0, s>>>(src, dst, channels, low[(level + 1) & 1], low[level & 1], acc, iw,
                                                      ih, lv);
    rc = launch_status("wavelet denoise launch");
    if (rc) return rc;
  }
  return MB200_OK;
}

}  // namespace mb200
