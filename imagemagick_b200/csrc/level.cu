// level.cu -- the level and stretch operators of MagickCore/enhance.c: LevelImage (:2913), LevelizeImage (:3062),
// MinMaxStretchImage (histogram.c:927, AutoLevelImage's body), ContrastStretchImage (:1544, NormalizeImage's body),
// LinearStretchImage (:3347) and GammaImage (:2322), in place on the channels with the Update trait.
//
// Reference arithmetic (Q16-HDRI; MagickRealType is double, ClampToQuantum a float cast):
//   Level     q = ClampToQuantum(QuantumRange * gamma_pow(PerceptibleReciprocal(white-black) * (q-black),
//                                                          PerceptibleReciprocal(gamma)))
//             then ClampImage on the same channels (< 0 -> 0, >= QuantumRange -> QuantumRange, NaN stays NaN)
//   Levelize  q = ClampToQuantum(gamma_pow(QuantumScale*q, gamma) * (white-black) + black), no clamp
//   gamma_pow(v, g) = v < 0 ? v : pow(v, g)
// The point kernel is unfused IEEE double in the reference's order and skips pow when the exponent is exactly 1.0
// (pow(v, 1) == v), so gamma-1 levels are bit exact; other exponents use CUDA's pow.
//
// MinMaxStretchImage takes GetImageRange (statistic.c:1851-1929) first.  Each row's minimum and maximum start from the
// row's first sample of channel 0 -- whatever that channel's traits -- and then take the Update channels with `<` / `>`:
// a row that starts with NaN stays NaN and is dropped by the merge, which starts from MagickMaximumValue /
// MagickMinimumValue.  The range is two launches (one block per row, then a one-block merge) into device memory, and the
// level kernel takes the reference's fabs(min-max) >= MagickEpsilon decision itself, so nothing is read back.  Ties of
// +0 and -0 are resolved in no particular order, as the reference's parallel row merge resolves them.
//
// EqualizeImage (enhance.c:2040-2290; also the second half of EmbossImage, effect.c:1600-1681):
//   1. histogram[bin][i]++ for every channel i of every pixel, bin = ScaleQuantumToMap(ClampToQuantum(intensity)) where
//      intensity is the pixel's GetPixelIntensity (Rec709 luma; the gray sample of gray images) when the channel mask
//      carries SyncChannels -- which the default mask (AllChannels) does -- and the channel's own value otherwise (:2125-2129);
//   2. map = running sum of the histogram; black = map[0], white = map[MaxMap];
//      equalize_map[j] = ScaleMapToQuantum(MaxMap * (map[j] - black) / (white - black))              (:2138-2169)
//   3. every channel with black != white: q = equalize_map[ScaleQuantumToMap(q)]                      (:2229-2260)
// Steps 1 and 3 are the two passes of equalize.cuh (integer counts: exact; table lookup: exact), step 2 -- 65 536 doubles
// per channel in the reference's own order -- runs on the host between them, so the result is bit-identical.
//
// ContrastStretch, LinearStretch and Gamma are EqualizeImage's two passes (equalize.cuh: histogram, table apply) with
// their own table, built on the host in the reference's order; ContrastStretch and LinearStretch read the histogram back
// (the stream is synchronised).  Gamma reads nothing back, but its table is a pageable upload, which CUDA orders after
// the stream's earlier work.
#include "launch.cuh"
#include "equalize.cuh"
#include "quantum.cuh"

#include <cuda_runtime.h>

#include <cmath>
#include <algorithm>
#include <vector>

namespace mb200 {
namespace {

constexpr double kEpsilon = 1.0e-12;                  // MagickEpsilon
constexpr double kMaximumValue = 1.79769313486231570E+308;   // MagickMaximumValue
constexpr double kMinimumValue = 2.22507385850720140E-308;   // MagickMinimumValue

__host__ __device__ __forceinline__ double perceptible_reciprocal(double x) {
  const double sign = x < 0.0 ? -1.0 : 1.0;
  if ((sign * x) >= kEpsilon) return 1.0 / x;
  return sign / kEpsilon;
}

// One level / levelize pass.  range: device {min, max} of GetImageRange (AutoLevel), or null for explicit points.
struct LevelArgs {
  double black, white;           // Level: the points, or (range) the amounts added to min / taken from max
  double scale;                  // Level: PerceptibleReciprocal(white - black); Levelize: white - black
  double exponent;               // Level: PerceptibleReciprocal(gamma); Levelize: gamma
  const double *range;
  unsigned update_mask;
  int levelize;
};

template <int CH, bool VEC>
__global__ void __launch_bounds__(256) level_kernel(float *buf, size_t npixels, LevelArgs a) {
  const size_t i = static_cast<size_t>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= npixels) return;
  double black = a.black, scale = a.scale;
  if (a.range) {                                                 // histogram.c:948-951 / :968-971
    black = __dadd_rn(__ldg(a.range), a.black);
    const double white = __dsub_rn(__ldg(a.range + 1), a.white);
    if (!(fabs(__dsub_rn(black, white)) >= kEpsilon)) return;
    scale = perceptible_reciprocal(__dsub_rn(white, black));
  }
  float *q = buf + i * CH;
  float v[CH];
  if constexpr (VEC) {
    const float4 t = *reinterpret_cast<const float4 *>(q);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[CH - 1] = t.w;
  } else {
#pragma unroll
    for (int c = 0; c < CH; ++c) v[c] = q[c];
  }
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    if (!((a.update_mask >> c) & 1u)) continue;
    const double x = static_cast<double>(v[c]);
    if (a.levelize) {                                            // enhance.c:3067-3068 LevelizeValue
      double t = __dmul_rn(QS, x);
      if (!(t < 0.0) && a.exponent != 1.0) t = pow(t, a.exponent);
      v[c] = static_cast<float>(__dadd_rn(__dmul_rn(t, a.scale), a.black));
    } else {                                                     // enhance.c:2900-2911 LevelPixel, then ClampImage
      double t = __dmul_rn(scale, __dsub_rn(x, black));
      if (!(t < 0.0) && a.exponent != 1.0) t = pow(t, a.exponent);
      const float f = static_cast<float>(__dmul_rn(QR, t));
      v[c] = f < 0.0f ? 0.0f : f >= 65535.0f ? 65535.0f : f;
    }
  }
  if constexpr (VEC) *reinterpret_cast<float4 *>(q) = make_float4(v[0], v[1], v[2], v[CH - 1]);
  else {
#pragma unroll
    for (int c = 0; c < CH; ++c) q[c] = v[c];
  }
}

// GetImageRange, one block per row: rows[2y] / rows[2y+1] = the row's minimum / maximum over the channels of `select`,
// seeded with the row's first sample of channel 0.
template <int CH, bool VEC>
__global__ void __launch_bounds__(256) range_rows_kernel(const float *__restrict__ buf, size_t width, unsigned select,
                                                         double *__restrict__ rows) {
  const float *row = buf + static_cast<size_t>(blockIdx.x) * width * CH;
  double lo = INFINITY, hi = -INFINITY;                          // identities of the `<` / `>` updates below
  for (size_t x = threadIdx.x; x < width; x += 256) {
    float v[CH];
    if constexpr (VEC) {
      const float4 t = __ldg(reinterpret_cast<const float4 *>(row + x * CH));
      v[0] = t.x; v[1] = t.y; v[2] = t.z; v[CH - 1] = t.w;
    } else {
#pragma unroll
      for (int c = 0; c < CH; ++c) v[c] = __ldg(row + x * CH + c);
    }
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      if (!((select >> c) & 1u)) continue;
      const double d = static_cast<double>(v[c]);
      if (d < lo) lo = d;                                        // NaN samples never win a comparison
      if (d > hi) hi = d;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double l = __shfl_down_sync(0xffffffffu, lo, o), h = __shfl_down_sync(0xffffffffu, hi, o);
    if (l < lo) lo = l;
    if (h > hi) hi = h;
  }
  __shared__ double s_lo[8], s_hi[8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { s_lo[warp] = lo; s_hi[warp] = hi; }
  __syncthreads();
  if (threadIdx.x == 0) {
    const double seed = static_cast<double>(row[0]);
    double row_lo = seed, row_hi = seed;                          // statistic.c:1894-1895
    for (int w = 0; w < 8; ++w) {
      if (s_lo[w] < row_lo) row_lo = s_lo[w];
      if (s_hi[w] > row_hi) row_hi = s_hi[w];
    }
    rows[2 * static_cast<size_t>(blockIdx.x)] = row_lo;
    rows[2 * static_cast<size_t>(blockIdx.x) + 1] = row_hi;
  }
}

// The reference's merge of the row results (statistic.c:1917-1923), one block: range = {min, max}.
__global__ void __launch_bounds__(1024) range_merge_kernel(const double *__restrict__ rows, size_t height,
                                                           double *__restrict__ range) {
  double lo = kMaximumValue, hi = kMinimumValue;
  for (size_t y = threadIdx.x; y < height; y += 1024) {
    const double l = rows[2 * y], h = rows[2 * y + 1];
    if (l < lo) lo = l;
    if (h > hi) hi = h;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double l = __shfl_down_sync(0xffffffffu, lo, o), h = __shfl_down_sync(0xffffffffu, hi, o);
    if (l < lo) lo = l;
    if (h > hi) hi = h;
  }
  __shared__ double s_lo[32], s_hi[32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { s_lo[warp] = lo; s_hi[warp] = hi; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 32; ++w) {
      if (s_lo[w] < lo) lo = s_lo[w];
      if (s_hi[w] > hi) hi = s_hi[w];
    }
    range[0] = lo;
    range[1] = hi;
  }
}

// IdentifyImageGray's pixel scan (attribute.c:1564-1626): bit 0 = some pixel is not gray (IsPixelGray), bit 1 = some
// pixel is not monochrome (IsPixelMonochrome).  Gray images give red, green and blue the gray sample.
template <int CH>
__global__ void __launch_bounds__(256) gray_kernel(const float *__restrict__ buf, size_t npixels, unsigned *flags) {
  const size_t i = static_cast<size_t>(blockIdx.x) * 256 + threadIdx.x;
  unsigned f = 0;
  if (i < npixels) {
    const float *p = buf + i * CH;
    const double r = p[0], g = p[CH >= 3 ? 1 : 0], b = p[CH >= 3 ? 2 : 0];
    const bool gray = fabs(r - g) < kEpsilon && fabs(g - b) < kEpsilon;
    const bool mono = gray && !(fabs(r) >= kEpsilon && fabs(r - QR) >= kEpsilon);
    f = (gray ? 0u : 1u) | (mono ? 0u : 2u);
  }
  f = __reduce_or_sync(0xffffffffu, f);
  if ((threadIdx.x & 31) == 0 && f) atomicOr(flags, f);
}

int launch_level_pass(float *buf, size_t npixels, int channels, const LevelArgs &a, cudaStream_t s) {
  unsigned grid;
  int rc = grid_of(npixels, 256, &grid, "level");
  if (rc) return rc;
  return with_channels(channels, aligned16(buf), "level", [&](auto ch, auto vec) {
    level_kernel<ch(), vec()><<<grid, 256, 0, s>>>(buf, npixels, a);
    return launch_status("level launch");
  });
}

// GetImageRange over the channels of `select` into range[0..1] (rows: 2 * height doubles of scratch)
int launch_range(const float *buf, size_t width, size_t height, int channels, unsigned select, double *rows, double *range,
                 cudaStream_t s) {
  if (height == 0 || height > 0x7fffffffull) return fail(MB200_EINVAL, "range: bad image size");
  const unsigned grid = static_cast<unsigned>(height);
  return with_channels(channels, aligned16(buf), "range", [&](auto ch, auto vec) {
    range_rows_kernel<ch(), vec()><<<grid, 256, 0, s>>>(buf, width, select, rows);
    range_merge_kernel<<<1, 1024, 0, s>>>(rows, height, range);
    return launch_status("range launch", 2);
  });
}

// The histogram pass of equalize.cuh into a fresh device buffer of nhist * kBins counts, read back into `counts`;
// char_bins: AutoThresholdImage's 256-bin intensity histogram (sync implied).
int histogram_readback(const float *buf, size_t npixels, int channels, int sync, std::vector<unsigned> *counts,
                       cudaStream_t s, bool char_bins = false) {
  unsigned grid;
  int rc = grid_of(npixels, 256, &grid, "histogram");
  if (rc) return rc;
  if (char_bins) sync = 1;
  const int nhist = sync ? 1 : channels;
  StreamAlloc d_counts(s);
  if ((rc = d_counts.alloc(sizeof(unsigned) * kBins * nhist, "histogram: allocation"))) return rc;
  cudaError_t e = cudaMemsetAsync(d_counts.ptr, 0, sizeof(unsigned) * kBins * nhist, s);
  if (e != cudaSuccess) return cuda_fail(e, "histogram readback");
  rc = with_channels(channels, "histogram", [&](auto ch) {
    if (char_bins) histogram_kernel<ch(), true><<<grid, 256, 0, s>>>(buf, npixels, sync, d_counts.as<unsigned>());
    else histogram_kernel<ch(), false><<<grid, 256, 0, s>>>(buf, npixels, sync, d_counts.as<unsigned>());
    return launch_status("histogram readback");
  });
  if (rc) return rc;
  counts->assign(static_cast<size_t>(kBins) * nhist, 0u);
  e = cudaMemcpyAsync(counts->data(), d_counts.ptr, counts->size() * sizeof(unsigned), cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  return e == cudaSuccess ? MB200_OK : cuda_fail(e, "histogram readback");
}

// The table pass of equalize.cuh: table[c][bin] for the channels of `enabled`.  copy_h2d returns once the host table
// has been consumed (a pageable copy is ordered after the stream's earlier work); the pass itself is not waited for.
int apply_table(float *buf, size_t npixels, int channels, const std::vector<float> &table, unsigned enabled,
                cudaStream_t s) {
  if (!enabled) return MB200_OK;
  unsigned grid;
  int rc = grid_of(npixels, 256, &grid, "table");
  if (rc) return rc;
  StreamAlloc d_table(s);
  if ((rc = d_table.alloc(table.size() * sizeof(float), "table: allocation"))) return rc;
  if ((rc = copy_h2d(d_table.ptr, table.data(), table.size() * sizeof(float), s))) return rc;
  return with_channels(channels, "table", [&](auto ch) {
    equalize_apply_kernel<ch()><<<grid, 256, 0, s>>>(buf, npixels, d_table.as<float>(), enabled);
    return launch_status("table launch");
  });
}

// ScaleMapToQuantum (quantum-private.h:465-475, HDRI)
float scale_map_to_quantum(double value) {
  if (value <= 0.0) return 0.0f;
  if (value >= 65535.0) return 65535.0f;
  return static_cast<float>(value);
}

}  // namespace

int launch_level(float *buf, size_t npixels, int channels, double black, double white, double gamma, unsigned update_mask,
                 bool levelize, void *stream) {
  LevelArgs a{};
  a.black = black;
  a.white = white;
  a.scale = levelize ? white - black : perceptible_reciprocal(white - black);
  a.exponent = levelize ? gamma : perceptible_reciprocal(gamma);
  a.update_mask = update_mask;
  a.levelize = levelize ? 1 : 0;
  return launch_level_pass(buf, npixels, channels, a, static_cast<cudaStream_t>(stream));
}

int launch_minmax_stretch(float *buf, size_t width, size_t height, int channels, double black, double white, double gamma,
                          bool per_channel, unsigned update_mask, void *stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  StreamAlloc rows(s);
  int rc = rows.alloc(sizeof(double) * 2 * (height + 1), "minmax stretch: allocation");
  if (rc) return rc;
  double *d_rows = rows.as<double>(), *d_range = d_rows + 2 * height;
  LevelArgs a{};
  a.black = black;
  a.white = white;
  a.exponent = perceptible_reciprocal(gamma);
  a.range = d_range;
  if (!per_channel) {                                            // histogram.c:944-953: all channels at once
    rc = launch_range(buf, width, height, channels, update_mask, d_rows, d_range, s);
    a.update_mask = update_mask;
    if (!rc) rc = launch_level_pass(buf, width * height, channels, a, s);
  } else {
    // histogram.c:957-973: the Update channels one at a time, each under SetImageChannelMask(1 << offset).  That mask
    // bit names the PixelChannel of the same number, so it selects the colour channel at that offset (gray 0, red 0,
    // green 1, blue 2) and never alpha (PixelChannel 4): the alpha offset's turn levels nothing.
    const int colour = channels >= 3 ? 3 : 1;
    for (int c = 0; c < colour && !rc; ++c) {
      if (!((update_mask >> c) & 1u)) continue;
      rc = launch_range(buf, width, height, channels, 1u << c, d_rows, d_range, s);
      a.update_mask = 1u << c;
      if (!rc) rc = launch_level_pass(buf, width * height, channels, a, s);
    }
  }
  return rc;
}

int launch_contrast_stretch(float *buf, size_t width, size_t height, int channels, double black_point, double white_point,
                            bool per_channel, unsigned update_mask, float *black, float *white, void *stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t npixels = width * height;
  std::vector<unsigned> counts;                                  // api.cu declines 2^32 pixels or more (32-bit counts)
  int rc = histogram_readback(buf, npixels, channels, per_channel ? 0 : 1, &counts, s);
  if (rc) return rc;
  // enhance.c:1650-1697 in the reference's order
  std::vector<float> table(static_cast<size_t>(kBins) * channels, 0.0f);
  unsigned enabled = 0;
  const double total = static_cast<double>(width) * static_cast<double>(height);
  for (int c = 0; c < channels; ++c) {
    const unsigned *h = counts.data() + static_cast<size_t>(per_channel ? c : 0) * kBins;
    double intensity = 0.0;
    long j;
    for (j = 0; j <= 65535; ++j) {
      intensity += static_cast<double>(h[j]);
      if (intensity > black_point) break;
    }
    black[c] = static_cast<float>(j);
    intensity = 0.0;
    for (j = 65535; j != 0; --j) {
      intensity += static_cast<double>(h[j]);
      if (intensity > (total - white_point)) break;
    }
    white[c] = static_cast<float>(j);
    const double gamma = perceptible_reciprocal(static_cast<double>(white[c] - black[c]));
    float *map = table.data() + static_cast<size_t>(c) * kBins;
    for (j = 0; j <= 65535; ++j) {
      if (j < static_cast<long>(black[c])) map[j] = 0.0f;
      else if (j > static_cast<long>(white[c])) map[j] = 65535.0f;
      else if (black[c] != white[c])
        map[j] = scale_map_to_quantum(65535.0 * gamma * (static_cast<double>(j) - static_cast<double>(black[c])));
    }
    if (((update_mask >> c) & 1u) && black[c] != white[c]) enabled |= 1u << c;
  }
  rc = apply_table(buf, npixels, channels, table, enabled, s);
  for (int c = channels; c < 4; ++c) black[c] = white[c] = 0.0f;
  return rc;
}

int launch_linear_stretch(float *buf, size_t width, size_t height, int channels, double black_point, double white_point,
                          unsigned update_mask, double *black_bin, double *white_bin, void *stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t npixels = width * height;
  std::vector<unsigned> counts;                                  // api.cu declines 2^32 pixels or more (32-bit counts)
  int rc = histogram_readback(buf, npixels, channels, 1, &counts, s);
  if (rc) return rc;
  // enhance.c:3398-3411
  double intensity = 0.0;
  long black, white;
  for (black = 0; black < 65535; ++black) {
    intensity += static_cast<double>(counts[black]);
    if (intensity >= black_point) break;
  }
  intensity = 0.0;
  for (white = 65535; white != 0; --white) {
    intensity += static_cast<double>(counts[white]);
    if (intensity >= white_point) break;
  }
  *black_bin = static_cast<double>(black);
  *white_bin = static_cast<double>(white);
  return launch_level(buf, npixels, channels, static_cast<double>(scale_map_to_quantum(static_cast<double>(black))),
                      static_cast<double>(scale_map_to_quantum(static_cast<double>(white))), 1.0, update_mask, false, s);
}

int launch_gamma(float *buf, size_t npixels, int channels, double gamma, unsigned update_mask, void *stream) {
  if (gamma == 1.0 || update_mask == 0) return MB200_OK;         // enhance.c:2351-2352
  // enhance.c:2356-2360 with the host's libm, as the reference builds it; all zeros for gamma 0
  std::vector<float> table(static_cast<size_t>(kBins) * channels, 0.0f);
  if (gamma != 0.0) {
    const double exponent = perceptible_reciprocal(gamma);
    for (unsigned i = 0; i < kBins; ++i) table[i] = scale_map_to_quantum(65535.0 * std::pow(static_cast<double>(i) / 65535.0, exponent));
    for (int c = 1; c < channels; ++c) std::copy(table.begin(), table.begin() + kBins, table.begin() + static_cast<size_t>(c) * kBins);
  }
  return apply_table(buf, npixels, channels, table, update_mask, static_cast<cudaStream_t>(stream));
}

int launch_identify_gray(const float *buf, size_t npixels, int channels, int *type, void *stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  unsigned grid;
  int rc = grid_of(npixels, 256, &grid, "identify gray");
  if (rc) return rc;
  StreamAlloc d_flags(s);
  if ((rc = d_flags.alloc(sizeof(unsigned), "identify gray: allocation"))) return rc;
  cudaError_t e = cudaMemsetAsync(d_flags.ptr, 0, sizeof(unsigned), s);
  if (e != cudaSuccess) return cuda_fail(e, "identify gray");
  rc = with_channels(channels, "identify gray", [&](auto ch) {
    gray_kernel<ch()><<<grid, 256, 0, s>>>(buf, npixels, d_flags.as<unsigned>());
    return launch_status("identify gray");
  });
  if (rc) return rc;
  unsigned flags = 0;
  e = cudaMemcpyAsync(&flags, d_flags.ptr, sizeof(unsigned), cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) return cuda_fail(e, "identify gray");
  *type = (flags & 1u) ? 0 : (flags & 2u) ? 1 : 2;
  return MB200_OK;
}

int auto_threshold_histogram(const float *buf, size_t npixels, int channels, unsigned counts[256], void *stream) {
  std::vector<unsigned> all;
  const int rc = histogram_readback(buf, npixels, channels, 1, &all, static_cast<cudaStream_t>(stream), true);
  if (rc) return rc;
  std::copy(all.begin(), all.begin() + 256, counts);
  return MB200_OK;
}

int launch_equalize(float *buf, size_t npixels, int channels, int sync_channels, void *stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (channels < 1 || channels > 4) return fail(MB200_EINVAL, "equalize: 1..4 channels");
  unsigned grid;
  int rc = grid_of(npixels, 256, &grid, "equalize");
  if (rc) return rc;
  std::vector<unsigned> counts;
  rc = histogram_readback(buf, npixels, channels, sync_channels, &counts, s);
  if (rc) return rc;
  // enhance.c:2138-2169 in the reference's order (running sums in double; 65 536 entries per channel)
  std::vector<float> table(static_cast<size_t>(kBins) * channels, 0.0f);
  unsigned enabled = 0;
  for (int c = 0; c < channels; ++c) {
    const unsigned *h = counts.data() + static_cast<size_t>(sync_channels ? 0 : c) * kBins;
    std::vector<double> map(kBins);
    double intensity = 0.0;
    for (unsigned j = 0; j < kBins; ++j) { intensity += static_cast<double>(h[j]); map[j] = intensity; }
    const double black = map[0], white = map[kBins - 1];
    if (black == white) continue;
    enabled |= 1u << c;
    for (unsigned j = 0; j < kBins; ++j)
      table[static_cast<size_t>(c) * kBins + j] = scale_map_to_quantum((65535.0 * (map[j] - black)) / (white - black));
  }
  return apply_table(buf, npixels, channels, table, enabled, s);
}

}  // namespace mb200
