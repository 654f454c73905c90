// threshold.cu -- AdaptiveThresholdImage (MagickCore/threshold.c:182), out of place.
//
// Reference arithmetic for one row y and one channel (Q16-HDRI; every sum a double starting from 0.0).  The window's
// origin is column -(w/2), row y - h/2 (integer division); virtual pixels clamp both coordinates (Edge / Undefined).
//   S = every sample of the window at x = 0, row-major (v outer, u inner);  B = the samples of window column w-1, v order
//   for x = 0 .. columns-1:
//     S = S - B;  B = 0.0 + the samples of window column x (v order);  S = S + sample(v, x+w-1) for v = 0 .. h-1
//     mean = S / (double) (w*h) + bias;  out = (double) centre <= mean ? 0 : QuantumRange
// Copy-trait channels take the centre sample.  S is one serial chain of IEEE additions per (row, channel): it is never
// reassociated, so a NaN or +-inf that enters it stays for the rest of the row (every later output is QuantumRange).
// The B values are fresh, independent column sums: B of window column j is the same double whenever it is formed, so
// both kernels form it from the samples they load for S at step j-w+1 and keep the last w of them in a ring.
//
// Tile family (adaptive_tile_kernel): one thread per (row, channel) chain, a CTA per band of kRows rows.  The band's
// kRows+h-1 source rows are staged kCols (+ w-1 halo) columns at a time into shared memory, double-buffered with
// per-element cp.async from clamped addresses (the edge copies TMA's zero fill cannot give, and any alignment), so each
// source sample is read (kRows+h-1)/kRows times.  The tile pitch is congruent to the channel count mod 32: lane t of a
// warp then reads word t + const (kRows x CH chains side by side), free of bank conflicts.  Results are staged and
// written back as full rows of the chunk.
// Direct family (adaptive_direct_kernel): the same arithmetic reading through L1 / L2, for windows whose tile does not
// fit in shared memory.  Both families give the same bits.
//
// AutoThresholdImage (:660): the threshold of Kapur (:391), OTSU (:491) and Triangle (:570) from the normalised 256-bin
// histogram, on the host in the reference's order with the same libm calls (auto_threshold_percent).
#include "mb200_internal.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>

namespace mb200 {
namespace {

constexpr int kRows = 32;        // chains' rows per CTA (tile family)
constexpr int kCols = 32;        // columns per staged chunk
constexpr float kQR = 65535.0f;

struct AdaptiveArgs {
  const float *src;
  float *dst;
  int width, height, w, h;
  double area, bias;
  unsigned update;
  int pitch;                     // tile row pitch in floats
};

__device__ __forceinline__ void cp_async4(float *smem, const float *gptr) {
  const unsigned addr = static_cast<unsigned>(__cvta_generic_to_shared(smem));
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(addr), "l"(gptr));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N)); }

template <int CH>
__global__ void __launch_bounds__(kRows * 4) adaptive_tile_kernel(const AdaptiveArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  constexpr int T = kRows * CH;
  constexpr int kOutPitch = kCols * CH + CH;
  const int tile_rows = kRows + a.h - 1, tile_cols = kCols + a.w - 1;
  const size_t tile_floats = static_cast<size_t>(tile_rows) * a.pitch;
  float *tiles = reinterpret_cast<float *>(smem);
  double *ring = reinterpret_cast<double *>(tiles + 2 * tile_floats);     // [slot][thread]
  float *out = reinterpret_cast<float *>(ring + static_cast<size_t>(a.w) * T);
  const int t = threadIdx.x, r = t / CH, c = t - r * CH;
  const int y0 = blockIdx.x * kRows, y = y0 + r;
  const int top = y0 - a.h / 2, left = -(a.w / 2);
  const int nchunks = (a.width + kCols - 1) / kCols;
  const bool live = y < a.height, update = (a.update >> c) & 1u;

  auto stage = [&](int k, float *buf) {
    const int per_row = tile_cols * CH, x_base = k * kCols + left;
    for (int tr = 0; tr < tile_rows; ++tr) {
      const float *row = a.src + static_cast<size_t>(min(max(top + tr, 0), a.height - 1)) * a.width * CH;
      for (int e = t; e < per_row; e += T) {
        const int tc = e / CH, cc = e - tc * CH;
        const int sx = min(max(x_base + tc, 0), a.width - 1);
        cp_async4(buf + tr * a.pitch + e, row + static_cast<size_t>(sx) * CH + cc);
      }
    }
    cp_async_commit();
  };

  double sum = 0.0;
  int slot = a.w - 1;                        // ring slot of window column x+w-1 (== that of column x-1)
  stage(0, tiles);
  for (int k = 0; k < nchunks; ++k) {
    if (k + 1 < nchunks) {
      stage(k + 1, tiles + ((k + 1) & 1) * tile_floats);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const int x0 = k * kCols, kw = min(kCols, a.width - x0);
    if (live) {
      const float *col = tiles + (k & 1) * tile_floats + r * a.pitch + c;    // tile row r, chunk column 0, channel c
      const float *centre = col + (a.h / 2) * a.pitch + (a.w / 2) * CH;
      if (!update) {
        for (int xl = 0; xl < kw; ++xl) out[r * kOutPitch + xl * CH + c] = centre[xl * CH];
      } else {
        if (k == 0) {                        // the initial window, row-major; B of every window column 0 .. w-1
          for (int v = 0; v < a.h; ++v)
            for (int u = 0; u < a.w; ++u) sum = sum + static_cast<double>(col[v * a.pitch + u * CH]);
          for (int u = 0; u < a.w; ++u) {
            double b = 0.0;
            for (int v = 0; v < a.h; ++v) b = b + static_cast<double>(col[v * a.pitch + u * CH]);
            ring[u * T + t] = b;
          }
        }
        for (int xl = 0; xl < kw; ++xl) {
          double *bs = ring + slot * T + t;
          sum = sum - *bs;
          const float *p = col + (xl + a.w - 1) * CH;
          double b = 0.0;
          for (int v = 0; v < a.h; ++v) {
            const double s = static_cast<double>(p[v * a.pitch]);
            b = b + s;
            sum = sum + s;
          }
          *bs = b;
          slot = slot + 1 == a.w ? 0 : slot + 1;
          const double mean = sum / a.area + a.bias;
          out[r * kOutPitch + xl * CH + c] = static_cast<double>(centre[xl * CH]) <= mean ? 0.0f : kQR;
        }
      }
    }
    __syncthreads();
    for (int rr = 0; rr < kRows && y0 + rr < a.height; ++rr) {
      float *q = a.dst + (static_cast<size_t>(y0 + rr) * a.width + x0) * CH;
      for (int e = t; e < kw * CH; e += T) q[e] = out[rr * kOutPitch + e];
    }
  }
}

template <int CH>
__global__ void __launch_bounds__(128) adaptive_direct_kernel(const AdaptiveArgs a, double *ring_base) {
  const long g = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (g >= static_cast<long>(a.height) * CH) return;
  const int y = static_cast<int>(g / CH), c = static_cast<int>(g - static_cast<long>(y) * CH);
  const int top = y - a.h / 2, left = -(a.w / 2);
  auto sample = [&](int v, int j) {          // window row v, window column j
    const int sy = min(max(top + v, 0), a.height - 1), sx = min(max(left + j, 0), a.width - 1);
    return static_cast<double>(__ldg(a.src + (static_cast<size_t>(sy) * a.width + sx) * CH + c));
  };
  float *q = a.dst + static_cast<size_t>(y) * a.width * CH + c;
  if (!((a.update >> c) & 1u)) {
    const float *p = a.src + static_cast<size_t>(y) * a.width * CH + c;
    for (int x = 0; x < a.width; ++x) q[static_cast<size_t>(x) * CH] = __ldg(p + static_cast<size_t>(x) * CH);
    return;
  }
  double *ring = ring_base + g;              // [slot][chain], stride height * CH
  const size_t stride = static_cast<size_t>(a.height) * CH;
  double sum = 0.0;
  for (int v = 0; v < a.h; ++v)
    for (int u = 0; u < a.w; ++u) sum = sum + sample(v, u);
  for (int u = 0; u < a.w; ++u) {
    double b = 0.0;
    for (int v = 0; v < a.h; ++v) b = b + sample(v, u);
    ring[u * stride] = b;
  }
  int slot = a.w - 1;
  const float *centre = a.src + static_cast<size_t>(y) * a.width * CH + c;
  for (int x = 0; x < a.width; ++x) {
    double *bs = ring + slot * stride;
    sum = sum - *bs;
    double b = 0.0;
    for (int v = 0; v < a.h; ++v) {
      const double s = sample(v, x + a.w - 1);
      b = b + s;
      sum = sum + s;
    }
    *bs = b;
    slot = slot + 1 == a.w ? 0 : slot + 1;
    const double mean = sum / a.area + a.bias;
    q[static_cast<size_t>(x) * CH] = static_cast<double>(__ldg(centre + static_cast<size_t>(x) * CH)) <= mean ? 0.0f : kQR;
  }
}

// Bytes of shared memory the tile family needs for a window, and its tile pitch (floats, == channels mod 32).
size_t tile_bytes(int channels, int w, int h, int *pitch) {
  const int cols = (kCols + w - 1) * channels;
  *pitch = cols + ((channels - cols % 32) + 32) % 32;
  return 2 * sizeof(float) * static_cast<size_t>(kRows + h - 1) * *pitch + sizeof(double) * static_cast<size_t>(w) * kRows * channels +
         sizeof(float) * static_cast<size_t>(kRows) * (kCols * channels + channels);
}

template <int CH>
int launch_adaptive_ch(const AdaptiveArgs &a, bool tile, size_t smem, cudaStream_t s) {
  if (tile) {
    const cudaError_t e = cudaFuncSetAttribute(adaptive_tile_kernel<CH>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               static_cast<int>(smem));
    if (e != cudaSuccess) return cuda_fail(e, "adaptive threshold: shared memory attribute");
    adaptive_tile_kernel<CH><<<(a.height + kRows - 1) / kRows, kRows * CH, smem, s>>>(a);
    count_family(kAdaptiveThresholdTile);
    count_launch();
    const cudaError_t le = cudaGetLastError();
    return le == cudaSuccess ? MB200_OK : cuda_fail(le, "adaptive threshold tile launch");
  }
  double *ring = nullptr;
  const size_t ring_bytes = sizeof(double) * a.w * static_cast<size_t>(a.height) * CH;
  cudaError_t e = cudaMallocAsync(reinterpret_cast<void **>(&ring), ring_bytes, temp_pool(), s);
  if (e != cudaSuccess) return cuda_fail(e, "adaptive threshold: ring allocation");
  const long chains = static_cast<long>(a.height) * CH;
  adaptive_direct_kernel<CH><<<static_cast<unsigned>((chains + 127) / 128), 128, 0, s>>>(a, ring);
  count_family(kAdaptiveThresholdDirect);
  count_launch();
  e = cudaGetLastError();
  cudaFreeAsync(ring, s);
  return e == cudaSuccess ? MB200_OK : cuda_fail(e, "adaptive threshold direct launch");
}

}  // namespace

int launch_adaptive_threshold(const float *src, float *dst, size_t width, size_t height, int channels, size_t w, size_t h,
                              double bias, unsigned update_mask, void *stream) {
  if (channels < 1 || channels > 4) return fail(MB200_EINVAL, "adaptive threshold: 1..4 channels");
  if (width > 0x7fffffffull / 8 || height > 0x7fffffffull / 8)
    return fail(MB200_EUNSUPPORTED, "adaptive threshold: image too large");
  if (w > MB200_ADAPTIVE_THRESHOLD_MAX_WINDOW || h > MB200_ADAPTIVE_THRESHOLD_MAX_WINDOW)
    return fail(MB200_EUNSUPPORTED, "adaptive threshold: window %zux%zu is larger than %d", w, h,
                MB200_ADAPTIVE_THRESHOLD_MAX_WINDOW);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  AdaptiveArgs a{src, dst, static_cast<int>(width), static_cast<int>(height), static_cast<int>(w), static_cast<int>(h),
                 static_cast<double>(static_cast<unsigned long long>(w) * h), bias, update_mask, 0};
  int device = 0, optin = 0;
  cudaGetDevice(&device);
  cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
  const size_t smem = tile_bytes(channels, a.w, a.h, &a.pitch);
  const bool tile = smem <= static_cast<size_t>(optin) && !tuning_knobs().no_adaptive_tile;
  switch (channels) {
    case 1: return launch_adaptive_ch<1>(a, tile, smem, s);
    case 2: return launch_adaptive_ch<2>(a, tile, smem, s);
    case 3: return launch_adaptive_ch<3>(a, tile, smem, s);
    default: return launch_adaptive_ch<4>(a, tile, smem, s);
  }
}

namespace {

constexpr int kMaxIntensity = 255;

double kapur_threshold(const double *histogram) {
  double cumulative[kMaxIntensity + 1], black[kMaxIntensity + 1], white[kMaxIntensity + 1];
  cumulative[0] = histogram[0];
  for (int i = 1; i <= kMaxIntensity; ++i) cumulative[i] = cumulative[i - 1] + histogram[i];
  const double epsilon = 2.22507385850720140E-308;             // MagickMinimumValue
  for (int j = 0; j <= kMaxIntensity; ++j) {
    black[j] = 0.0;
    if (cumulative[j] > epsilon) {
      double entropy = 0.0;
      for (int i = 0; i <= j; ++i)
        if (histogram[i] > epsilon) entropy -= histogram[i] / cumulative[j] * std::log(histogram[i] / cumulative[j]);
      black[j] = entropy;
    }
    white[j] = 0.0;
    if ((1.0 - cumulative[j]) > epsilon) {
      double entropy = 0.0;
      for (int i = j + 1; i <= kMaxIntensity; ++i)
        if (histogram[i] > epsilon)
          entropy -= histogram[i] / (1.0 - cumulative[j]) * std::log(histogram[i] / (1.0 - cumulative[j]));
      white[j] = entropy;
    }
  }
  double maximum = black[0] + white[0];
  size_t threshold = 0;
  for (int j = 1; j <= kMaxIntensity; ++j)
    if ((black[j] + white[j]) > maximum) {
      maximum = black[j] + white[j];
      threshold = static_cast<size_t>(j);
    }
  return 100.0 * threshold / kMaxIntensity;
}

double otsu_threshold(const double *histogram) {
  double myu[kMaxIntensity + 1], omega[kMaxIntensity + 1];
  omega[0] = histogram[0];
  myu[0] = 0.0;
  for (int i = 1; i <= kMaxIntensity; ++i) {
    omega[i] = omega[i - 1] + histogram[i];
    myu[i] = myu[i - 1] + i * histogram[i];
  }
  double threshold = 0.0, max_sigma = 0.0;
  for (int i = 0; i < kMaxIntensity; ++i) {
    double sigma = 0.0;
    if ((omega[i] != 0.0) && (omega[i] != 1.0))
      sigma = std::pow(myu[kMaxIntensity] * omega[i] - myu[i], 2.0) / (omega[i] * (1.0 - omega[i]));
    if (sigma > max_sigma) {
      max_sigma = sigma;
      threshold = static_cast<double>(i);
    }
  }
  return 100.0 * threshold / kMaxIntensity;
}

double triangle_threshold(const double *histogram) {
  long start = 0, end = 0, max = 0;
  for (long i = 0; i <= kMaxIntensity; ++i)
    if (histogram[i] > 0.0) { start = i; break; }
  for (long i = kMaxIntensity; i >= 0; --i)
    if (histogram[i] > 0.0) { end = i; break; }
  double count = 0.0;
  for (long i = 0; i <= kMaxIntensity; ++i)
    if (histogram[i] > count) { max = i; count = histogram[i]; }
  const double x1 = static_cast<double>(max), y1 = histogram[max];
  double x2 = static_cast<double>(end);
  if ((max - start) >= (end - max)) x2 = static_cast<double>(start);
  const double y2 = 0.0, a = y1 - y2, b = x2 - x1, c = (-1.0) * (a * x1 + b * y1);
  const double inverse_ratio = 1.0 / std::sqrt(a * a + b * b + c * c);
  long threshold = 0;
  double max_distance = 0.0;
  if (x2 == static_cast<double>(start)) {
    for (long i = start; i < max; ++i) {
      const double segment = inverse_ratio * (a * i + b * histogram[i] + c), distance = std::sqrt(segment * segment);
      if ((distance > max_distance) && (segment > 0.0)) { threshold = i; max_distance = distance; }
    }
  } else {
    for (long i = end; i > max; --i) {
      const double segment = inverse_ratio * (a * i + b * histogram[i] + c), distance = std::sqrt(segment * segment);
      if ((distance > max_distance) && (segment < 0.0)) { threshold = i; max_distance = distance; }
    }
  }
  return 100.0 * threshold / kMaxIntensity;
}

}  // namespace

double auto_threshold_percent(const unsigned counts[256], int method) {
  double histogram[kMaxIntensity + 1], sum = 0.0;
  for (int i = 0; i <= kMaxIntensity; ++i) histogram[i] = static_cast<double>(counts[i]);
  for (int i = 0; i <= kMaxIntensity; ++i) sum += histogram[i];
  const double sign = sum < 0.0 ? -1.0 : 1.0;                   // PerceptibleReciprocal
  const double gamma = (sign * sum) >= 1.0e-12 ? 1.0 / sum : sign / 1.0e-12;
  for (int i = 0; i <= kMaxIntensity; ++i) histogram[i] = gamma * histogram[i];
  if (method == MB200_KapurThresholdMethod) return kapur_threshold(histogram);
  if (method == MB200_TriangleThresholdMethod) return triangle_threshold(histogram);
  return otsu_threshold(histogram);
}

}  // namespace mb200
