// resize.cu -- one axis of ResizeImage: the weighted gather of HorizontalFilter
// (MagickCore/resize.c:3333-3547) and VerticalFilter (:3549-3759).
//
// Per output sample o the host (resize_filter.cpp) has already produced exactly the
// reference's contribution list: first source index start[o], tap count count[o] and
// the density-normalised double weights.  The device evaluates
//     plain channel : out = (float) sum_j w_j * p_j                          (:3456-3468)
//     blend channel : a_j = w_j*QS*A_j ; out = (float)(PerceptibleReciprocal(sum a_j) *
//                                                     sum a_j*p_j)           (:3472-3484)
// in FP64.  The alpha weighting is applied as one premultiply per tap per pixel
// (t = w*A; acc_c += t*p_c); sum t is at the same time the alpha channel's own result
// and (up to the constant QS, which cancels) gamma.
//
// Mapping (generic kernels): one thread per output pixel (all channels, float4 loads for RGBA).
//  axis 1 (vertical): lanes span 32 consecutive pixels of a row => 512-byte coalesced
//    row reads; a thread produces several consecutive output rows so the overlapping
//    source rows are re-read from L1; weights are warp-uniform broadcast loads.
//  axis 0 (horizontal): lanes span consecutive OUTPUT columns; weights are stored
//    tap-major ([tap][o]) so their loads are coalesced; source reads of neighbouring
//    lanes fall in the same / adjacent 128-byte lines.
#include "mb200_internal.h"

#include <cuda_runtime.h>

namespace mb200 {
namespace {

constexpr double kQuantumScale = 1.0 / 65535.0;
constexpr double kEpsilon = 1.0e-12;

struct ResizeArgs {
  const float *src;
  float *dst;
  int width, height;      // source
  int out_w, out_h;       // destination
  int out_n;              // outputs along the filtered axis
  const int *start;
  const int *count;
  const double *weights;  // tap-major: weights[j*out_n + o]
  int lines_per_thread;
  int o_begin, o_end;     // generic kernels: output sub-range along the filtered axis
};

template <int CH>
struct Pixel { float v[CH]; };

template <int CH>
__device__ __forceinline__ Pixel<CH> load_pixel(const float *p) {
  Pixel<CH> r;
  if (CH == 4) {
    const float4 t = __ldg(reinterpret_cast<const float4 *>(p));
    r.v[0] = t.x; r.v[1] = t.y; r.v[2] = t.z; r.v[CH - 1] = t.w;
  } else if (CH == 2) {
    const float2 t = __ldg(reinterpret_cast<const float2 *>(p));
    r.v[0] = t.x; r.v[CH - 1] = t.y;
  } else {
#pragma unroll
    for (int c = 0; c < CH; ++c) r.v[c] = __ldg(p + c);
  }
  return r;
}

template <int CH>
__device__ __forceinline__ void store_pixel(float *p, const float (&o)[CH]) {
  if (CH == 4) *reinterpret_cast<float4 *>(p) = make_float4(o[0], o[1], o[2], o[CH - 1]);
  else if (CH == 2) *reinterpret_cast<float2 *>(p) = make_float2(o[0], o[CH - 1]);
  else {
#pragma unroll
    for (int c = 0; c < CH; ++c) p[c] = o[c];
  }
}

template <int CH>
__device__ __forceinline__ void accumulate(double (&acc)[CH], double w, const Pixel<CH> &px) {
  constexpr bool kAlpha = (CH == 2 || CH == 4);
  if (kAlpha) {
    const double t = w * static_cast<double>(px.v[CH - 1]);
#pragma unroll
    for (int c = 0; c < CH - 1; ++c) acc[c] = fma(t, static_cast<double>(px.v[c]), acc[c]);
    acc[CH - 1] += t;
  } else {
#pragma unroll
    for (int c = 0; c < CH; ++c) acc[c] = fma(w, static_cast<double>(px.v[c]), acc[c]);
  }
}

template <int CH>
__device__ __forceinline__ void finish(const double (&acc)[CH], float (&out)[CH]) {
  constexpr bool kAlpha = (CH == 2 || CH == 4);
  if (kAlpha) {
    const double gamma = kQuantumScale * acc[CH - 1];
    if (fabs(gamma) >= kEpsilon) {
      const double r = 1.0 / acc[CH - 1];
#pragma unroll
      for (int c = 0; c < CH - 1; ++c) out[c] = static_cast<float>(r * acc[c]);
    } else {
      const double r = gamma < 0.0 ? -1.0 / kEpsilon : 1.0 / kEpsilon;
#pragma unroll
      for (int c = 0; c < CH - 1; ++c) out[c] = static_cast<float>(r * (kQuantumScale * acc[c]));
    }
    out[CH - 1] = static_cast<float>(acc[CH - 1]);
  } else {
#pragma unroll
    for (int c = 0; c < CH; ++c) out[c] = static_cast<float>(acc[c]);
  }
}

// vertical: grid (ceil(width/128), ceil(out_h/lines_per_thread))
template <int CH>
__global__ void __launch_bounds__(128) resize_vertical_kernel(const ResizeArgs a) {
  const int x = blockIdx.x * 128 + threadIdx.x;
  if (x >= a.width) return;
  const int o0 = a.o_begin + blockIdx.y * a.lines_per_thread;
  const int o1 = min(o0 + a.lines_per_thread, a.o_end);
  const float *col = a.src + static_cast<size_t>(x) * CH;
  const size_t pitch = static_cast<size_t>(a.width) * CH;
  for (int o = o0; o < o1; ++o) {
    const int first = __ldg(a.start + o), n = __ldg(a.count + o);
    if (n <= 0) continue;                               // resize.c:3440 leaves the row untouched
    double acc[CH];
#pragma unroll
    for (int c = 0; c < CH; ++c) acc[c] = 0.0;
    const float *p = col + static_cast<size_t>(first) * pitch;
    for (int j = 0; j < n; ++j, p += pitch) {
      const double w = __ldg(a.weights + static_cast<size_t>(j) * a.out_n + o);
      accumulate<CH>(acc, w, load_pixel<CH>(p));
    }
    float out[CH];
    finish<CH>(acc, out);
    store_pixel<CH>(a.dst + (static_cast<size_t>(o) * a.out_w + x) * CH, out);
  }
}

// horizontal: grid (ceil(out_w/128), ceil(height/lines_per_thread))
template <int CH>
__global__ void __launch_bounds__(128) resize_horizontal_kernel(const ResizeArgs a) {
  const int o = a.o_begin + blockIdx.x * 128 + threadIdx.x;
  if (o >= a.o_end) return;
  const int y0 = blockIdx.y * a.lines_per_thread;
  const int y1 = min(y0 + a.lines_per_thread, a.height);
  const int first = __ldg(a.start + o), n = __ldg(a.count + o);
  if (n <= 0) return;
  for (int y = y0; y < y1; ++y) {
    double acc[CH];
#pragma unroll
    for (int c = 0; c < CH; ++c) acc[c] = 0.0;
    const float *p = a.src + (static_cast<size_t>(y) * a.width + first) * CH;
    for (int j = 0; j < n; ++j, p += CH) {
      const double w = __ldg(a.weights + static_cast<size_t>(j) * a.out_n + o);
      accumulate<CH>(acc, w, load_pixel<CH>(p));
    }
    float out[CH];
    finish<CH>(acc, out);
    store_pixel<CH>(a.dst + (static_cast<size_t>(y) * a.out_w + o) * CH, out);
  }
}


// ------------------------------------------------------------------------------------------
// Regular-pattern kernels: integer-ratio reductions (e.g. Lanczos 2x: every output draws N = 12
// consecutive source samples and the window advances by S = 2 per output).  A thread produces RO
// consecutive outputs from the K = S*(RO-1)+N source samples they share; each sample is loaded,
// converted to double and alpha-premultiplied ONCE and feeds every output whose window holds it
// (statically known => no window tests, fully unrolled).  Weights stay per-output (the reference's
// weights differ in the last bits from output to output): wreg[o][N], warp-uniform loads with
// immediate offsets.  Blocks that are not regular (image edges) take the generic gather path.
// ------------------------------------------------------------------------------------------
template <int CH, int S, int N, int RO>
__device__ __forceinline__ bool block_is_regular(const ResizeArgs &a, int o0, int limit) {
  if (o0 + RO > limit) return false;
  const int lo = __ldg(a.start + o0);
  bool regular = true;
#pragma unroll
  for (int r = 0; r < RO; ++r)
    regular = regular && (__ldg(a.start + o0 + r) == lo + S * r) && (__ldg(a.count + o0 + r) == N);
  return regular;
}

template <int CH>
__device__ __forceinline__ void to_premultiplied(const Pixel<CH> &px, double (&q)[CH]) {
#pragma unroll
  for (int c = 0; c < CH; ++c) q[c] = static_cast<double>(px.v[c]);
  if (CH == 2 || CH == 4) {
#pragma unroll
    for (int c = 0; c < CH - 1; ++c) q[c] *= q[CH - 1];
  }
}

// vertical: grid (ceil(width/128), ceil(out_h/RO))
template <int CH, int S, int N, int RO>
__global__ void __launch_bounds__(128) resize_vertical_regular_kernel(const ResizeArgs a, const double *__restrict__ wreg) {
  const int x = blockIdx.x * 128 + threadIdx.x;
  if (x >= a.width) return;
  const int o0 = blockIdx.y * RO;
  const size_t pitch = static_cast<size_t>(a.width) * CH;
  const float *col = a.src + static_cast<size_t>(x) * CH;
  if (!block_is_regular<CH, S, N, RO>(a, o0, a.out_h)) {         // warp-uniform: edge blocks
    for (int o = o0; o < min(o0 + RO, a.out_h); ++o) {
      const int first = __ldg(a.start + o), n = __ldg(a.count + o);
      if (n <= 0) continue;
      double acc[CH];
#pragma unroll
      for (int c = 0; c < CH; ++c) acc[c] = 0.0;
      const float *p = col + static_cast<size_t>(first) * pitch;
      for (int j = 0; j < n; ++j, p += pitch)
        accumulate<CH>(acc, __ldg(a.weights + static_cast<size_t>(j) * a.out_n + o), load_pixel<CH>(p));
      float out[CH];
      finish<CH>(acc, out);
      store_pixel<CH>(a.dst + (static_cast<size_t>(o) * a.out_w + x) * CH, out);
    }
    return;
  }
  constexpr int K = S * (RO - 1) + N;          // source rows shared by the RO outputs
  constexpr int PF = 8;                        // rows in flight
  const float *p = col + static_cast<size_t>(__ldg(a.start + o0)) * pitch;
  const double *wb = wreg + static_cast<size_t>(o0) * N;
  double acc[RO][CH];
#pragma unroll
  for (int r = 0; r < RO; ++r)
#pragma unroll
    for (int c = 0; c < CH; ++c) acc[r][c] = 0.0;
  Pixel<CH> pre[PF];
#pragma unroll
  for (int k = 0; k < PF && k < K; ++k) pre[k] = load_pixel<CH>(p + static_cast<size_t>(k) * pitch);
#pragma unroll
  for (int k = 0; k < K; ++k) {
    const Pixel<CH> px = pre[k % PF];
    if (k + PF < K) pre[k % PF] = load_pixel<CH>(p + static_cast<size_t>(k + PF) * pitch);
    double q[CH];
    to_premultiplied<CH>(px, q);
#pragma unroll
    for (int r = 0; r < RO; ++r) {
      const int j = k - S * r;                  // compile-time
      if (j >= 0 && j < N) {
        const double w = __ldg(wb + r * N + j);
#pragma unroll
        for (int c = 0; c < CH; ++c) acc[r][c] = fma(w, q[c], acc[r][c]);
      }
    }
  }
#pragma unroll
  for (int r = 0; r < RO; ++r) {
    float out[CH];
    finish<CH>(acc[r], out);
    store_pixel<CH>(a.dst + (static_cast<size_t>(o0 + r) * a.out_w + x) * CH, out);
  }
}

// horizontal: CTA = 4 warps, warp w -> outputs [ob + w*RO, +RO) of 32 rows (lane = row); the CTA's
// source span is staged in shared memory (odd pixel pitch => conflict-free lane-per-row LDS.128).
// grid (ceil(out_w/(4*RO)), ceil(height/32)); dynamic smem = 32*pitch*CH floats.
template <int CH, int S, int N, int RO>
__global__ void __launch_bounds__(128) resize_horizontal_regular_kernel(const ResizeArgs a, const double *__restrict__ wreg,
                                                                        int pitch) {
  extern __shared__ __align__(16) float tile[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ob = blockIdx.x * (4 * RO);
  const int ybase = blockIdx.y * 32;
  const int olast = min(ob + 4 * RO, a.out_w) - 1;
  const int tile_lo = __ldg(a.start + ob);
  const int span = min(__ldg(a.start + olast) + __ldg(a.count + olast) - tile_lo, pitch);
  for (int idx = threadIdx.x; idx < 32 * span; idx += 128) {
    const int r = idx / span, px = idx - r * span;
    const int yy = min(ybase + r, a.height - 1);
    const Pixel<CH> v = load_pixel<CH>(a.src + (static_cast<size_t>(yy) * a.width + tile_lo + px) * CH);
    float o[CH];
#pragma unroll
    for (int c = 0; c < CH; ++c) o[c] = v.v[c];
    store_pixel<CH>(tile + (static_cast<size_t>(r) * pitch + px) * CH, o);
  }
  __syncthreads();
  const int o0 = ob + warp * RO;
  const int y = ybase + lane;
  if (o0 >= a.out_w || y >= a.height) return;
  const float *trow = tile + static_cast<size_t>(lane) * pitch * CH;
  float *drow = a.dst + static_cast<size_t>(y) * a.out_w * CH;
  if (!block_is_regular<CH, S, N, RO>(a, o0, a.out_w)) {
    for (int o = o0; o < min(o0 + RO, a.out_w); ++o) {
      const int first = __ldg(a.start + o), n = __ldg(a.count + o);
      if (n <= 0) continue;
      double acc[CH];
#pragma unroll
      for (int c = 0; c < CH; ++c) acc[c] = 0.0;
      for (int j = 0; j < n; ++j) {
        Pixel<CH> px;
#pragma unroll
        for (int c = 0; c < CH; ++c) px.v[c] = trow[(first - tile_lo + j) * CH + c];
        accumulate<CH>(acc, __ldg(a.weights + static_cast<size_t>(j) * a.out_n + o), px);
      }
      float out[CH];
      finish<CH>(acc, out);
      store_pixel<CH>(drow + static_cast<size_t>(o) * CH, out);
    }
    return;
  }
  constexpr int K = S * (RO - 1) + N;
  const float *p = trow + static_cast<size_t>(__ldg(a.start + o0) - tile_lo) * CH;
  const double *wb = wreg + static_cast<size_t>(o0) * N;
  double acc[RO][CH];
#pragma unroll
  for (int r = 0; r < RO; ++r)
#pragma unroll
    for (int c = 0; c < CH; ++c) acc[r][c] = 0.0;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    Pixel<CH> px;
    if (CH == 4) {
      const float4 t = *reinterpret_cast<const float4 *>(p + k * 4);
      px.v[0] = t.x; px.v[1] = t.y; px.v[2] = t.z; px.v[CH - 1] = t.w;
    } else {
#pragma unroll
      for (int c = 0; c < CH; ++c) px.v[c] = p[k * CH + c];
    }
    double q[CH];
    to_premultiplied<CH>(px, q);
#pragma unroll
    for (int r = 0; r < RO; ++r) {
      const int j = k - S * r;
      if (j >= 0 && j < N) {
        const double w = __ldg(wb + r * N + j);
#pragma unroll
        for (int c = 0; c < CH; ++c) acc[r][c] = fma(w, q[c], acc[r][c]);
      }
    }
  }
#pragma unroll
  for (int r = 0; r < RO; ++r) {
    float out[CH];
    finish<CH>(acc[r], out);
    store_pixel<CH>(drow + static_cast<size_t>(o0 + r) * CH, out);
  }
}

template <int CH, int S, int N>
int launch_regular(const ResizeArgs &a, int axis, const double *wreg, int max_span, cudaStream_t s) {
  constexpr int kRO = 8;
  if (axis == 1) {
    dim3 grid((a.width + 127) / 128, (a.out_h + kRO - 1) / kRO);
    if (grid.y > 65535) return MB200_EUNSUPPORTED;
    resize_vertical_regular_kernel<CH, S, N, kRO><<<grid, 128, 0, s>>>(a, wreg);
  } else {
    const int pitch = max_span | 1;
    const size_t smem = static_cast<size_t>(32) * pitch * CH * sizeof(float);
    if (smem > 48 * 1024) return MB200_EUNSUPPORTED;
    dim3 grid((a.out_w + 4 * kRO - 1) / (4 * kRO), (a.height + 31) / 32);
    if (grid.y > 65535) return MB200_EUNSUPPORTED;
    resize_horizontal_regular_kernel<CH, S, N, kRO><<<grid, 128, smem, s>>>(a, wreg, pitch);
  }
  return MB200_OK;
}

template <int CH>
int launch_regular_ch(const ResizeArgs &a, int axis, int stride, int ntaps, const double *wreg, int max_span,
                      cudaStream_t s) {
  if (stride == 2 && ntaps == 12) return launch_regular<CH, 2, 12>(a, axis, wreg, max_span, s);   // 3-lobe, 2x
  if (stride == 2 && ntaps == 8) return launch_regular<CH, 2, 8>(a, axis, wreg, max_span, s);     // 2-lobe / cubic, 2x
  if (stride == 2 && ntaps == 4) return launch_regular<CH, 2, 4>(a, axis, wreg, max_span, s);     // triangle, 2x
  if (stride == 3 && ntaps == 18) return launch_regular<CH, 3, 18>(a, axis, wreg, max_span, s);
  if (stride == 4 && ntaps == 24) return launch_regular<CH, 4, 24>(a, axis, wreg, max_span, s);
  if (stride == 4 && ntaps == 16) return launch_regular<CH, 4, 16>(a, axis, wreg, max_span, s);
  return MB200_EUNSUPPORTED;
}

}  // namespace

int launch_resize_axis(const float *src, size_t width, size_t height, int channels, float *dst, int axis,
                       const ResizeAxis &t, bool regular, void *stream) {
  const size_t out_n = t.out_n;
  if (width == 0 || height == 0 || out_n == 0 || channels < 1 || channels > 4)
    return fail(MB200_EINVAL, "resize: bad geometry");
  if (width > 0x3fffffffull || height > 0x3fffffffull || out_n > 0x3fffffffull)
    return fail(MB200_EINVAL, "resize: image too large");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  ResizeArgs a{};
  a.src = src; a.dst = dst;
  a.width = static_cast<int>(width); a.height = static_cast<int>(height);
  a.out_n = static_cast<int>(out_n);
  a.start = t.d_start; a.count = t.d_count; a.weights = t.d_weights;
  a.lines_per_thread = 8;
  if (axis == 1) { a.out_w = a.width; a.out_h = a.out_n; }
  else { a.out_w = a.out_n; a.out_h = a.height; }
  a.o_begin = 0;
  a.o_end = a.out_n;
  if (regular && t.d_wreg != nullptr) {
    int rc = MB200_EUNSUPPORTED;
    switch (channels) {
      case 1: rc = launch_regular_ch<1>(a, axis, t.reg_stride, t.reg_taps, t.d_wreg, t.max_span, s); break;
      case 2: rc = launch_regular_ch<2>(a, axis, t.reg_stride, t.reg_taps, t.d_wreg, t.max_span, s); break;
      case 3: rc = launch_regular_ch<3>(a, axis, t.reg_stride, t.reg_taps, t.d_wreg, t.max_span, s); break;
      default: rc = launch_regular_ch<4>(a, axis, t.reg_stride, t.reg_taps, t.d_wreg, t.max_span, s); break;
    }
    if (rc == MB200_OK) {
      count_launch();
      count_family(kResizeRegular);
      const cudaError_t e = cudaGetLastError();
      if (e != cudaSuccess) return cuda_fail(e, "resize launch");
      return MB200_OK;
    }
  }
  if (axis == 1) {
    dim3 grid((a.width + 127) / 128, (a.out_n + a.lines_per_thread - 1) / a.lines_per_thread);
    if (grid.y > 65535) return fail(MB200_EINVAL, "resize: too many rows");
    switch (channels) {
      case 1: resize_vertical_kernel<1><<<grid, 128, 0, s>>>(a); break;
      case 2: resize_vertical_kernel<2><<<grid, 128, 0, s>>>(a); break;
      case 3: resize_vertical_kernel<3><<<grid, 128, 0, s>>>(a); break;
      default: resize_vertical_kernel<4><<<grid, 128, 0, s>>>(a); break;
    }
  } else {
    dim3 grid((a.out_n + 127) / 128, (a.height + a.lines_per_thread - 1) / a.lines_per_thread);
    if (grid.y > 65535) return fail(MB200_EINVAL, "resize: too many rows");
    switch (channels) {
      case 1: resize_horizontal_kernel<1><<<grid, 128, 0, s>>>(a); break;
      case 2: resize_horizontal_kernel<2><<<grid, 128, 0, s>>>(a); break;
      case 3: resize_horizontal_kernel<3><<<grid, 128, 0, s>>>(a); break;
      default: resize_horizontal_kernel<4><<<grid, 128, 0, s>>>(a); break;
    }
  }
  count_launch();
  count_family(kResizeGather);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "resize launch");
  return MB200_OK;
}

}  // namespace mb200
