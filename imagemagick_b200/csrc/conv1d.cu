// conv1d.cu -- one pass of a separable (1-D) convolution: the kernel behind
// BlurImage's two passes (MagickCore/effect.c:788 "blur:RxS;blur:RxS+90").
//
// Semantics follow MorphologyPrimitive's ConvolveMorphology for height-1 kernels (row
// path, MagickCore/morphology.c:2897-2979) and width-1 kernels (column fast path,
// :2654-2807): reflected taps, edge-clamped source (cache.c:2663), double accumulation,
// alpha-weighted blending of the colour channels when the image has alpha, result
// cast to float (quantum.h:88).
//
// GPU mapping.  The op is a memory-streaming stencil whose co-limit is the FP64 pipe
// (33 taps x 4 channels of double FMA per pixel for sigma=4).  Design:
//  * one thread per float component line; it walks along the filter axis keeping NT
//    rotating FP64 accumulators in registers, so every source sample is loaded and
//    converted to double ONCE and feeds NT FMAs whose tap operands are immediates in
//    the kernel-parameter constant bank (no tap loads, no shared-memory traffic per FMA);
//  * alpha weighting is done by premultiplying the sample once (q = A*p); the weight
//    sum gamma is exactly the alpha component's own accumulator, fetched with a warp
//    shuffle from the pixel's alpha lane -- 4 FMAs per tap per pixel instead of the
//    reference's 7 flops;
//  * column pass: lanes span 32 consecutive components of a row => every load/store
//    is one fully coalesced 128-byte line; a register ring keeps NT row loads in
//    flight per thread;
//  * row pass: a (rows x segment) tile is staged in shared memory with coalesced
//    float4 loads (odd pixel pitch => conflict-free LDS for the 8-rows x 4-channels
//    lane layout).
// No tensor cores: this is not a dense contraction.
#include "launch.cuh"
#include "conv_common.cuh"

#include <cuda_runtime.h>

#include <cstdint>
#include <cstdlib>
#include <type_traits>

namespace mb200 {
namespace {

template <int NT>
struct Taps { double k[NT]; };

struct Conv1dArgs {
  const float *src;
  float *dst;
  int width, height, channels;
  int rc;        // width * channels (floats per row)
  int off;       // samples before the output position covered by the window (ox / oy)
  int strip;     // outputs per thread along the filter axis
  int seg_w;     // row pass: source pixels staged per tile row (strip + NT - 1)
  int pitch;     // row pass: shared-memory tile pitch in pixels (odd)
  int ntaps;     // taps of the real window; the kernel template carries NT >= ntaps slots (taps[ntaps..NT) are zero)
  double bias;
  unsigned long long *changed;
  // fused UnsharpMaskImage epilogue (column pass of the pair kernels, EPI = 1): the source image of the operator,
  // gain and QuantumRange * threshold (effect.c:4299, :4358-4363)
  const float *aux;
  double gain, qthreshold;
};

// Per-thread constants of the output stage.  With sum' = sum K*(A*p) and gsum' = sum K*A the
// reference's  PerceptibleReciprocal(QS*gsum') * (bias + QS*sum')  (morphology.c:3197) equals
// (bias/QS + sum') / gsum'; alpha / plain lanes use a denominator of 1.
struct Finish {
  double bias_eff;   // bias (plain, alpha lane) or bias/QS (blend lane)
  bool blend;
};

// out = (bias_eff + sum) * 1/den, den = blend ? gsum : 1, with the reference's |gamma| < MagickEpsilon clamp
// (PerceptibleReciprocal == 1/clamp(gamma)).
__device__ __forceinline__ float finish(const Finish &f, double sum, double gsum) {
  const double pixel = f.bias_eff + sum;
  const double den = clamp_denominator(f.blend ? gsum : 1.0);
  return static_cast<float>(fast_reciprocal(den) * pixel);
}

template <int NT> struct Ring { static constexpr int value = NT; };
template <> struct Ring<25> { static constexpr int value = 5; };
template <> struct Ring<33> { static constexpr int value = 11; };
template <> struct Ring<49> { static constexpr int value = 7; };
template <> struct Ring<65> { static constexpr int value = 13; };

// ---------------------------------------------------------------- column pass
// grid: (ceil(rc / THREADS), ceil(height / strip)); one thread per component column.
// strip + NT - 1 is a whole number of NT-step rotations, so the unrolled body has no exits.
template <int NT, int MODE, int THREADS, int MINB>
__global__ void __launch_bounds__(THREADS, MINB) conv_col_kernel(const Conv1dArgs a, const Taps<NT> taps) {
  constexpr int PF = Ring<NT>::value;          // source rows kept in flight per thread
  static_assert(NT % PF == 0, "ring must divide the rotation");
  const int col_raw = blockIdx.x * THREADS + threadIdx.x;
  const bool active = col_raw < a.rc;
  const int col = active ? col_raw : a.rc - 1;
  const int lane = threadIdx.x & 31;
  const int alane = MODE ? (lane | (MODE - 1)) : lane;
  const bool is_alpha = MODE ? ((col % MODE) == MODE - 1) : false;
  const int y0 = blockIdx.y * a.strip;
  const int nout = active ? min(a.strip, a.height - y0) : 0;
  const int total = a.strip + NT - 1;
  const int hmax = a.height - 1;
  const unsigned pitch_bytes = static_cast<unsigned>(a.rc) * 4u;
  const char *base = reinterpret_cast<const char *>(a.src + col);
  char *outp = reinterpret_cast<char *>(a.dst + col) + static_cast<size_t>(y0) * pitch_bytes;
  Finish fin;
  fin.blend = MODE && !is_alpha;
  fin.bias_eff = fin.blend ? a.bias * 65535.0 : a.bias;

  double acc[NT];
  float pre[PF];
#pragma unroll
  for (int q = 0; q < NT; ++q) acc[q] = 0.0;
  int ysrc = y0 - a.off;                       // source row of step 0
#pragma unroll
  for (int s = 0; s < PF; ++s) {
    const unsigned yy = static_cast<unsigned>(min(max(ysrc + s, 0), hmax));
    pre[s] = __ldg(reinterpret_cast<const float *>(base + static_cast<size_t>(yy) * pitch_bytes));
  }
  ysrc += PF;                                  // next row to fetch

  int j = -(NT - 1);                           // output row (relative to y0) finished at this step
  // The rotation is unrolled PF steps at a time (not NT): after each block the accumulators are
  // physically rotated by PF slots, so the static tap pattern repeats and the loop body stays
  // small enough for the instruction cache (NT*NT FMAs would not).
#pragma unroll 1
  for (int mb = 0; mb < total; mb += PF) {
#pragma unroll
    for (int s = 0; s < PF; ++s) {
      float vf = pre[s];
      {  // refill this ring slot with the row PF steps ahead (edge-clamped)
        const unsigned yy = static_cast<unsigned>(min(max(ysrc, 0), hmax));
        pre[s] = __ldg(reinterpret_cast<const float *>(base + static_cast<size_t>(yy) * pitch_bytes));
        ++ysrc;
      }
      double v = static_cast<double>(vf);
      if (MODE) {
        float af = __shfl_sync(0xffffffffu, vf, alane);
        af = is_alpha ? 1.0f : af;
        v *= static_cast<double>(af);
      }
      if (a.ntaps != NT && __any_sync(0xffffffffu, nonfinite_bits(vf))) {     // padded taps must not touch it
#pragma unroll
        for (int q = 0; q < NT; ++q)
          if ((s - q + NT) % NT < a.ntaps) acc[q] = fma(taps.k[(s - q + NT) % NT], v, acc[q]);
      } else {
#pragma unroll
        for (int q = 0; q < NT; ++q) acc[q] = fma(taps.k[(s - q + NT) % NT], v, acc[q]);
      }
      const int qf = (s + 1) % NT;
      const double sum = acc[qf];
      acc[qf] = 0.0;
      double gsum = 1.0;
      if (MODE) gsum = shfl_double(sum, alane);
      const float out = finish(fin, sum, gsum);
      if (static_cast<unsigned>(j) < static_cast<unsigned>(nout)) *reinterpret_cast<float *>(outp) = out;
      if (j >= 0) outp += pitch_bytes;
      ++j;
    }
    if (PF != NT) {                              // rotate: new acc[q] = old acc[(q + PF) % NT]
      double tmp[PF];
#pragma unroll
      for (int q = 0; q < PF; ++q) tmp[q] = acc[q];
#pragma unroll
      for (int q = 0; q < NT - PF; ++q) acc[q] = acc[q + PF];
#pragma unroll
      for (int q = 0; q < PF; ++q) acc[NT - PF + q] = tmp[q];
    }
  }
}

// ------------------------------------------------------------------- row pass
// block: 128 threads = 4 warps; a warp covers RPW = 32/channels rows x channels lanes.
// grid: (ceil(width / strip), ceil(height / rows_per_cta)).
template <int NT, int MODE, int MINB>
__global__ void __launch_bounds__(128, MINB) conv_row_kernel(const Conv1dArgs a, const Taps<NT> taps) {
  extern __shared__ __align__(16) float tile[];
  const int ch = a.channels;
  const int rpw = 32 / ch;
  const int rows_per_cta = 4 * rpw;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int x0 = blockIdx.x * a.strip;
  const int ybase = blockIdx.y * rows_per_cta;
  const int total = a.strip + NT - 1;
  const int wmax = a.width - 1, hmax = a.height - 1;

  // ---- stage the tile: rows_per_cta x total source pixels, x edge-clamped (whole pixels when they are 16-byte aligned;
  // the matrix and pair kernels decline unaligned sources and leave them to this kernel)
  if (ch == 4 && (reinterpret_cast<uintptr_t>(a.src) & 15) == 0) {
    const int n = rows_per_cta * total;
    for (int idx = threadIdx.x; idx < n; idx += 128) {
      const int r = idx / total, px = idx - r * total;
      const int yy = min(ybase + r, hmax);
      const int xx = min(max(x0 + px - a.off, 0), wmax);
      const float4 v = __ldg(reinterpret_cast<const float4 *>(a.src) + (static_cast<size_t>(yy) * a.width + xx));
      *reinterpret_cast<float4 *>(tile + (static_cast<size_t>(r) * a.pitch + px) * 4) = v;
    }
  } else {
    const int n = rows_per_cta * total * ch;
    const int rowf = total * ch;
    for (int idx = threadIdx.x; idx < n; idx += 128) {
      const int r = idx / rowf, e = idx - r * rowf;
      const int px = e / ch, c = e - px * ch;
      const int yy = min(ybase + r, hmax);
      const int xx = min(max(x0 + px - a.off, 0), wmax);
      tile[(static_cast<size_t>(r) * a.pitch + px) * ch + c] =
          __ldg(a.src + (static_cast<size_t>(yy) * a.width + xx) * ch + c);
    }
  }
  __syncthreads();

  const bool lane_ok = lane < rpw * ch;
  const int lr = lane_ok ? lane / ch : 0, c = lane_ok ? lane % ch : 0;
  const int r = warp * rpw + lr;
  const int y = ybase + r;
  const bool active = lane_ok && y < a.height;
  const int nout = active ? min(a.strip, a.width - x0) : 0;
  const int alane = MODE ? (lane | (MODE - 1)) : lane;
  const bool is_alpha = MODE ? (c == MODE - 1) : false;
  const float *tp = tile + static_cast<size_t>(r) * a.pitch * ch + c;
  float *outp = a.dst + (static_cast<size_t>(min(y, hmax)) * a.width + x0) * ch + c;
  Finish fin;
  fin.blend = MODE && !is_alpha;
  fin.bias_eff = fin.blend ? a.bias * 65535.0 : a.bias;

  double acc[NT];
#pragma unroll
  for (int q = 0; q < NT; ++q) acc[q] = 0.0;

  int j = -(NT - 1);
  constexpr int BLK = Ring<NT>::value;         // unrolled steps per block; accumulators rotate by BLK after it
#pragma unroll 1
  for (int mb = 0; mb < total; mb += BLK) {
#pragma unroll
    for (int s = 0; s < BLK; ++s) {
      const float vf = *tp;
      tp += ch;
      double v = static_cast<double>(vf);
      if (MODE) {
        float af = __shfl_sync(0xffffffffu, vf, alane);
        af = is_alpha ? 1.0f : af;
        v *= static_cast<double>(af);
      }
      if (a.ntaps != NT && __any_sync(0xffffffffu, nonfinite_bits(vf))) {     // padded taps must not touch it
#pragma unroll
        for (int q = 0; q < NT; ++q)
          if ((s - q + NT) % NT < a.ntaps) acc[q] = fma(taps.k[(s - q + NT) % NT], v, acc[q]);
      } else {
#pragma unroll
        for (int q = 0; q < NT; ++q) acc[q] = fma(taps.k[(s - q + NT) % NT], v, acc[q]);
      }
      const int qf = (s + 1) % NT;
      const double sum = acc[qf];
      acc[qf] = 0.0;
      double gsum = 1.0;
      if (MODE) gsum = shfl_double(sum, alane);
      const float out = finish(fin, sum, gsum);
      if (static_cast<unsigned>(j) < static_cast<unsigned>(nout)) *outp = out;
      if (j >= 0) outp += ch;
      ++j;
    }
    if (BLK != NT) {                             // rotate: new acc[q] = old acc[(q + BLK) % NT]
      double tmp[BLK];
#pragma unroll
      for (int q = 0; q < BLK; ++q) tmp[q] = acc[q];
#pragma unroll
      for (int q = 0; q < NT - BLK; ++q) acc[q] = acc[q + BLK];
#pragma unroll
      for (int q = 0; q < BLK; ++q) acc[NT - BLK + q] = tmp[q];
    }
  }
}

// ======================================================================================
// Two-components-per-thread kernels for RGBA ("pair" kernels, the default for 4 channels).
// A thread owns two adjacent components of a pixel -- (R,G) on even lanes, (B,A) on odd lanes --
// and therefore two independent rotations of NT accumulators.  Per pair of outputs this halves the
// per-step overhead the single-component kernels pay (one 64-bit load/store, one alpha shuffle,
// one reciprocal, three instead of four conversions), which matters because every half-rate
// FP64 / quarter-rate conversion instruction costs issue time (tools/micro/mix.cu).
// ======================================================================================

// Output stage of a pair: r = 1/clamp(den) (PerceptibleReciprocal on QS*den, morphology.c:3197),
// colour components are scaled by r, the alpha component (odd lane, .y) is stored unscaled.
__device__ __forceinline__ float2 finish_pair(bool odd, double sum0, double sum1, double gsum) {
  const double r = fast_reciprocal(clamp_denominator(gsum));
  const double m1 = odd ? 1.0 : r;              // the alpha component (odd lane, .y) is stored unscaled
  return make_float2(static_cast<float>(sum0 * r), static_cast<float>(sum1 * m1));
}

// ---- pair stream kernel, both axes.  A thread owns one component pair and walks along the
//      filter axis with a register ring of PF samples in flight.
//      AXIS 1 (column pass): CTA = 128 threads = 256 consecutive components of a row (1 KB, fully
//        coalesced); step = one row.          grid (ceil(rc/256), ceil(height/strip))
//      AXIS 0 (row pass):    CTA = 128 threads = 64 rows x 2 pairs; step = one pixel (16 B); a
//        lane pair reads the 16 B of its pixel, consecutive steps of a lane fall in the same 128-B
//        line (L1-resident), so no shared-memory staging or barrier is needed.
//                                              grid (ceil(width/strip), ceil(height/64))
// IO selects the element types: 0 = float Quantum in, float Quantum out (one full pass);
// 1 = float in, RAW double sums out (first half of a rank-1 2-D kernel: no normalisation, no rounding);
// 2 = raw double sums in, float Quantum out (second half).  With IO 1 + 2 a separable 2-D kernel
// (e.g. "gaussian:RxS") is evaluated with kw + kh instead of kw * kh taps per sample while keeping the
// intermediate in double, i.e. without the float rounding a two-kernel list would introduce.
// PADDED: the launch carries fewer real taps than NT slots (see nonfinite_bits above).  EPI = 1: UnsharpMaskImage's
// point pass fused into the output stage (AXIS 1, IO 0 only).
template <int NT, int MINB, int AXIS, int IO, bool L2PF = false, bool PADDED = false, int EPI = 0>
__global__ void __launch_bounds__(128, MINB) conv_pair_kernel(const Conv1dArgs a, const Taps<NT> taps) {
  static_assert(EPI == 0 || (AXIS == 1 && IO == 0), "the fused epilogue belongs to the final column pass");
  constexpr int PF = Ring<NT>::value;
  constexpr unsigned kInB = (IO == 2) ? 8u : 4u, kOutB = (IO == 1) ? 8u : 4u;   // bytes per component
  using InT = typename std::conditional<IO == 2, double2, float2>::type;
  const int lane = threadIdx.x & 31;
  const bool odd = (threadIdx.x & 1) != 0;
  const int alpha_lane = lane | 1;
  const unsigned in_pitch = static_cast<unsigned>(a.rc) * kInB, out_pitch = static_cast<unsigned>(a.rc) * kOutB;
  int first, nout, limit;                 // first output / number of outputs / clamp limit along the axis
  const char *base;                       // address of sample 0 of this thread's line
  char *outp;
  unsigned step, ostep;                   // bytes between consecutive samples (input / output)
  if (AXIS == 1) {
    const int npairs = a.rc >> 1;
    const int pair_raw = blockIdx.x * 128 + threadIdx.x;
    const bool active = pair_raw < npairs;
    const int pair = active ? pair_raw : npairs - 1;
    first = blockIdx.y * a.strip;
    nout = active ? min(a.strip, a.height - first) : 0;
    limit = a.height - 1;
    step = in_pitch;
    ostep = out_pitch;
    base = reinterpret_cast<const char *>(a.src) + static_cast<size_t>(pair) * (2 * kInB);
    outp = reinterpret_cast<char *>(a.dst) + static_cast<size_t>(pair) * (2 * kOutB) + static_cast<size_t>(first) * out_pitch;
  } else {
    const int row_raw = blockIdx.y * 64 + (threadIdx.x >> 1);
    const bool active = row_raw < a.height;
    const int row = active ? row_raw : a.height - 1;
    first = blockIdx.x * a.strip;
    nout = active ? min(a.strip, a.width - first) : 0;
    limit = a.width - 1;
    step = 4 * kInB;
    ostep = 4 * kOutB;
    base = reinterpret_cast<const char *>(a.src) + static_cast<size_t>(row) * in_pitch + (odd ? 2 * kInB : 0);
    outp = reinterpret_cast<char *>(a.dst) + static_cast<size_t>(row) * out_pitch + (odd ? 2 * kOutB : 0) +
           static_cast<size_t>(first) * ostep;
  }
  const int total = a.strip + NT - 1;

  double acc0[NT], acc1[NT];
  InT pre[PF];
#pragma unroll
  for (int q = 0; q < NT; ++q) { acc0[q] = 0.0; acc1[q] = 0.0; }
  const int isrc0 = first - a.off;          // source index of step 0
#pragma unroll
  for (int s = 0; s < PF; ++s) {
    const unsigned ii = static_cast<unsigned>(min(max(isrc0 + s, 0), limit));
    pre[s] = __ldg(reinterpret_cast<const InT *>(base + static_cast<size_t>(ii) * step));
  }

  // EPI: the operator's source pixel of every output, fetched PF steps ahead of the step that needs it (a load issued
  // in the output stage itself would expose a DRAM round trip per step: measured 2x on the whole operator).
  float2 epi[EPI ? PF : 1];
  const char *epi_base = nullptr;
  if (EPI == 1) {
    epi_base = reinterpret_cast<const char *>(a.aux) + (outp - reinterpret_cast<char *>(a.dst)) -
               static_cast<size_t>(first) * ostep;       // element (row 0) of this thread's column pair
#pragma unroll
    for (int s = 0; s < PF; ++s) {
      const unsigned r = static_cast<unsigned>(min(max(first - (NT - 1) + s, 0), limit));
      epi[s] = __ldg(reinterpret_cast<const float2 *>(epi_base + static_cast<size_t>(r) * ostep));
    }
  }
  // The SASS of this loop issues ~50 non-FP64 instructions per step next to 70 DFMA + 4 DMUL, so with two warps per
  // scheduler the ISSUE slots, not the FP64 pipe alone, bound it.  A variant with an unclamped interior loop needed 255
  // registers (two loop bodies) and was slower; the FP64 mma.sync formulation of conv_mma.cu cuts the issue count 8x.
  int isrc = isrc0 + PF;
  int j = -(NT - 1);
#pragma unroll 1
  for (int mb = 0; mb < total; mb += PF) {       // PF unrolled steps, then rotate the accumulators by PF
#pragma unroll
    for (int s = 0; s < PF; ++s) {
      const InT vf = pre[s];
      {
        const unsigned ii = static_cast<unsigned>(min(max(isrc, 0), limit));
        pre[s] = __ldg(reinterpret_cast<const InT *>(base + static_cast<size_t>(ii) * step));
        if (L2PF) {             // L2 prefetch far ahead: the ring's LDGs then complete at L2 latency
          const unsigned ip = static_cast<unsigned>(min(isrc + a.seg_w, limit));
          asm volatile("prefetch.global.L2 [%0];" ::"l"(base + static_cast<size_t>(ip) * step));
        }
        ++isrc;
      }
      // (premultiplying one step ahead, as the cp.async kernel does, costs this kernel 5 %: 220 registers)
      double v0, v1;
      if (IO == 2) {
        v0 = vf.x; v1 = vf.y;                       // already premultiplied sums
      } else {
        const float af = __shfl_sync(0xffffffffu, static_cast<float>(vf.y), alpha_lane);
        const double da = static_cast<double>(af);
        v0 = static_cast<double>(vf.x) * da;
        v1 = static_cast<double>(vf.y) * (odd ? 1.0 : da);
      }
      if (PADDED && __any_sync(0xffffffffu, nonfinite_bits(vf.x) || nonfinite_bits(vf.y))) {
#pragma unroll
        for (int q = 0; q < NT; ++q) {
          if ((s - q + NT) % NT < a.ntaps) {
            const double k = taps.k[(s - q + NT) % NT];
            acc0[q] = fma(k, v0, acc0[q]);
            acc1[q] = fma(k, v1, acc1[q]);
          }
        }
      } else {
#pragma unroll
        for (int q = 0; q < NT; ++q) {
          const double k = taps.k[(s - q + NT) % NT];
          acc0[q] = fma(k, v0, acc0[q]);
          acc1[q] = fma(k, v1, acc1[q]);
        }
      }
      const int qf = (s + 1) % NT;
      const double sum0 = acc0[qf], sum1 = acc1[qf];
      acc0[qf] = 0.0;
      acc1[qf] = 0.0;
      if (IO == 1) {
        if (static_cast<unsigned>(j) < static_cast<unsigned>(nout)) *reinterpret_cast<double2 *>(outp) = make_double2(sum0, sum1);
      } else {
        const double gsum = shfl_double(sum1, alpha_lane);
        float2 out = finish_pair(odd, sum0, sum1, gsum);
        if (EPI == 1) {            // source pixel of output j (prefetched), then refill the slot for output j + PF
          const float2 p = epi[s];
          const unsigned r = static_cast<unsigned>(min(max(first + j + PF, 0), limit));
          epi[s] = __ldg(reinterpret_cast<const float2 *>(epi_base + static_cast<size_t>(r) * ostep));
          out.x = unsharp_point(p.x, out.x, a.gain, a.qthreshold);
          out.y = unsharp_point(p.y, out.y, a.gain, a.qthreshold);
        }
        if (static_cast<unsigned>(j) < static_cast<unsigned>(nout)) *reinterpret_cast<float2 *>(outp) = out;
      }
      if (j >= 0) outp += ostep;
      ++j;
    }
    if (PF != NT) {
      double t0[PF], t1[PF];
#pragma unroll
      for (int q = 0; q < PF; ++q) { t0[q] = acc0[q]; t1[q] = acc1[q]; }
#pragma unroll
      for (int q = 0; q < NT - PF; ++q) { acc0[q] = acc0[q + PF]; acc1[q] = acc1[q + PF]; }
#pragma unroll
      for (int q = 0; q < PF; ++q) { acc0[NT - PF + q] = t0[q]; acc1[NT - PF + q] = t1[q]; }
    }
  }
}

// ---- pair stream kernel with a shared-memory prefetch ring (cp.async / LDGSTS), both axes.
// Same arithmetic and thread mapping as conv_pair_kernel; only the way source samples reach the
// thread differs.  With the register ring every in-flight LDG needs one of the six hardware
// scoreboards, which it has to share with the F2F / SHFL / MUFU results of the output stage: ncu
// showed 13 % (column) / 30 % (row) of all stall samples on output STGs that were waiting, through
// such a shared scoreboard, for an unrelated prefetch issued a few hundred cycles earlier.  cp.async
// groups are counted separately (DEPBAR.LE), cost no registers, and the ring depth is no longer tied
// to the rotation length.
//   AXIS 1: per-warp ring of NS rows x 256 B; a lane copies and later reads its own 8 bytes (no
//           cross-lane hazard, no barrier); LDS issued one step ahead.
//   AXIS 0: per-warp ring of 8-pixel chunks of its 16 rows (full 128-B line requests, 144-B row pitch
//           => conflict-free LDS.64); edge replication is applied by the loader.
template <int NT, int MINB, int AXIS, int IO, bool PADDED = false, int EPI = 0>
__global__ void __launch_bounds__(128, MINB) conv_pair_async_kernel(const Conv1dArgs a, const Taps<NT> taps) {
  static_assert(IO == 0 || IO == 1, "float input only");
  static_assert(EPI == 0 || (AXIS == 1 && IO == 0), "the fused epilogue belongs to the final column pass");
  // The asm statements below are volatile (ordered among themselves: copy -> commit -> wait -> LDS) but
  // carry no "memory" clobber: the ring is touched by nothing else, and the output STGs must stay free
  // to sink below the next step's copies (otherwise every step exposes the F2F -> STG latency).
  constexpr int UN = Ring<NT>::value;
  constexpr unsigned kOutB = (IO == 1) ? 8u : 4u;
  constexpr int NS = 16;                              // AXIS 1: rows in the ring
  constexpr int NC = 4, kPitch = 144, kSlot = 16 * kPitch;   // AXIS 0: chunk slots
  constexpr int kWarpBytes = AXIS == 1 ? NS * 256 : NC * kSlot;
  __shared__ __align__(128) unsigned char ring_all[4 * kWarpBytes];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool odd = (lane & 1) != 0;
  const int alpha_lane = lane | 1;
  const unsigned ring_s = static_cast<unsigned>(__cvta_generic_to_shared(ring_all + warp * kWarpBytes));
  const unsigned in_pitch = static_cast<unsigned>(a.rc) * 4u, out_pitch = static_cast<unsigned>(a.rc) * kOutB;
  int first, nout;
  char *outp;
  unsigned ostep;
  const int total = a.strip + NT - 1;

  // ---- loader state
  const char *lbase;            // AXIS 1: this lane's column; AXIS 0: image base
  int limit, isrc0;
  unsigned rd;                  // shared-memory address of this lane's next sample
  int chunk = 0, px_in = 0, c0 = 0, nchunks = 0, lrow0 = 0;
  if (AXIS == 1) {
    const int npairs = a.rc >> 1;
    const int pair_raw = blockIdx.x * 128 + threadIdx.x;
    const bool active = pair_raw < npairs;
    const int pair = active ? pair_raw : npairs - 1;
    first = blockIdx.y * a.strip;
    nout = active ? min(a.strip, a.height - first) : 0;
    limit = a.height - 1;
    ostep = out_pitch;
    lbase = reinterpret_cast<const char *>(a.src) + static_cast<size_t>(pair) * 8;
    outp = reinterpret_cast<char *>(a.dst) + static_cast<size_t>(pair) * (2 * kOutB) + static_cast<size_t>(first) * out_pitch;
    isrc0 = first - a.off;
    rd = ring_s + lane * 8;
  } else {
    const int row_raw = blockIdx.y * 64 + (threadIdx.x >> 1);
    const bool active = row_raw < a.height;
    first = blockIdx.x * a.strip;
    nout = active ? min(a.strip, a.width - first) : 0;
    limit = a.width - 1;
    ostep = 4 * kOutB;
    lbase = reinterpret_cast<const char *>(a.src);
    outp = reinterpret_cast<char *>(a.dst) + static_cast<size_t>(active ? row_raw : 0) * out_pitch + (odd ? 2 * kOutB : 0) +
           static_cast<size_t>(first) * ostep;
    isrc0 = first - a.off;
    c0 = isrc0 >= 0 ? isrc0 / 8 : -((7 - isrc0) / 8);            // floor(isrc0 / 8)
    px_in = isrc0 - 8 * c0;
    nchunks = (px_in + ((total + UN - 1) / UN) * UN + 7) / 8;
    lrow0 = blockIdx.y * 64 + warp * 16;
    rd = ring_s + (lane >> 1) * kPitch + (odd ? 8 : 0) + px_in * 16;
  }
  // AXIS 1: one row (step k) per group; AXIS 0: one 8-pixel chunk of the warp's 16 rows per group
  auto issue = [&](int k) {
    if (AXIS == 1) {
      const unsigned ii = static_cast<unsigned>(min(max(isrc0 + k, 0), limit));
      const unsigned dst = ring_s + static_cast<unsigned>(k & (NS - 1)) * 256u + lane * 8;
      asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(dst), "l"(lbase + static_cast<size_t>(ii) * in_pitch));
    } else if (k < nchunks) {
      const int x = min(max((c0 + k) * 8 + (lane & 7), 0), limit);
      const unsigned slot = ring_s + static_cast<unsigned>(k & (NC - 1)) * kSlot;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int r = 4 * i + (lane >> 3);
        const int y = min(lrow0 + r, a.height - 1);
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(slot + r * kPitch + (lane & 7) * 16),
                     "l"(lbase + static_cast<size_t>(y) * in_pitch + static_cast<size_t>(x) * 16));
      }
    }
    asm volatile("cp.async.commit_group;" );
  };
  constexpr int kAhead = AXIS == 1 ? NS - 1 : NC;    // groups issued before the loop
#pragma unroll
  for (int k = 0; k < kAhead; ++k) issue(k);

  double acc0[NT], acc1[NT];
#pragma unroll
  for (int q = 0; q < NT; ++q) { acc0[q] = 0.0; acc1[q] = 0.0; }
  float2 vnext;
  if (AXIS == 1) asm volatile("cp.async.wait_group %0;" ::"n"(NS - 2));
  else { asm volatile("cp.async.wait_group %0;" ::"n"(NC - 1)); __syncwarp(); }
  asm volatile("ld.shared.v2.f32 {%0,%1}, [%2];" : "=f"(vnext.x), "=f"(vnext.y) : "r"(rd));
  double nv0, nv1;                                 // premultiplied sample of the next step
  bool nbad = false;                               // ... and whether any lane's sample of that step is non-finite
  {
    const float af = __shfl_sync(0xffffffffu, vnext.y, alpha_lane);
    const double da = static_cast<double>(af);
    nv0 = static_cast<double>(vnext.x) * da;
    nv1 = static_cast<double>(vnext.y) * (odd ? 1.0 : da);
    if (PADDED) nbad = __any_sync(0xffffffffu, nonfinite_bits(vnext.x) || nonfinite_bits(vnext.y));
  }

  int j = -(NT - 1);
  int step = 0;
  float2 epi[EPI ? UN : 1];                      // see conv_pair_kernel
  const char *epi_base = nullptr;
  if (EPI == 1) {
    epi_base = reinterpret_cast<const char *>(a.aux) + (outp - reinterpret_cast<char *>(a.dst)) -
               static_cast<size_t>(first) * ostep;
#pragma unroll
    for (int s = 0; s < UN; ++s) {
      const unsigned r = static_cast<unsigned>(min(max(first + j + s, 0), limit));
      epi[s] = __ldg(reinterpret_cast<const float2 *>(epi_base + static_cast<size_t>(r) * ostep));
    }
  }
#pragma unroll 1
  for (int mb = 0; mb < total; mb += UN) {       // UN unrolled steps, then rotate the accumulators by UN
#pragma unroll
    for (int s = 0; s < UN; ++s) {
      const double v0 = nv0, v1 = nv1;
      const bool bad = nbad;
      // fetch the next step's sample and keep the ring full
      if (AXIS == 1) {
        asm volatile("cp.async.wait_group %0;" ::"n"(NS - 3));      // row step+1 has landed
        rd = ring_s + static_cast<unsigned>((step + 1) & (NS - 1)) * 256u + lane * 8;
        asm volatile("ld.shared.v2.f32 {%0,%1}, [%2];" : "=f"(vnext.x), "=f"(vnext.y) : "r"(rd));
        issue(step + NS - 1);                                                  // into the slot read at step-1
      } else {
        rd += 16;
        if (++px_in == 8) {                        // warp-uniform: chunk exhausted
          px_in = 0;
          __syncwarp();
          issue(chunk + NC);
          ++chunk;
          asm volatile("cp.async.wait_group %0;" ::"n"(NC - 1));
          __syncwarp();
          rd = ring_s + static_cast<unsigned>(chunk & (NC - 1)) * kSlot + (lane >> 1) * kPitch + (odd ? 8 : 0);
        }
        asm volatile("ld.shared.v2.f32 {%0,%1}, [%2];" : "=f"(vnext.x), "=f"(vnext.y) : "r"(rd));
      }
      ++step;
      {                                            // next step's SHFL -> F2F -> DMUL chain, under this step's FMAs
        const float af = __shfl_sync(0xffffffffu, vnext.y, alpha_lane);
        const double da = static_cast<double>(af);
        nv0 = static_cast<double>(vnext.x) * da;
        nv1 = static_cast<double>(vnext.y) * (odd ? 1.0 : da);
        if (PADDED) nbad = __any_sync(0xffffffffu, nonfinite_bits(vnext.x) || nonfinite_bits(vnext.y));
      }
      if (PADDED && bad) {
#pragma unroll
        for (int q = 0; q < NT; ++q) {
          const int t = (s - q + NT) % NT;
          if (t == 0) { acc0[q] = taps.k[0] * v0; acc1[q] = taps.k[0] * v1; }
          else if (t < a.ntaps) { acc0[q] = fma(taps.k[t], v0, acc0[q]); acc1[q] = fma(taps.k[t], v1, acc1[q]); }
        }
      } else {
#pragma unroll
        for (int q = 0; q < NT; ++q) {
          const int t = (s - q + NT) % NT;
          const double k = taps.k[t];
          if (t == 0) { acc0[q] = k * v0; acc1[q] = k * v1; }          // first tap of a new output: no zeroing needed
          else { acc0[q] = fma(k, v0, acc0[q]); acc1[q] = fma(k, v1, acc1[q]); }
        }
      }
      const int qf = (s + 1) % NT;                 // this slot has just received its last tap
      const double sum0 = acc0[qf], sum1 = acc1[qf];
      if (IO == 1) {
        if (static_cast<unsigned>(j) < static_cast<unsigned>(nout)) *reinterpret_cast<double2 *>(outp) = make_double2(sum0, sum1);
      } else {
        const double gsum = shfl_double(sum1, alpha_lane);
        float2 out = finish_pair(odd, sum0, sum1, gsum);
        if (EPI == 1) {
          const float2 p = epi[s];
          const unsigned r = static_cast<unsigned>(min(max(first + j + UN, 0), limit));
          epi[s] = __ldg(reinterpret_cast<const float2 *>(epi_base + static_cast<size_t>(r) * ostep));
          out.x = unsharp_point(p.x, out.x, a.gain, a.qthreshold);
          out.y = unsharp_point(p.y, out.y, a.gain, a.qthreshold);
        }
        if (static_cast<unsigned>(j) < static_cast<unsigned>(nout)) *reinterpret_cast<float2 *>(outp) = out;
      }
      if (j >= 0) outp += ostep;
      ++j;
    }
    if (UN != NT) {
      double t0[UN], t1[UN];
#pragma unroll
      for (int q = 0; q < UN; ++q) { t0[q] = acc0[q]; t1[q] = acc1[q]; }
#pragma unroll
      for (int q = 0; q < NT - UN; ++q) { acc0[q] = acc0[q + UN]; acc1[q] = acc1[q + UN]; }
#pragma unroll
      for (int q = 0; q < UN; ++q) { acc0[NT - UN + q] = t0[q]; acc1[NT - UN + q] = t1[q]; }
    }
  }
  asm volatile("cp.async.wait_group 0;" );
}

// The RGBA pair kernels of one pass.  PADDED / EPI select the instantiation; everything else is the r01 choice.  Returns
// the family of the kernel it launched, or kLaunchFamilies when the grid does not fit (nothing launched).
// (3 CTAs per SM for the NT = 33 cp.async kernels -- __launch_bounds__(128, 3), 168 registers, spills -- were slower than
//  2: the third warp per scheduler does not pay for the spilled accumulators.)
template <int NT, bool PADDED>
LaunchFamily launch_pair(const Conv1dArgs &a, const Taps<NT> &taps, int axis, int io, bool fuse_unsharp,
                         const TuningKnobs &t, cudaStream_t stream) {
  if (axis == 1) {
    dim3 grid((a.rc / 2 + 127) / 128, (a.height + a.strip - 1) / a.strip);
    if (grid.y > 65535) return kLaunchFamilies;
    // NT = 33 is FP64-bound: the register-ring kernel (+ L2 prefetch) wins; shorter windows are closer to
    // the HBM roof and gain from the cp.async ring (sigma=2: 1.36 -> 1.22 ms for the whole blur).
    const bool async = (t.pair_async_col < 0 ? NT < 33 : t.pair_async_col != 0) && t.pair_async != 0;
    if (io == 2) conv_pair_kernel<NT, 2, 1, 2, false, PADDED><<<grid, 128, 0, stream>>>(a, taps);
    else if (io == 1 && async) conv_pair_async_kernel<NT, 2, 1, 1, PADDED><<<grid, 128, 0, stream>>>(a, taps);
    else if (io == 1) conv_pair_kernel<NT, 2, 1, 1, NT == 33, PADDED><<<grid, 128, 0, stream>>>(a, taps);
    else if (fuse_unsharp && async) conv_pair_async_kernel<NT, 2, 1, 0, PADDED, 1><<<grid, 128, 0, stream>>>(a, taps);
    else if (fuse_unsharp) conv_pair_kernel<NT, 2, 1, 0, NT == 33, PADDED, 1><<<grid, 128, 0, stream>>>(a, taps);
    else if (async) conv_pair_async_kernel<NT, 2, 1, 0, PADDED><<<grid, 128, 0, stream>>>(a, taps);
    else conv_pair_kernel<NT, 2, 1, 0, NT == 33, PADDED><<<grid, 128, 0, stream>>>(a, taps);
    return async && io != 2 ? kConvPairAsync : kConvPair;
  } else {
    dim3 grid((a.width + a.strip - 1) / a.strip, (a.height + 63) / 64);
    if (grid.y > 65535) return kLaunchFamilies;
    const bool async = t.pair_async != 0;
    if (io == 1 && async) conv_pair_async_kernel<NT, 2, 0, 1, PADDED><<<grid, 128, 0, stream>>>(a, taps);
    else if (io == 1) conv_pair_kernel<NT, 2, 0, 1, false, PADDED><<<grid, 128, 0, stream>>>(a, taps);
    else if (io == 2) conv_pair_kernel<NT, 2, 0, 2, false, PADDED><<<grid, 128, 0, stream>>>(a, taps);
    else if (async) conv_pair_async_kernel<NT, 2, 0, 0, PADDED><<<grid, 128, 0, stream>>>(a, taps);
    else conv_pair_kernel<NT, 2, 0, 0, false, PADDED><<<grid, 128, 0, stream>>>(a, taps);
    return async && io != 2 ? kConvPairAsync : kConvPair;
  }
}

template <int NT, int MODE>
int launch_nt(const Conv1dArgs &base, int axis, const double *taps_host, int ntaps, int io, bool *fused,
              cudaStream_t stream) {
  Taps<NT> taps;
  for (int i = 0; i < NT; ++i) taps.k[i] = i < ntaps ? taps_host[i] : 0.0;   // zero padding past the window
  Conv1dArgs a = base;
  a.ntaps = ntaps;
  const TuningKnobs t = tuning_knobs();
  if (io != 0 && !(MODE == 4 && NT <= 33)) return MB200_EUNSUPPORTED;
  const bool pair_ok = MODE == 4 && a.bias == 0.0 && NT <= 33 && (io != 0 || t.pair != 0) &&
                       ((reinterpret_cast<uintptr_t>(a.src) | reinterpret_cast<uintptr_t>(a.dst)) & 15) == 0;
  if (io != 0 && !pair_ok) return MB200_EUNSUPPORTED;
  if (pair_ok) {
    if constexpr (MODE == 4 && NT <= 33) {
      // strip = 16 rotations.  (A list-scheduling model of the launch -- equal-cost CTAs on 2 slots per SM -- preferred
      // 27 rotations for 8192 rows, 6 % fewer modelled steps; measured it is 5 % SLOWER, 0.822 vs 0.778 ms: CTAs that
      // run alone on an SM in the last wave get the whole FP64 pipe, so the tail balances itself.)
      a.strip = (axis == 1 ? t.col_rot : t.row_pair_rot) * NT + 1;
      a.seg_w = 16;                                  // rows of L2 prefetch ahead of the register ring (L2PF kernels)
      const bool fuse = axis == 1 && io == 0 && a.aux != nullptr && (reinterpret_cast<uintptr_t>(a.aux) & 15) == 0;
      const LaunchFamily family = ntaps != NT ? launch_pair<NT, true>(a, taps, axis, io, fuse, t, stream)
                                              : launch_pair<NT, false>(a, taps, axis, io, fuse, t, stream);
      if (family == kLaunchFamilies) return MB200_EUNSUPPORTED;
      count_family(family);
      if (fused) *fused = fuse;
    }
  } else if (axis == 1) {
    constexpr int kThreads = 128;
    constexpr int kMinBlocks = NT <= 33 ? 4 : 2;
    a.strip = t.col_rot * NT + 1;   // strip + NT - 1 is a whole number of rotations
    dim3 grid((a.rc + kThreads - 1) / kThreads, (a.height + a.strip - 1) / a.strip);
    if (grid.y > 65535) return MB200_EUNSUPPORTED;
    conv_col_kernel<NT, MODE, kThreads, kMinBlocks><<<grid, kThreads, 0, stream>>>(a, taps);
    count_family(kConvGeneric);
  } else {
    constexpr int kMinBlocks = NT <= 33 ? 4 : 2;
    // strip + NT - 1 is a whole number of rotations and the strip is at least ~64 outputs
    constexpr int kRot = (63 + NT - 1) / NT < 3 ? 3 : (63 + NT - 1) / NT;
    a.strip = (t.row_rot > 0 ? t.row_rot : kRot) * NT + 1;
    a.seg_w = a.strip + NT - 1;
    a.pitch = a.seg_w | 1;
    const int rows_per_cta = 4 * (32 / a.channels);
    const size_t smem = static_cast<size_t>(rows_per_cta) * a.pitch * a.channels * sizeof(float);
    dim3 grid((a.width + a.strip - 1) / a.strip, (a.height + rows_per_cta - 1) / rows_per_cta);
    if (smem > 200 * 1024 || grid.y > 65535) return MB200_EUNSUPPORTED;
    if (smem > 48 * 1024)            // per device attribute: set on every launch that needs it (a few microseconds)
      cudaFuncSetAttribute(conv_row_kernel<NT, MODE, kMinBlocks>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    conv_row_kernel<NT, MODE, kMinBlocks><<<grid, 128, smem, stream>>>(a, taps);
    count_family(kConvGeneric);
  }
  return launch_status("conv1d launch");
}

template <int NT>
int launch_mode(const Conv1dArgs &a, int axis, const double *taps, int ntaps, int io, bool *fused, cudaStream_t s) {
  if (a.channels == 4) return launch_nt<NT, 4>(a, axis, taps, ntaps, io, fused, s);
  if (io != 0) return MB200_EUNSUPPORTED;
  if (a.channels == 2) return launch_nt<NT, 2>(a, axis, taps, ntaps, io, fused, s);
  return launch_nt<NT, 0>(a, axis, taps, ntaps, io, fused, s);
}

}  // namespace

int launch_conv1d(const float *src, float *dst, size_t width, size_t height, int channels, int axis,
                  const double *taps, int ntaps, int origin_offset, double bias, double /*gamma_scale*/,
                  unsigned long long *d_changed, void *stream, int io, const UnsharpEpilogue *epilogue,
                  bool *epilogue_fused) {
  if (epilogue_fused) *epilogue_fused = false;
  if (width == 0 || height == 0 || channels < 1 || channels > 4 || ntaps < 1)
    return fail(MB200_EINVAL, "conv1d: bad geometry");
  if (width * channels > 0x1fffffffull || height > 0x7fffffffull) return MB200_EUNSUPPORTED;   // 32-bit byte pitch
  if (d_changed != nullptr) return MB200_EUNSUPPORTED;   // `changed` counting lives in the generic kernel
  if (channels == 4 && bias == 0.0 && ntaps <= 33) {     // RGBA: the FP64 matrix path (conv_mma.cu) when enabled
    const int rc = launch_conv_mma(src, dst, width, height, axis, taps, ntaps, origin_offset, stream, io, epilogue,
                                   epilogue_fused);
    if (rc != MB200_EUNSUPPORTED) return rc;
  }
  Conv1dArgs a{};
  a.src = src; a.dst = dst;
  a.width = static_cast<int>(width); a.height = static_cast<int>(height); a.channels = channels;
  a.rc = a.width * channels;
  a.off = origin_offset;
  a.bias = bias;
  a.changed = d_changed;
  if (epilogue && epilogue->source) { a.aux = epilogue->source; a.gain = epilogue->gain; a.qthreshold = epilogue->quantum_threshold; }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (ntaps <= 9) return launch_mode<9>(a, axis, taps, ntaps, io, epilogue_fused, s);
  if (ntaps <= 17) return launch_mode<17>(a, axis, taps, ntaps, io, epilogue_fused, s);
  if (ntaps <= 25) return launch_mode<25>(a, axis, taps, ntaps, io, epilogue_fused, s);
  if (ntaps <= 33) return launch_mode<33>(a, axis, taps, ntaps, io, epilogue_fused, s);
  if (ntaps <= 49) return launch_mode<49>(a, axis, taps, ntaps, io, epilogue_fused, s);
  if (ntaps <= 65) return launch_mode<65>(a, axis, taps, ntaps, io, epilogue_fused, s);
  return MB200_EUNSUPPORTED;   // caller falls back to the generic 2-D kernel
}

}  // namespace mb200
