// conv_mma.cu -- one pass of a separable (1-D) convolution on RGBA images, evaluated on the FP64 matrix path
// (mma.sync.m8n8k4.f64, SASS DMMA.8x8x4; windows of 18-33 taps on mma.sync.m16n8k16.f64, see conv_mma_wide_kernel).  Same semantics as conv1d.cu (MorphologyPrimitive's ConvolveMorphology for
// height-1 / width-1 kernels, MagickCore/morphology.c:2897-2979 and :2654-2807: reflected taps, edge-clamped source,
// double accumulation, alpha-weighted colour channels, one rounding to float).
//
// Why a matrix formulation for a stencil.  The DFMA streaming kernels of conv1d.cu are bound by ISSUE SLOTS next to
// the FP64 pipe (two warps per scheduler because 66 FP64 accumulators need ~210-230 registers).  DMMA runs on the
// FP64 tensor cores (tools/micro/dmma.cu measures its rate) and one instruction carries 256 FMAs: ~7 instructions per
// DMMA instead of 1.7 per DFMA, 8 accumulator registers per tile, four CTAs per SM.  The price is the band structure:
// 8 consecutive outputs of a 33-tap window touch 40 source samples, i.e. ten 8x4 Toeplitz tiles of which 17.5 % of the
// cells are zero (17 taps: 29 %, 9 taps: 44 %).
//
//   D[m][n] += A[m][k] * B[k][n]     m = 8 consecutive outputs along the filter axis
//                                    k = 4 consecutive source samples (one of NKS k-steps)
//                                    n = 8 independent component lines
//   A = taps as a banded Toeplitz tile: A_s[m][k] = tap[4 s + k - m] (zero outside the window) -- NKS doubles per
//       lane, loaded once per thread and reused for the whole strip;
//   B = source samples, converted to double and alpha-premultiplied ONCE when they are staged into a per-warp
//       shared-memory ring (q = A*p; the weight sum of the blend is the alpha line's own result, as in conv1d.cu);
//   D = two doubles per lane and tile.  Tiles come in (R,G) / (B,A) plane pairs whose n index is mapped so that a
//       lane ends up with all four sums of ONE pixel: one reciprocal per pixel, no shuffles, one 16-byte store.
//
// A warp is self-contained (its own ring, __syncwarp only): it owns 8 pixels x all rows of a strip (AXIS 1) or 8 image
// lines x all pixels of a strip (AXIS 0) and advances 8 outputs per iteration: stage 8 new source positions (2 pixels
// per lane, loaded one iteration ahead), 4 tiles x NKS DMMAs, output stage.
//
// Non-finite samples.  Every tile multiplies samples outside an output's window by a ZERO tap; 0 * (inf | NaN) would
// poison outputs the reference computes from finite samples only.  The loader therefore tests every sample's exponent
// field and keeps one flag per 8-position block of the ring; an output block whose window holds a flagged block is
// evaluated by a scalar DFMA loop over the window's own taps instead (rare: HDRI images with inf / NaN pixels).
#include "mb200_internal.h"
#include "conv_common.cuh"
#include "tma.cuh"

#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>

namespace mb200 {
namespace {

template <int NKS>
struct MmaTaps { double k[4 * NKS]; };      // window order, zero past the window

struct MmaArgs {
  const void *src;
  void *dst;
  int width, height;      // pixels
  int off;                // samples of the window before the output position
  int ntaps;
  int strip;              // outputs per strip along the filter axis (multiple of 8; of 16 for the wide tiles)
  const float *aux;       // EPI = 1: UnsharpMaskImage's source image
  double gain, qthreshold;
  int l2pf;               // prefetch.global.L2 ahead of the register prefetch
};

__device__ __forceinline__ void dmma(double (&d)[2], double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
      : "+d"(d[0]), "+d"(d[1]) : "d"(a), "d"(b));
}

// Raw loads of one block (two pixels per lane) kept in registers for one iteration.
template <int IO> struct Raw;
template <> struct Raw<0> { float4 a; };
template <> struct Raw<2> { double2 a, b; };

template <int NKS, int AXIS, int IO, int EPI, int MINB>
__global__ void __launch_bounds__(128, MINB) conv_mma_kernel(const MmaArgs a, const MmaTaps<NKS> taps) {
  static_assert(NKS % 2 == 0, "the prologue stages whole 8-position blocks");
  static_assert(EPI == 0 || (AXIS == 1 && IO == 0), "the fused epilogue belongs to the final column pass");
  constexpr int NPRE = (4 * NKS - 8) / 8;          // blocks staged before the first output block
  constexpr int NB = NPRE + 2;                     // ring blocks: window (NPRE + 1) + the one being refilled
  constexpr int RR = 8 * NB;                       // ring positions along the filter axis
  constexpr int PW = 36;                           // AXIS 1: doubles per ring row: [RG of 8 px | BA of 8 px | pad 4]
  constexpr int PL = 2 * RR + 8;                   // AXIS 0: doubles per image line of a plane (== 8 mod 16)
  constexpr int kWarpDoubles = AXIS == 1 ? RR * PW : 16 * PL;
  constexpr int kInB = IO == 2 ? 32 : 16, kOutB = IO == 1 ? 32 : 16;      // bytes per pixel
  constexpr int RIO = IO == 2 ? 2 : 0;
  extern __shared__ __align__(16) double ring_all[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double *ring = ring_all + warp * kWarpDoubles;
  const unsigned ring_s = static_cast<unsigned>(__cvta_generic_to_shared(ring));
  const int k4 = lane & 3, n8 = lane >> 2;         // fragment coordinates: A[m = n8][k = k4], B[k4][n8], D[n8][2 k4 + e]

  int first, nout, limit, par0;
  if (AXIS == 1) {
    par0 = (blockIdx.x * 4 + warp) * 8;            // first pixel column of this warp
    if (par0 >= a.width) return;                   // (no CTA-wide barrier anywhere: a warp may leave)
    first = blockIdx.y * a.strip;
    nout = min(a.strip, a.height - first);
    limit = a.height - 1;
  } else {
    par0 = (blockIdx.y * 4 + warp) * 8;            // first image line of this warp
    if (par0 >= a.height) return;
    first = blockIdx.x * a.strip;
    nout = min(a.strip, a.width - first);
    limit = a.width - 1;
  }
  const int nblocks = (nout + 7) >> 3;
  const bool mma_l2pf = a.l2pf != 0;
  const size_t in_pitch = static_cast<size_t>(a.width) * kInB, out_pitch = static_cast<size_t>(a.width) * kOutB;

  // ---- loader: two pixels per lane and block
  const int lq = lane & 7, lh = lane >> 3;
  const char *lbase[2];
  int uoff[2];
  unsigned st_off[2];                               // ring offset (doubles) of the RG pair inside block slot 0
  if (AXIS == 1) {
    const int xs = min(par0 + lq, a.width - 1);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      lbase[i] = static_cast<const char *>(a.src) + static_cast<size_t>(xs) * kInB;
      uoff[i] = lh + 4 * i;
      st_off[i] = static_cast<unsigned>(uoff[i] * PW + 2 * lq);
    }
  } else {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int line = lh + 4 * i;
      lbase[i] = static_cast<const char *>(a.src) + static_cast<size_t>(min(par0 + line, a.height - 1)) * in_pitch;
      uoff[i] = lq;
      st_off[i] = static_cast<unsigned>(line * PL + 2 * lq);
    }
  }
  constexpr unsigned kBlockStride = AXIS == 1 ? 8 * PW : 16;     // ring doubles per block slot
  constexpr unsigned kBA = AXIS == 1 ? 16 : 8 * PL;               // RG -> BA plane
  const size_t lstep = AXIS == 1 ? in_pitch : static_cast<size_t>(kInB);
  const int base = first - a.off;                   // source position of ring block 0, element 0

  Raw<RIO> raw[2];
  auto fetch = [&](int j) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const unsigned pos = static_cast<unsigned>(min(max(base + 8 * j + uoff[i], 0), limit));
      const char *p = lbase[i] + static_cast<size_t>(pos) * lstep;
      if constexpr (IO == 2) {
        raw[i].a = __ldg(reinterpret_cast<const double2 *>(p));
        raw[i].b = __ldg(reinterpret_cast<const double2 *>(p) + 1);
      } else {
        raw[i].a = __ldg(reinterpret_cast<const float4 *>(p));
      }
    }
  };
  // L2 prefetch kL2Ahead blocks beyond the register prefetch: the LDGs of `fetch` then complete at L2 latency.  Short
  // windows run so few DMMAs per iteration that two blocks of loads in flight per warp do not cover DRAM latency
  // (9 taps: 0.52 ms per pass against 0.33 ms of HBM time before this).
  constexpr int kL2Ahead = 8;
  auto prefetch_l2 = [&](int j) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const unsigned pos = static_cast<unsigned>(min(max(base + 8 * j + uoff[i], 0), limit));
      asm volatile("prefetch.global.L2 [%0];" ::"l"(lbase[i] + static_cast<size_t>(pos) * lstep));
    }
  };
  unsigned badmask = 0;
  auto stage = [&](int slot) {                      // registers -> ring block `slot`; updates the block's flag
    bool bad = false;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      double v0, v1, v2, v3;
      if constexpr (IO == 2) {
        v0 = raw[i].a.x; v1 = raw[i].a.y; v2 = raw[i].b.x; v3 = raw[i].b.y;
        bad = bad || nonfinite_bits(v0) || nonfinite_bits(v1) || nonfinite_bits(v2) || nonfinite_bits(v3);
      } else {
        const float4 f = raw[i].a;
        const unsigned m = max(max(__float_as_uint(f.x) & 0x7fffffffu, __float_as_uint(f.y) & 0x7fffffffu),
                               max(__float_as_uint(f.z) & 0x7fffffffu, __float_as_uint(f.w) & 0x7fffffffu));
        bad = bad || m >= 0x7f800000u;
        const double da = static_cast<double>(f.w);
        v0 = static_cast<double>(f.x) * da;
        v1 = static_cast<double>(f.y) * da;
        v2 = static_cast<double>(f.z) * da;
        v3 = da;
      }
      double *q = ring + st_off[i] + static_cast<unsigned>(slot) * kBlockStride;
      *reinterpret_cast<double2 *>(q) = make_double2(v0, v1);
      *reinterpret_cast<double2 *>(q + kBA) = make_double2(v2, v3);
    }
    const bool any = __any_sync(0xffffffffu, bad);
    badmask = any ? (badmask | (1u << slot)) : (badmask & ~(1u << slot));
  };

  // ---- tap tiles: A_s[m][k] = tap[4 s + k - m]
  double afrag[NKS];
#pragma unroll
  for (int s = 0; s < NKS; ++s) {
    const int t = 4 * s + k4 - n8;
    const double v = taps.k[min(max(t, 0), 4 * NKS - 1)];
    afrag[s] = (t >= 0 && t < a.ntaps) ? v : 0.0;
  }

  // ---- B fragment addressing
  const unsigned frag_off = AXIS == 1 ? static_cast<unsigned>(k4 * PW + n8)
                                      : static_cast<unsigned>(2 * k4 + (n8 >> 1) * PL + (n8 & 1));
  constexpr unsigned kUStride = AXIS == 1 ? PW : 2;            // ring doubles per position
  constexpr unsigned kT1 = kBA;                                 // (group 0, BA)
  constexpr unsigned kT2 = AXIS == 1 ? 8 : 4 * PL;              // (group 1, RG)
  constexpr unsigned kT3 = kT2 + kBA;                           // (group 1, BA)
  // scalar path / output coordinates of this lane: output m = n8 of the block, pixel (AXIS 1) or line (AXIS 0) 4 g + k4
  const unsigned lane_px_off = AXIS == 1 ? static_cast<unsigned>(2 * k4) : static_cast<unsigned>(k4 * PL);
  constexpr unsigned kGroup = AXIS == 1 ? 8 : 4 * PL;

  // ---- output stage of one block: the lane holds pixel (m = n8, 4 g + k4) with all four sums
  char *outp;                                       // output of (block, m = n8, group 0); lags the MMAs by one block
  const char *epip = nullptr;
  if (AXIS == 1) {
    outp = static_cast<char *>(a.dst) + static_cast<size_t>(first + n8) * out_pitch + static_cast<size_t>(par0 + k4) * kOutB;
    if (EPI) epip = reinterpret_cast<const char *>(a.aux) + static_cast<size_t>(first + n8) * out_pitch + static_cast<size_t>(par0 + k4) * kOutB;
  } else {
    outp = static_cast<char *>(a.dst) + static_cast<size_t>(par0 + k4) * out_pitch + static_cast<size_t>(first + n8) * kOutB;
  }
  const size_t ostep = AXIS == 1 ? 8 * out_pitch : static_cast<size_t>(8 * kOutB);        // per block
  const size_t gstep = AXIS == 1 ? static_cast<size_t>(4 * kOutB) : 4 * out_pitch;        // group 0 -> group 1
  bool gvalid[2];
#pragma unroll
  for (int g = 0; g < 2; ++g) gvalid[g] = (par0 + 4 * g + k4) < (AXIS == 1 ? a.width : a.height);
  auto output = [&](const double (&acc)[4][2], const float4 (&epi)[2], bool mvalid) {
#pragma unroll
    for (int g = 0; g < 2; ++g) {
      const double sr = acc[2 * g][0], sg = acc[2 * g][1], sbv = acc[2 * g + 1][0], sa = acc[2 * g + 1][1];
      char *o = outp + g * gstep;
      if (IO == 1) {
        if (mvalid && gvalid[g]) {
          *reinterpret_cast<double2 *>(o) = make_double2(sr, sg);
          *reinterpret_cast<double2 *>(o + 16) = make_double2(sbv, sa);
        }
      } else {
        const double r = fast_reciprocal(clamp_denominator(sa));
        float4 out = make_float4(static_cast<float>(sr * r), static_cast<float>(sg * r), static_cast<float>(sbv * r),
                                 static_cast<float>(sa));
        if (EPI) {
          out.x = unsharp_point(epi[g].x, out.x, a.gain, a.qthreshold);
          out.y = unsharp_point(epi[g].y, out.y, a.gain, a.qthreshold);
          out.z = unsharp_point(epi[g].z, out.z, a.gain, a.qthreshold);
          out.w = unsharp_point(epi[g].w, out.w, a.gain, a.qthreshold);
        }
        if (mvalid && gvalid[g]) *reinterpret_cast<float4 *>(o) = out;
      }
    }
  };

  // ---- prologue: the NPRE + 1 blocks of the first window (all loads in flight together), then the block after it
  {
    Raw<RIO> pre[NPRE + 1][2];
#pragma unroll
    for (int j = 0; j <= NPRE; ++j) { fetch(j); pre[j][0] = raw[0]; pre[j][1] = raw[1]; }
#pragma unroll
    for (int j = 0; j <= NPRE; ++j) { raw[0] = pre[j][0]; raw[1] = pre[j][1]; stage(j); }
  }
  Raw<RIO> ahead[2];                                 // the block after the one in `raw` (loads two iterations in flight)
  fetch(NPRE + 2);
  ahead[0] = raw[0]; ahead[1] = raw[1];
  fetch(NPRE + 1);

  // ---- main loop, software pipelined by hand: iteration b issues the DMMAs of block b and, in the same basic block,
  // stages the next source block into the ring slot no window of this iteration reads and runs the output stage of
  // block b - 1.  The warp issues in order, so the conversions / reciprocals / stores ride in the gaps between its DMMAs
  // instead of forming phases of their own in which the FP64 pipe is left to the other warps (first version, separate
  // phases: pipe 78 % busy).
  int st_slot = NPRE + 1, sb = 0;                    // slot staged in this iteration / first slot of the window
  double prev[4][2];
  float4 epi_prev[2], epi_cur[2];
#pragma unroll
  for (int t = 0; t < 4; ++t) { prev[t][0] = 0.0; prev[t][1] = 1.0; }
#pragma unroll
  for (int g = 0; g < 2; ++g) epi_prev[g] = epi_cur[g] = make_float4(0.f, 0.f, 0.f, 0.f);
  bool prev_valid = false;                           // block -1 does not exist

#pragma unroll 1
  for (int b = 0; b < nblocks; ++b) {
    __syncwarp();
    const bool mvalid = 8 * b + n8 < nout;
    if (EPI) {
#pragma unroll
      for (int g = 0; g < 2; ++g)
        if (mvalid && gvalid[g]) epi_cur[g] = __ldg(reinterpret_cast<const float4 *>(epip + g * gstep));
      epip += ostep;
    }
    double acc[4][2];
#pragma unroll
    for (int t = 0; t < 4; ++t) { acc[t][0] = 0.0; acc[t][1] = 0.0; }
    {
      // B fragments through a 3-deep register ring, loaded two k-steps ahead of the DMMAs that consume them
      double bq[3][4];
      unsigned ua[NKS];
      {
        int ub = 8 * sb;
#pragma unroll
        for (int s = 0; s < NKS; ++s) {
          ua[s] = ring_s + (frag_off + static_cast<unsigned>(ub) * kUStride) * 8u;
          ub += 4;
          if (ub == RR) ub = 0;
        }
      }
      auto lds4 = [&](double (&bv)[4], unsigned addr) {
        asm volatile("ld.shared.f64 %0, [%1];" : "=d"(bv[0]) : "r"(addr));
        asm volatile("ld.shared.f64 %0, [%1+%2];" : "=d"(bv[1]) : "r"(addr), "n"(kT1 * 8));
        asm volatile("ld.shared.f64 %0, [%1+%2];" : "=d"(bv[2]) : "r"(addr), "n"(kT2 * 8));
        asm volatile("ld.shared.f64 %0, [%1+%2];" : "=d"(bv[3]) : "r"(addr), "n"(kT3 * 8));
      };
      lds4(bq[0], ua[0]);
      lds4(bq[1], ua[1]);
#pragma unroll
      for (int s = 0; s < NKS; ++s) {
        if (s + 2 < NKS) lds4(bq[(s + 2) % 3], ua[s + 2]);
        dmma(acc[0], afrag[s], bq[s % 3][0]);
        dmma(acc[1], afrag[s], bq[s % 3][1]);
        dmma(acc[2], afrag[s], bq[s % 3][2]);
        dmma(acc[3], afrag[s], bq[s % 3][3]);
      }
    }
    const unsigned window_bad = badmask & ~(1u << st_slot);     // flags of the slots this block's windows read
    // next source block -> ring (the slot outside this iteration's windows), the one after it -> registers
    stage(st_slot);
    raw[0] = ahead[0]; raw[1] = ahead[1];
    {
      const Raw<RIO> keep0 = raw[0], keep1 = raw[1];
      fetch(b + NPRE + 3);
      if (mma_l2pf) prefetch_l2(b + NPRE + 3 + kL2Ahead);
      ahead[0] = raw[0]; ahead[1] = raw[1];
      raw[0] = keep0; raw[1] = keep1;
    }
    // output stage of the previous block
    output(prev, epi_prev, prev_valid);
    if (b > 0) outp += ostep;

    if (window_bad != 0) {
      // a window of this block holds a non-finite sample: the window's own taps only, in scalar FMAs
#pragma unroll
      for (int g = 0; g < 2; ++g) {
        double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
        int u = 8 * sb + n8;
        if (u >= RR) u -= RR;
        for (int t = 0; t < a.ntaps; ++t) {
          const double *p = ring + static_cast<unsigned>(u) * kUStride + lane_px_off + g * kGroup;
          const double2 rg = *reinterpret_cast<const double2 *>(p);
          const double2 ba = *reinterpret_cast<const double2 *>(p + kBA);
          const double k = taps.k[t];
          s0 = fma(k, rg.x, s0); s1 = fma(k, rg.y, s1); s2 = fma(k, ba.x, s2); s3 = fma(k, ba.y, s3);
          if (++u == RR) u = 0;
        }
        acc[2 * g][0] = s0; acc[2 * g][1] = s1; acc[2 * g + 1][0] = s2; acc[2 * g + 1][1] = s3;
      }
    }
#pragma unroll
    for (int t = 0; t < 4; ++t) { prev[t][0] = acc[t][0]; prev[t][1] = acc[t][1]; }
    if (EPI) { epi_prev[0] = epi_cur[0]; epi_prev[1] = epi_cur[1]; }
    prev_valid = mvalid;
    st_slot = st_slot + 1 == NB ? 0 : st_slot + 1;
    if (++sb == NB) sb = 0;
  }
  output(prev, epi_prev, prev_valid);
}

// ---- the wide-tile pass: mma.sync.m16n8k16.f64 (SASS DMMA.16x8x16), RGBA float in / float out.
//
//   D[m][n] += A_s[m][k] * B_s[k][n]    m = 16 consecutive outputs, k = 16 consecutive source samples (k-step s of NKS),
//                                       n = 8 component lines;  A_s[m][k] = tap[16 s + k - m]
//
// One DMMA.16x8x16 carries 2048 FMAs: 4 tiles x NKS = 12 DMMAs per 16 outputs x 8 pixel lines of a 33-tap window, where
// conv_mma_kernel issues 80 DMMA.8x8x4 (tools/micro/dmma.cu and dmma_feed.cu measure both shapes).  Fragment
// coordinates (g = lane / 4, t = lane % 4): A element i at (m = g + 8 (i & 1), k = t + 4 (i >> 1)), B element i at
// (k = t + 4 i, n = g), D element i at (m = g + 8 (i >> 1), n = 2 t + (i & 1)).  The n mapping is conv_mma_kernel's, so a
// lane ends up with all four sums of pixel line 4 G + t (tile group G) at outputs g and g + 8.
//
// Everything else is conv_mma_kernel's scheme at 16-position blocks: a per-warp ring of NKS + 1 blocks (the window and
// the block being refilled), samples converted and premultiplied once when staged, one non-finite flag per block, and the DMMAs of block b, the staging of block b + NKS and the output stage of block
// b - 1 in one basic block.  Outputs start at multiples of 16 of the image position (the launcher rounds the strip up),
// so an output's k-grouping, and its bits, do not depend on the strip.
template <int NKS>
struct WideTaps { double k[16 * NKS]; };    // window order, zero past the window

// ---- the TMA-fed wide pass on a persistent grid.  Same staging, DMMAs, non-finite flags and output stage as above; what
// differs is where the source blocks come from and which strips a warp walks.
//
// Loads.  A warp's raw source blocks (16 positions x 8 lines of float4 = 2 KB: 8 px x 16 rows in the column pass, 16 px x
// 8 lines in the row pass) arrive in a per-warp shared-memory ring of kWideStages slots, each filled by one
// cp.async.bulk.tensor.2d that lane 0 issues, with an mbarrier transaction count per slot.  A slot is refilled as soon
// as the warp has read it into registers, so kWideStages - 1 blocks (6 KB) stay in flight per warp without holding any
// registers.  The quarter-warp reads 128 contiguous bytes of a box row: conflict-free LDS.128 without a swizzle.
// The TMA unit zero-fills outside the image where the reference clamps to the edge, so boxes are issued at clamped
// coordinates (inside the image whenever the image is at least 16 positions long) and each position is clamped inside
// its box when it is read: the staged samples are exactly those of min(max(pos, 0), last).
//
// Schedule.  The grid is as many CTAs as fit on the device at once (2 per SM); the (band of 8 lines, strip) tiles are
// split into one contiguous run per warp, band-major, in whole strips: the runs differ by at most one strip (8192^2 at strip 512:
// 16 or 15 of 16 384 tiles per warp over 1 056 warps, ~3 % of the pass in tail).  Consecutive strips of one band are one
// segment: the ring carries on across them without a new prologue.  Outputs still start at multiples of 16 of the
// image position, so the bits depend neither on the strip nor on the split.
constexpr int kWideStages = 4;
constexpr unsigned kWideBoxBytes = 2048;

template <int NKS, int AXIS, int EPI>
__global__ void __launch_bounds__(128, 2) conv_mma_wide_kernel(const MmaArgs a, const WideTaps<NKS> taps,
                                                                const __grid_constant__ CUtensorMap tmap) {
  static_assert(EPI == 0 || AXIS == 1, "the fused epilogue belongs to the final column pass");
  constexpr int NB = NKS + 1;                      // ring blocks: the window + the one being refilled
  constexpr int RR = 16 * NB;                      // ring positions along the filter axis
  constexpr int PW = 36;                           // AXIS 1: doubles per ring row: [RG of 8 px | BA of 8 px | pad 4]
  constexpr int PL = 2 * RR + 8;                   // AXIS 0: doubles per image line of a plane (== 8 mod 16)
  constexpr int kWarpDoubles = AXIS == 1 ? RR * PW : 16 * PL;
  constexpr int W = 4, S = kWideStages;            // warps per CTA, raw slots per warp
  extern __shared__ __align__(128) unsigned char smem_all[];
  __shared__ __align__(8) unsigned long long bars[W][S];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // TMA destinations must be 128-byte aligned: the raw slots of the four warps first, then the double rings
  unsigned char *smem = smem_all + ((128u - (static_cast<unsigned>(__cvta_generic_to_shared(smem_all)) & 127u)) & 127u);
  const unsigned raw_s = static_cast<unsigned>(__cvta_generic_to_shared(smem)) + warp * S * kWideBoxBytes;
  double *ring = reinterpret_cast<double *>(smem + W * S * kWideBoxBytes) + warp * kWarpDoubles;
  const unsigned ring_s = static_cast<unsigned>(__cvta_generic_to_shared(ring));
  const unsigned bar_s = static_cast<unsigned>(__cvta_generic_to_shared(&bars[warp][0]));
  const int t4 = lane & 3, g8 = lane >> 2;

  // ---- this warp's run of tiles
  const int len = AXIS == 1 ? a.height : a.width;  // extent along the filter axis
  const int limit = len - 1;
  const int nstrips = (len + a.strip - 1) / a.strip;
  const long long ntiles = static_cast<long long>(((AXIS == 1 ? a.width : a.height) + 7) >> 3) * nstrips;
  const long long nwarps = static_cast<long long>(gridDim.x) * W, gw = static_cast<long long>(blockIdx.x) * W + warp;
  const long long per = ntiles / nwarps, extra = ntiles % nwarps;
  const long long t_begin = gw * per + min(gw, extra), t_end = t_begin + per + (gw < extra ? 1 : 0);
  if (t_begin >= t_end) return;                    // (no CTA-wide barrier anywhere: a warp may leave)
  struct Seg { long long end; int band, first, nout; };
  auto segment = [&](long long t) {                // the strips of t's band from t on, up to the end of the run
    Seg sg;
    sg.band = static_cast<int>(t / nstrips);
    const long long band_end = static_cast<long long>(sg.band + 1) * nstrips;
    sg.end = min(t_end, band_end);
    sg.first = static_cast<int>(t - static_cast<long long>(sg.band) * nstrips) * a.strip;
    sg.nout = min(static_cast<int>(sg.end - static_cast<long long>(sg.band) * nstrips) * a.strip, len) - sg.first;
    return sg;
  };
  // box of the 16 source positions from p0: inside the image where it is long enough; clamped positions index into it
  auto box_start = [&](int p0) { return min(max(p0, 0), max(limit - 15, 0)); };

  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < S; ++k) mbar_init(bar_s + 8 * k, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncwarp();

  // ---- producer: the raw blocks of every segment in the order they are consumed (a segment of nblocks output blocks
  // reads nblocks + NKS - 1 source blocks), kept S blocks ahead of the consumer
  Seg pseg = segment(t_begin);
  int pj = 0;
  unsigned np = 0, nc = 0;                         // blocks issued / consumed by this warp
  auto issue_next = [&]() {                        // warp-uniform
    if (pseg.band < 0) return;
    const int s0 = box_start(pseg.first - a.off + 16 * pj);
    if (lane == 0) {
      const unsigned k = np % S, bar = bar_s + 8 * k;
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // the slot's generic-proxy reads precede the refill
      mbar_expect_tx(bar, kWideBoxBytes);
      if (AXIS == 1) tma_load_2d(raw_s + k * kWideBoxBytes, &tmap, pseg.band * 32, s0, bar);
      else tma_load_2d(raw_s + k * kWideBoxBytes, &tmap, s0 * 4, pseg.band * 8, bar);
    }
    ++np;
    if (++pj == ((pseg.nout + 15) >> 4) + NKS - 1) {
      pj = 0;
      if (pseg.end < t_end) pseg = segment(pseg.end);
      else pseg.band = -1;
    }
  };
#pragma unroll
  for (int k = 0; k < S; ++k) issue_next();

  // ---- consumer lanes: four pixels per lane and block
  const int lq = lane & 7, lh = lane >> 3;
  int uoff[4];
  unsigned raw_off[4];                             // byte offset inside a box, without the position along the filter axis
  unsigned st_off[4];                              // ring offset (doubles) of the RG pair inside block slot 0
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if (AXIS == 1) {                               // rows lh + 4 i of the block, pixel column lq
      uoff[i] = lh + 4 * i;
      raw_off[i] = static_cast<unsigned>(lq * 16);
      st_off[i] = static_cast<unsigned>(uoff[i] * PW + 2 * lq);
    } else {                                       // image line lh + 4 (i >> 1), positions lq + 8 (i & 1) of the block
      const int line = lh + 4 * (i >> 1);
      uoff[i] = lq + 8 * (i & 1);
      raw_off[i] = static_cast<unsigned>(line * 256);
      st_off[i] = static_cast<unsigned>(line * PL + 2 * uoff[i]);
    }
  }
  constexpr unsigned kPosBytes = AXIS == 1 ? 128 : 16;           // raw box bytes per position along the filter axis
  constexpr unsigned kBlockStride = AXIS == 1 ? 16 * PW : 32;     // ring doubles per block slot
  constexpr unsigned kBA = AXIS == 1 ? 16 : 8 * PL;               // RG -> BA plane

  float4 raw[4];
  int base = 0;                                    // source position of the segment's ring block 0, element 0
  auto take = [&](int j) {                         // raw block j of the segment -> registers; refill its slot
    const unsigned k = nc % S;
    mbar_wait(bar_s + 8 * k, (nc / S) & 1u);
    const int p0 = base + 16 * j, s0 = box_start(p0);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const unsigned pos = static_cast<unsigned>(min(max(p0 + uoff[i], 0), limit) - s0);
      const unsigned addr = raw_s + k * kWideBoxBytes + raw_off[i] + pos * kPosBytes;
      asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];"
                   : "=f"(raw[i].x), "=f"(raw[i].y), "=f"(raw[i].z), "=f"(raw[i].w) : "r"(addr) : "memory");
    }
    ++nc;
    __syncwarp();                                  // every lane has read the slot
    issue_next();
  };
  unsigned badmask = 0;
  auto stage = [&](int slot) {                     // registers -> ring block `slot`; updates the block's flag
    bool bad = false;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float4 f = raw[i];
      const unsigned m = max(max(__float_as_uint(f.x) & 0x7fffffffu, __float_as_uint(f.y) & 0x7fffffffu),
                             max(__float_as_uint(f.z) & 0x7fffffffu, __float_as_uint(f.w) & 0x7fffffffu));
      bad = bad || m >= 0x7f800000u;
      const double da = static_cast<double>(f.w);
      double *q = ring + st_off[i] + static_cast<unsigned>(slot) * kBlockStride;
      *reinterpret_cast<double2 *>(q) = make_double2(static_cast<double>(f.x) * da, static_cast<double>(f.y) * da);
      *reinterpret_cast<double2 *>(q + kBA) = make_double2(static_cast<double>(f.z) * da, da);
    }
    const bool any = __any_sync(0xffffffffu, bad);
    badmask = any ? (badmask | (1u << slot)) : (badmask & ~(1u << slot));
  };

  // ---- tap tiles: element i of A_s is tap[16 s + t4 + 4 (i >> 1) - g8 - 8 (i & 1)] = atap[c + 2] with
  // c = 4 s + (i >> 1) - 2 (i & 1): 4 NKS + 2 distinct doubles per lane instead of 8 NKS
  constexpr int NA = 4 * NKS + 2;
  double atap[NA];
#pragma unroll
  for (int c = 0; c < NA; ++c) {
    const int t = 4 * (c - 2) + t4 - g8;
    const double v = taps.k[min(max(t, 0), 16 * NKS - 1)];
    atap[c] = (t >= 0 && t < a.ntaps) ? v : 0.0;
  }

  // ---- B fragment addressing: element i of k-step s reads ring position 16 (sb + s) + t4 + 4 i, column g8
  const unsigned frag_off = AXIS == 1 ? static_cast<unsigned>(t4 * PW + g8)
                                      : static_cast<unsigned>(2 * t4 + (g8 >> 1) * PL + (g8 & 1));
  constexpr unsigned kUStride = AXIS == 1 ? PW : 2;             // ring doubles per position
  constexpr unsigned kT2 = AXIS == 1 ? 8 : 4 * PL;              // tile group 1
  constexpr unsigned kTile[4] = {0, kBA, kT2, kT2 + kBA};       // (G, plane) = (0, RG), (0, BA), (1, RG), (1, BA)
  const unsigned lane_px_off = AXIS == 1 ? static_cast<unsigned>(2 * t4) : static_cast<unsigned>(t4 * PL);

  const size_t pitch = static_cast<size_t>(a.width) * 16;
  const size_t ostep = AXIS == 1 ? 16 * pitch : 16 * 16;          // per block
  const size_t gstep = AXIS == 1 ? 4 * 16 : 4 * pitch;            // G 0 -> 1
  const size_t hstep = AXIS == 1 ? 8 * pitch : 8 * 16;            // output g8 -> g8 + 8

#pragma unroll 1
  for (long long tile = t_begin; tile < t_end;) {
    const Seg sg = segment(tile);
    tile = sg.end;
    const int par0 = sg.band * 8, first = sg.first, nout = sg.nout;
    const int nblocks = (nout + 15) >> 4;
    base = first - a.off;

    // ---- output stage: the lane holds pixel line 4 G + t4 at outputs g8 and g8 + 8 of a block
    char *outp;                                    // output of (block, m = g8, G = 0); lags the MMAs by one block
    if (AXIS == 1) {
      outp = static_cast<char *>(a.dst) + static_cast<size_t>(first + g8) * pitch + static_cast<size_t>(par0 + t4) * 16;
    } else {
      outp = static_cast<char *>(a.dst) + static_cast<size_t>(par0 + t4) * pitch + static_cast<size_t>(first + g8) * 16;
    }
    bool gvalid[2];
#pragma unroll
    for (int g = 0; g < 2; ++g) gvalid[g] = (par0 + 4 * g + t4) < (AXIS == 1 ? a.width : a.height);
    auto output = [&](const double (&acc)[4][4], const float4 (&epi)[2][2], int mrem) {    // mrem: outputs left in the block
#pragma unroll
      for (int g = 0; g < 2; ++g)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const double sr = acc[2 * g][2 * h], sg = acc[2 * g][2 * h + 1], sbv = acc[2 * g + 1][2 * h],
                       sa = acc[2 * g + 1][2 * h + 1];
          const double r = fast_reciprocal(clamp_denominator(sa));
          float4 out = make_float4(static_cast<float>(sr * r), static_cast<float>(sg * r), static_cast<float>(sbv * r),
                                   static_cast<float>(sa));
          if (EPI) {
            out.x = unsharp_point(epi[g][h].x, out.x, a.gain, a.qthreshold);
            out.y = unsharp_point(epi[g][h].y, out.y, a.gain, a.qthreshold);
            out.z = unsharp_point(epi[g][h].z, out.z, a.gain, a.qthreshold);
            out.w = unsharp_point(epi[g][h].w, out.w, a.gain, a.qthreshold);
          }
          if (g8 + 8 * h < mrem && gvalid[g]) *reinterpret_cast<float4 *>(outp + g * gstep + h * hstep) = out;
        }
    };

    // ---- prologue: the NKS blocks of the first window, then the block after it into registers
    badmask = 0;
#pragma unroll
    for (int j = 0; j < NKS; ++j) {
      take(j);
      stage(j);
    }
    if (nblocks > 1) take(NKS);

    int st_slot = NKS, sb = 0;                     // slot staged in this iteration / first slot of the window
    double prev[4][4];
#pragma unroll
    for (int t = 0; t < 4; ++t)
#pragma unroll
      for (int i = 0; i < 4; ++i) prev[t][i] = (i & 1) ? 1.0 : 0.0;
    float4 epi_prev[2][2], epi_cur[2][2];
#pragma unroll
    for (int g = 0; g < 2; ++g)
#pragma unroll
      for (int h = 0; h < 2; ++h) epi_prev[g][h] = epi_cur[g][h] = make_float4(0.f, 0.f, 0.f, 0.f);
    int prev_rem = 0;                              // block -1 does not exist

#pragma unroll 1
    for (int b = 0; b < nblocks; ++b) {
      __syncwarp();
      const int mrem = nout - 16 * b;
      const unsigned window_bad = badmask & ~(1u << st_slot);     // flags of the slots this block's windows read
      // Output stage of the previous block and staging of the next one come BEFORE this block's DMMAs in the source, so
      // that `prev` and the staged registers are dead while the accumulators are live; ptxas interleaves them with the
      // DMMAs, which are in the same basic block.
      output(prev, epi_prev, prev_rem);
      if (b > 0) outp += ostep;
      if (EPI) {                                   // the source pixels of block b: aux at outp's offset (outp is at block b here)
        const char *epip = reinterpret_cast<const char *>(a.aux) + (outp - static_cast<char *>(a.dst));
#pragma unroll
        for (int g = 0; g < 2; ++g)
#pragma unroll
          for (int h = 0; h < 2; ++h)
            if (g8 + 8 * h < mrem && gvalid[g])
              epi_cur[g][h] = __ldg(reinterpret_cast<const float4 *>(epip + g * gstep + h * hstep));
      }
      // next source block -> ring (the slot no window of this iteration reads; the __syncwarp above orders it after the
      // previous iteration's reads)
      if (b + 1 < nblocks) stage(st_slot);
      double acc[4][4];
#pragma unroll
      for (int t = 0; t < 4; ++t)
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[t][i] = 0.0;
      {
        // B fragments, one (k-step, tile) at a time, loaded one DMMA ahead (a DMMA.16x8x16 occupies the pipe for ~64
        // cycles, longer than an LDS takes)
        unsigned ua[NKS];
#pragma unroll
        for (int s = 0; s < NKS; ++s) {
          const int blk = sb + s >= NB ? sb + s - NB : sb + s;
          ua[s] = ring_s + (frag_off + static_cast<unsigned>(blk) * kBlockStride) * 8u;
        }
        auto lds4 = [&](double (&bv)[4], int q) {
          const unsigned addr = ua[q >> 2] + kTile[q & 3] * 8;        // (q is unrolled: the offsets fold into the LDS)
#pragma unroll
          for (int i = 0; i < 4; ++i)
            asm volatile("ld.shared.f64 %0, [%1];" : "=d"(bv[i]) : "r"(addr + 4 * i * kUStride * 8));
        };
        double bq[2][4];
        lds4(bq[0], 0);
#pragma unroll
        for (int q = 0; q < 4 * NKS; ++q) {
          if (q + 1 < 4 * NKS) lds4(bq[(q + 1) & 1], q + 1);
          const double *av = atap + 4 * (q >> 2);   // element i: av[(i >> 1) + 2 - 2 (i & 1)]
          double (&d)[4] = acc[q & 3];
          const double (&bv)[4] = bq[q & 1];
          asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
                       "{%12,%13,%14,%15}, {%0,%1,%2,%3};"
                       : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
                       : "d"(av[2]), "d"(av[0]), "d"(av[3]), "d"(av[1]), "d"(av[4]), "d"(av[2]), "d"(av[5]), "d"(av[3]),
                         "d"(bv[0]), "d"(bv[1]), "d"(bv[2]), "d"(bv[3]));
        }
      }
      // the source block staged in the next iteration -> registers
      if (b + 2 < nblocks) take(b + NKS + 1);
      if (window_bad != 0) {
        // a window of this block holds a non-finite sample: the window's own taps only, in scalar FMAs
#pragma unroll
        for (int g = 0; g < 2; ++g)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
            int u = 16 * sb + g8 + 8 * h;
            if (u >= RR) u -= RR;
            for (int t = 0; t < a.ntaps; ++t) {
              const double *p = ring + static_cast<unsigned>(u) * kUStride + lane_px_off + g * kT2;
              const double2 rg = *reinterpret_cast<const double2 *>(p);
              const double2 ba = *reinterpret_cast<const double2 *>(p + kBA);
              const double k = taps.k[t];
              s0 = fma(k, rg.x, s0); s1 = fma(k, rg.y, s1); s2 = fma(k, ba.x, s2); s3 = fma(k, ba.y, s3);
              if (++u == RR) u = 0;
            }
            acc[2 * g][2 * h] = s0; acc[2 * g][2 * h + 1] = s1; acc[2 * g + 1][2 * h] = s2; acc[2 * g + 1][2 * h + 1] = s3;
          }
      }
#pragma unroll
      for (int t = 0; t < 4; ++t)
#pragma unroll
        for (int i = 0; i < 4; ++i) prev[t][i] = acc[t][i];
      if (EPI) {
#pragma unroll
        for (int g = 0; g < 2; ++g)
#pragma unroll
          for (int h = 0; h < 2; ++h) epi_prev[g][h] = epi_cur[g][h];
      }
      prev_rem = mrem;
      st_slot = st_slot + 1 == NB ? 0 : st_slot + 1;
      if (++sb == NB) sb = 0;
    }
    output(prev, epi_prev, prev_rem);
  }
}

template <int NKS, int AXIS, int EPI>
int launch_wide(const MmaArgs &a, const double *taps_host, cudaStream_t stream) {
  constexpr int RR = 16 * (NKS + 1);
  constexpr int kWarpDoubles = AXIS == 1 ? RR * 36 : 16 * (2 * RR + 8);
  constexpr size_t smem = 4 * (kWarpDoubles * sizeof(double) + kWideStages * kWideBoxBytes) + 128;
  WideTaps<NKS> taps;
  for (int i = 0; i < 16 * NKS; ++i) taps.k[i] = i < a.ntaps ? taps_host[i] : 0.0;
  // 2 CTAs per SM: the register budget of __launch_bounds__(128, 2), and the rings plus the 1 KB the SM reserves per CTA
  constexpr int kCtasPerSm = 2;
  static_assert(kCtasPerSm * (smem + 1024) <= 228 * 1024, "two CTAs' rings must fit in an SM's shared memory");
  // Column pass: 128-byte box rows, and the neighbouring band's 128 bytes belong to another warp at another point of its
  // run, so the L2 fetches what a box reads and no more.
  CUtensorMap tmap;
  if (!make_rgba_tensor_map(static_cast<const float *>(a.src), a.width, a.height, AXIS == 1 ? 32 : 64, AXIS == 1 ? 16 : 8,
                            CU_TENSOR_MAP_SWIZZLE_NONE,
                            AXIS == 1 ? CU_TENSOR_MAP_L2_PROMOTION_L2_128B : CU_TENSOR_MAP_L2_PROMOTION_L2_256B, &tmap))
    return MB200_EUNSUPPORTED;                     // no tensor-map encoder in the driver: the caller's DFMA kernels
  auto kernel = conv_mma_wide_kernel<NKS, AXIS, EPI>;
  // per device attribute: set on every launch (a few microseconds)
  cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  const long long lines = AXIS == 1 ? a.width : a.height, len = AXIS == 1 ? a.height : a.width;
  const long long tiles = (lines + 7) / 8 * ((len + a.strip - 1) / a.strip);
  const int grid = static_cast<int>(std::min<long long>(static_cast<long long>(kCtasPerSm) * sm_count(), (tiles + 3) / 4));
  kernel<<<grid, 128, smem, stream>>>(a, taps, tmap);
  count_launch();
  count_family(kConvMma);
  count_family(kConvMmaWide);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "conv_mma_wide launch");
  return MB200_OK;
}

template <int NKS>
int launch_wide_nks(const MmaArgs &a, const double *taps_host, int axis, bool epi, cudaStream_t stream) {
  if (axis == 0) return launch_wide<NKS, 0, 0>(a, taps_host, stream);
  if (epi) return launch_wide<NKS, 1, 1>(a, taps_host, stream);
  return launch_wide<NKS, 1, 0>(a, taps_host, stream);
}

template <int NKS, int AXIS, int IO, int EPI>
int launch_one(const MmaArgs &a, const MmaTaps<NKS> &taps, int minb, cudaStream_t stream) {
  constexpr int NB = (4 * NKS - 8) / 8 + 2, RR = 8 * NB;
  constexpr int kWarpDoubles = AXIS == 1 ? RR * 36 : 16 * (2 * RR + 8);
  constexpr size_t smem = 4 * kWarpDoubles * sizeof(double);
  dim3 grid;
  if (AXIS == 1) grid = dim3((a.width + 31) / 32, (a.height + a.strip - 1) / a.strip);
  else grid = dim3((a.width + a.strip - 1) / a.strip, (a.height + 31) / 32);
  if (grid.y > 65535) return MB200_EUNSUPPORTED;
  auto go = [&](auto kernel) {
    if (smem > 48 * 1024) cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    kernel<<<grid, 128, smem, stream>>>(a, taps);
  };
  if (minb >= 4) go(conv_mma_kernel<NKS, AXIS, IO, EPI, 4>);
  else go(conv_mma_kernel<NKS, AXIS, IO, EPI, 3>);
  count_launch();
  count_family(kConvMma);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "conv_mma launch");
  return MB200_OK;
}

template <int NKS>
int launch_nks(const MmaArgs &a, const double *taps_host, int axis, int io, bool epi, int minb, cudaStream_t stream) {
  MmaTaps<NKS> taps;
  for (int i = 0; i < 4 * NKS; ++i) taps.k[i] = i < a.ntaps ? taps_host[i] : 0.0;
  if (axis == 1) {
    if (io == 1) return launch_one<NKS, 1, 1, 0>(a, taps, minb, stream);
    if (io == 2) return launch_one<NKS, 1, 2, 0>(a, taps, minb, stream);
    if (epi) return launch_one<NKS, 1, 0, 1>(a, taps, minb, stream);
    return launch_one<NKS, 1, 0, 0>(a, taps, minb, stream);
  }
  if (io == 1) return launch_one<NKS, 0, 1, 0>(a, taps, minb, stream);
  if (io == 2) return launch_one<NKS, 0, 2, 0>(a, taps, minb, stream);
  return launch_one<NKS, 0, 0, 0>(a, taps, minb, stream);
}

}  // namespace

// RGBA, bias 0, 16-byte aligned images, <= 33 taps.  MB200_EUNSUPPORTED => the caller uses the DFMA kernels of conv1d.cu.
int launch_conv_mma(const void *src, void *dst, size_t width, size_t height, int axis, const double *taps, int ntaps,
                    int origin_offset, void *stream, int io, const UnsharpEpilogue *epilogue, bool *epilogue_fused) {
  if (epilogue_fused) *epilogue_fused = false;
  // Default (-1): every float-in / float-out pass of <= 33 taps: one DMMA carries 256 FMAs where the DFMA kernels are
  // bound by issue slots next to the FP64 pipe (the two paths have not been timed against each other on the H100).  The rank-1 passes with a double intermediate (io 1 / 2) keep the DFMA
  // kernels.
  const TuningKnobs knobs = tuning_knobs();
  const int mode = knobs.conv_mma;
  if (mode == 0 || (mode < 0 && io != 0)) return MB200_EUNSUPPORTED;
  if (ntaps < 1 || ntaps > 33 || width * 32 > 0x7fffffffull || height > 0x3fffffffull) return MB200_EUNSUPPORTED;
  if (((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) != 0) return MB200_EUNSUPPORTED;
  MmaArgs a{};
  a.src = src; a.dst = dst;
  a.width = static_cast<int>(width); a.height = static_cast<int>(height);
  a.off = origin_offset;
  a.ntaps = ntaps;
  a.strip = (knobs.mma_strip + 7) & ~7;
  // -1: windows of <= 9 taps (measured: 9 taps 1.05 -> 0.98 ms, 25 taps 1.37 -> 1.40 ms)
  a.l2pf = knobs.mma_l2pf < 0 ? (ntaps <= 9 ? 1 : 0) : knobs.mma_l2pf;
  const bool epi = axis == 1 && io == 0 && epilogue && epilogue->source && (reinterpret_cast<uintptr_t>(epilogue->source) & 15) == 0;
  if (epi) { a.aux = epilogue->source; a.gain = epilogue->gain; a.qthreshold = epilogue->quantum_threshold; }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  int rc;
  // The wide tiles for windows of 18-33 taps (DESIGN §5.1); shorter windows keep the 8x8x4 tiles, since 47-72 % of a
  // 16-row band tile would be zeros.  Wide strips start at multiples of 16 so that the bits do not depend on mma_strip.
  if (io == 0 && ntaps >= 18 && knobs.mma_wide != 0) {
    a.strip = (knobs.mma_strip + 15) & ~15;
    rc = launch_wide_nks<3>(a, taps, axis, epi, s);
  } else if (ntaps <= 9) rc = launch_nks<4>(a, taps, axis, io, epi, knobs.mma_minb, s);
  else if (ntaps <= 17) rc = launch_nks<6>(a, taps, axis, io, epi, knobs.mma_minb, s);
  else if (ntaps <= 25) rc = launch_nks<8>(a, taps, axis, io, epi, knobs.mma_minb, s);
  else rc = launch_nks<10>(a, taps, axis, io, epi, knobs.mma_minb, s);
  if (rc == MB200_OK && epilogue_fused) *epilogue_fused = epi;
  return rc;
}

}  // namespace mb200
