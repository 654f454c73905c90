// resize_stream.cu -- streaming kernels for one axis of ResizeImage over UNIFORM SEGMENTS of the
// contribution table (integer-ratio reductions).
//
// HorizontalFilter / VerticalFilter (MagickCore/resize.c:3333-3547, :3549-3759) evaluate the filter
// weights per output from  bisect = (o + 0.5)/factor + MagickEpsilon  (:3398-3443).  For an integer
// reduction ratio  start - bisect  is the same real number for every output, and in floating point it
// is the same double for every output whose bisect lies in the same binade (the epsilon is absorbed
// identically).  The reference's table therefore consists of a dozen runs of outputs with
// BIT-IDENTICAL weights, the same tap count N and a window that advances by S samples per output
// (8192 -> 4096 Lanczos3: runs of 96, 384 and 3581 outputs cover all but 35 of them).  The host
// (api.cu) finds those runs by comparing the reference's own weights bit for bit; nothing is
// approximated.
//
// Inside a run the operator is a strided 1-D convolution, so it is evaluated like conv1d.cu: a
// thread walks ALONG the filtered axis over a strip of outputs and keeps the R = ceil(N/S) outputs
// whose windows contain the current source sample as rotating FP64 accumulators in registers; the N
// weights live in registers for the whole strip.  Every source sample is loaded, converted and
// alpha-premultiplied exactly once and feeds <= R x 4 FMAs in the reference's tap order; one output
// completes every S steps (double accumulation, one rounding to float, resize.c:3472-3484).
//
//  vertical (axis 1): lane = pixel column, 512-byte coalesced row reads, register prefetch ring.
//  horizontal (axis 0): lane = image row.  Each warp stages 16-pixel (256-byte, line-aligned)
//    chunks of its 32 rows into a private shared-memory ring -- by TMA (two cp.async.bulk.tensor.2d boxes of
//    8 pixels x 32 rows per chunk, 128-byte swizzle, mbarrier transaction counts; resize_h_tma_kernel, the default) or
//    with per-lane cp.async (LDGSTS; resize_h_stream_kernel) -- full-line global requests, no block barriers -- and
//    reads its own row back with conflict-free LDS.128.  Outputs are 16-byte stores; eight consecutive steps of a lane
//    fill a line.
//
// Outputs outside the streamed runs (the image borders, where the window is clipped, and the very
// short low-binade runs) are produced by the generic gather kernels of resize.cu.
#include "launch.cuh"

#include "tma.cuh"

#include <cuda_runtime.h>

#include <algorithm>
#include <cstdlib>

namespace mb200 {
namespace {

constexpr double kQuantumScale = 1.0 / 65535.0;
constexpr double kEpsilon = 1.0e-12;
constexpr int kMaxSegments = MB200_RESIZE_MAX_SEGMENTS;

struct StreamArgs {
  const float *src;
  float *dst;
  int width, height;      // source image
  int out_w, out_h;       // destination image
  int in_n;               // source extent along the filtered axis
  int strip;              // outputs per strip
  int nseg;
  int seg_o[kMaxSegments];        // first output of the run
  int seg_n[kMaxSegments];        // outputs in the run
  int seg_src[kMaxSegments];      // start[] of its first output
  int seg_strip0[kMaxSegments];   // index of its first strip
  const double *wsets;            // [nseg][N] weights of each run
  int nstrips;                    // CTAs beyond the strips produce the border outputs (gather)
  int nborder, out_n;
  const int *border;              // outputs outside the runs
  const int *start, *count;       // the reference's contribution table (resize.cu layout)
  const double *weights;          // tap-major [tap][out_n]
};

// 1/g to ~1 ulp: MUFU.RCP64H seed + two Newton steps (same helper as conv1d.cu).
__device__ __forceinline__ double fast_reciprocal(double g) {
  double r0;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r0) : "d"(g));
  const double e0 = fma(-g, r0, 1.0);
  const double r1 = fma(r0, e0, r0);              // ~2^-40
  const double e1 = fma(-g, r1, 1.0);
  return fma(r1, e1, r1);                         // ~1 ulp of double: keeps the first pass of a two-pass operator
}                                                 // bit-identical to the reference's quotient in all but ~1e-8 of the samples

// resize.c:3472-3484 for RGBA with acc[3] = sum w*A (QuantumScale cancels), acc[c] = sum w*A*p_c:
// out_c = PerceptibleReciprocal(QS*acc[3]) * QS*acc[c]; branch-free by clamping the denominator.
__device__ __forceinline__ float4 finish_rgba(const double (&acc)[4]) {
  constexpr double kTiny = kEpsilon / kQuantumScale;
  const bool perceptible = fabs(kQuantumScale * acc[3]) >= kEpsilon;
  const double den = perceptible ? acc[3] : (acc[3] < 0.0 ? -kTiny : kTiny);
  const double r = fast_reciprocal(den);
  return make_float4(static_cast<float>(r * acc[0]), static_cast<float>(r * acc[1]), static_cast<float>(r * acc[2]),
                     static_cast<float>(acc[3]));
}

template <int S, int N>
struct Rot {
  static constexpr int R = (N + S - 1) / S;     // live outputs
  static constexpr int P = R * S;               // rotation period in source steps
  static constexpr int BODY = P < 8 ? 8 : P;    // unrolled steps per loop iteration (multiple of P)
  static constexpr int PF = BODY % 12 == 0 ? 12 : BODY % 8 == 0 ? 8 : BODY % 7 == 0 ? 7 : BODY % 6 == 0 ? 6 : 4;
  static_assert(BODY % P == 0 && BODY % PF == 0, "ring / period mismatch");
};

// one source sample into the live accumulators; m = step within the rotation period (static).
// Slot q holds the output whose window started at step S*q of this (or the previous) period.  A window's first tap
// starts its sum from +0 as the reference's pixel = 0.0 does (resize.c:3493): fma(w, q, +0) is w*q except that a -0
// product becomes +0, so a window of -0 products gives +0, not -0.  Same DFMA pipe as the DMUL it replaces.
template <int S, int N>
__device__ __forceinline__ void feed(double (&acc)[Rot<S, N>::R][4], const double (&W)[N], const float4 v, int m) {
  constexpr int R = Rot<S, N>::R, P = Rot<S, N>::P;
  const double a = static_cast<double>(v.w);
  const double q0 = static_cast<double>(v.x) * a, q1 = static_cast<double>(v.y) * a, q2 = static_cast<double>(v.z) * a;
#pragma unroll
  for (int q = 0; q < R; ++q) {
    const int j = (m - S * q + 2 * P) % P;        // tap index of this sample in slot q's window
    if (j == 0) {
      acc[q][0] = fma(W[0], q0, 0.0);
      acc[q][1] = fma(W[0], q1, 0.0);
      acc[q][2] = fma(W[0], q2, 0.0);
      acc[q][3] = fma(W[0], a, 0.0);
    } else if (j < N) {
      acc[q][0] = fma(W[j], q0, acc[q][0]);
      acc[q][1] = fma(W[j], q1, acc[q][1]);
      acc[q][2] = fma(W[j], q2, acc[q][2]);
      acc[q][3] = fma(W[j], a, acc[q][3]);
    }
  }
}
// slot that receives its last tap at step m of the period, or -1
template <int S, int N>
__device__ __forceinline__ constexpr int done_slot(int m) {
  constexpr int P = Rot<S, N>::P;
  const int jd = (m - (N - 1) + 2 * P) % P;
  return jd % S == 0 ? jd / S : -1;
}

// One border output (window clipped by the image edge, or a run too short to stream): plain gather
// over the reference's contribution list.  axis 1: line = column x; axis 0: line = row y.
template <int AXIS>
__device__ __forceinline__ void border_output(const StreamArgs &a, int o, int line) {
  const int first = __ldg(a.start + o), n = __ldg(a.count + o);
  if (n <= 0) return;                                 // resize.c:3440 leaves the output untouched
  const size_t step = AXIS == 1 ? static_cast<size_t>(a.width) * 4 : 4;
  const float *p = AXIS == 1 ? a.src + (static_cast<size_t>(first) * a.width + line) * 4
                             : a.src + (static_cast<size_t>(line) * a.width + first) * 4;
  double acc[4] = {0.0, 0.0, 0.0, 0.0};
  for (int j = 0; j < n; ++j, p += step) {
    const double w = __ldg(a.weights + static_cast<size_t>(j) * a.out_n + o);
    const float4 v = __ldg(reinterpret_cast<const float4 *>(p));
    const double al = static_cast<double>(v.w);
    acc[0] = fma(w, static_cast<double>(v.x) * al, acc[0]);
    acc[1] = fma(w, static_cast<double>(v.y) * al, acc[1]);
    acc[2] = fma(w, static_cast<double>(v.z) * al, acc[2]);
    acc[3] = fma(w, al, acc[3]);
  }
  float *q = AXIS == 1 ? a.dst + (static_cast<size_t>(o) * a.out_w + line) * 4
                       : a.dst + (static_cast<size_t>(line) * a.out_w + o) * 4;
  *reinterpret_cast<float4 *>(q) = finish_rgba(acc);
}

struct Strip { int o0, nout, src0, set; };
__device__ __forceinline__ Strip locate(const StreamArgs &a, int b, int stride) {
  int k = 0;
#pragma unroll
  for (int t = 1; t < kMaxSegments; ++t)
    if (t < a.nseg && b >= a.seg_strip0[t]) k = t;
  const int rel = (b - a.seg_strip0[k]) * a.strip;
  Strip s;
  s.o0 = a.seg_o[k] + rel;
  s.nout = min(a.strip, a.seg_n[k] - rel);
  s.src0 = a.seg_src[k] + stride * rel;
  s.set = k;
  return s;
}

// ---------------------------------------------------------------------------------- vertical
// grid (ceil(width/128), total strips); thread = one RGBA pixel column.
template <int S, int N>
__global__ void __launch_bounds__(128, 3) resize_v_stream_kernel(const StreamArgs a) {
  using T = Rot<S, N>;
  constexpr int R = T::R, P = T::P, BODY = T::BODY, PF = T::PF;
  const int x_raw = blockIdx.x * 128 + threadIdx.x;
  const bool active = x_raw < a.width;
  const int x = active ? x_raw : a.width - 1;
  if (static_cast<int>(blockIdx.y) >= a.nstrips) {   // border rows: one output row per CTA row
    if (active) border_output<1>(a, __ldg(a.border + (blockIdx.y - a.nstrips)), x);
    return;
  }
  const Strip st = locate(a, blockIdx.y, S);
  double W[N];
#pragma unroll
  for (int j = 0; j < N; ++j) W[j] = __ldg(a.wsets + st.set * N + j);
  const int niter = (S * (st.nout - 1) + N + BODY - 1) / BODY;
  const size_t pitch = static_cast<size_t>(a.width) * 4;
  const float *col = a.src + static_cast<size_t>(x) * 4;
  // loads past the strip's last tap (ring over-run, rounded-up last iteration) re-read that row from L1
  const int last = min(a.in_n - 1, st.src0 + S * (st.nout - 1) + N - 1);
  int row = st.src0;                                 // source row of the next ring load
  float4 pre[PF];
#pragma unroll
  for (int s = 0; s < PF; ++s, ++row)
    pre[s] = __ldg(reinterpret_cast<const float4 *>(col + static_cast<size_t>(min(row, last)) * pitch));
  double acc[R][4];
#pragma unroll
  for (int q = 0; q < R; ++q) { acc[q][0] = acc[q][1] = acc[q][2] = acc[q][3] = 0.0; }
  int c = -R;                                        // R-1 slots complete once before output 0 does
  const size_t opitch = static_cast<size_t>(a.out_w) * 4;
  float *outp = a.dst + (static_cast<ptrdiff_t>(st.o0 - (R - 1)) * a.out_w + x) * 4;
#pragma unroll 1
  for (int t = 0; t < niter; ++t) {
#pragma unroll
    for (int b = 0; b < BODY; ++b) {
      const int m = b % P;
      const float4 v = pre[b % PF];
      pre[b % PF] = __ldg(reinterpret_cast<const float4 *>(col + static_cast<size_t>(min(row, last)) * pitch));
      ++row;
      feed<S, N>(acc, W, v, m);
      const int qd = done_slot<S, N>(m);
      if (qd >= 0) {
        ++c;
        if (c >= 0 && c < st.nout && active) *reinterpret_cast<float4 *>(outp) = finish_rgba(acc[qd]);
        outp += opitch;
      }
    }
  }
}

// -------------------------------------------------------------------------------- horizontal
// grid (total strips, ceil(height/128)); warp = 32 rows (lane = row), private cp.async ring.
// CHUNK = pixels per row per ring slot: 8 (128 B, one line) or 16 (256 B: better DRAM page locality, half the
// resident warps).  Row pitch = CHUNK*16 + 16 bytes: an odd multiple of 16 => (pitch/16 * row + k) mod 8 distinct.
template <int CHUNK> struct HRing {
  static constexpr int kRowPitch = CHUNK * 16 + 16;
  static constexpr int kSlotBytes = 32 * kRowPitch;
};

__device__ __forceinline__ void cp_async16(unsigned smem_addr, const void *gptr) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_addr), "l"(gptr));
}
// volatile orders these among themselves and with the LDS below; no "memory" clobber so that the
// output stores stay free to move across them.
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;"); }
template <int K>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(K)); }

template <int S, int N, int NSLOT, int MINB, int CHUNK>
__global__ void __launch_bounds__(128, MINB) resize_h_stream_kernel(const StreamArgs a) {
  using T = Rot<S, N>;
  constexpr int kChunkPx = CHUNK, kRowPitch = HRing<CHUNK>::kRowPitch, kSlotBytes = HRing<CHUNK>::kSlotBytes;
  constexpr int kLanesPerRow = CHUNK, kRowsPerInstr = 32 / CHUNK, kInstr = 32 / kRowsPerInstr;
  constexpr int R = T::R, P = T::P, BODY = T::BODY;
  extern __shared__ __align__(128) unsigned char ring_all[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned ring_s =
      static_cast<unsigned>(__cvta_generic_to_shared(ring_all + static_cast<size_t>(warp) * NSLOT * kSlotBytes));
  const int row0 = blockIdx.y * 128 + warp * 32;
  if (row0 >= a.height) return;
  if (static_cast<int>(blockIdx.x) >= a.nstrips) {   // border columns: thread = row, CTA = one output column
    if (row0 + lane < a.height) border_output<0>(a, __ldg(a.border + (blockIdx.x - a.nstrips)), row0 + lane);
    return;
  }
  const Strip st = locate(a, blockIdx.x, S);
  double W[N];
#pragma unroll
  for (int j = 0; j < N; ++j) W[j] = __ldg(a.wsets + st.set * N + j);
  const int niter = (S * (st.nout - 1) + N + BODY - 1) / BODY;
  const int p0 = st.src0;                            // absolute source pixel of step 0
  const int c0 = p0 / kChunkPx;                      // first chunk (line aligned)
  const int nchunks = (p0 + S * (st.nout - 1) + N + kChunkPx - 1) / kChunkPx - c0;   // steps past the last tap read stale slots
  // loader role: instruction j copies pixel (lane % CHUNK) of row (32/CHUNK)*j + lane / CHUNK
  const int lrow = lane / kLanesPerRow, lpx = lane % kLanesPerRow;
  const size_t pitch_b = static_cast<size_t>(a.width) * 16;
  const unsigned char *srcb = reinterpret_cast<const unsigned char *>(a.src);
  const int last_px = a.in_n - 1;
  auto issue = [&](int chunk_rel) {
    if (chunk_rel < nchunks) {
      const int px = min((c0 + chunk_rel) * kChunkPx + lpx, last_px);
      const unsigned slot = ring_s + static_cast<unsigned>(chunk_rel % NSLOT) * kSlotBytes;
#pragma unroll
      for (int j = 0; j < kInstr; ++j) {
        const int r = kRowsPerInstr * j + lrow;
        const int y = min(row0 + r, a.height - 1);
        cp_async16(slot + r * kRowPitch + lpx * 16, srcb + static_cast<size_t>(y) * pitch_b + static_cast<size_t>(px) * 16);
      }
    }
    cp_async_commit();
  };
#pragma unroll
  for (int c = 0; c < NSLOT; ++c) issue(c);

  const int y = row0 + lane;
  const bool active = y < a.height;
  double acc[R][4];
#pragma unroll
  for (int q = 0; q < R; ++q) { acc[q][0] = acc[q][1] = acc[q][2] = acc[q][3] = 0.0; }
  int c = -R;
  float *outp = a.dst + (static_cast<ptrdiff_t>(active ? y : 0) * a.out_w + (st.o0 - (R - 1))) * 4;
  int chunk = 0;                                    // chunk being consumed (relative)
  int px_in = p0 - c0 * kChunkPx;                   // pixel within the chunk
  cp_async_wait<NSLOT - 1>();
  __syncwarp();
  unsigned rd = ring_s + lane * kRowPitch + px_in * 16;   // this lane's next LDS address (slot 0)
  float4 vnext;                                            // sample of the next step (LDS one step ahead)
  asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(vnext.x), "=f"(vnext.y), "=f"(vnext.z), "=f"(vnext.w) : "r"(rd));
#pragma unroll 1
  for (int t = 0; t < niter; ++t) {
#pragma unroll
    for (int b = 0; b < BODY; ++b) {
      const int m = b % P;
      const float4 v = vnext;
      rd += 16;
      if (++px_in == kChunkPx) {                    // warp-uniform: chunk exhausted
        px_in = 0;
        __syncwarp();                               // every lane is done reading the slot
        issue(chunk + NSLOT);                       // refill it (same slot: (chunk + NSLOT) % NSLOT)
        ++chunk;
        cp_async_wait<NSLOT - 1>();                 // chunk is complete; NSLOT-1 later ones stay in flight
        __syncwarp();
        rd = ring_s + static_cast<unsigned>(chunk % NSLOT) * kSlotBytes + lane * kRowPitch;
      }
      asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(vnext.x), "=f"(vnext.y), "=f"(vnext.z), "=f"(vnext.w) : "r"(rd));
      feed<S, N>(acc, W, v, m);
      const int qd = done_slot<S, N>(m);
      if (qd >= 0) {
        ++c;
        if (c >= 0 && c < st.nout && active) *reinterpret_cast<float4 *>(outp) = finish_rgba(acc[qd]);
        outp += 4;
      }
    }
  }
  cp_async_wait<0>();
}

// ------------------------------------------------------------------------ horizontal, TMA staging
// The same streaming loop as resize_h_stream_kernel; only the way the 16-pixel chunks reach the warp's ring differs.
// One elected lane issues two cp.async.bulk.tensor.2d loads per chunk (box = 8 pixels x 32 rows = 128 B x 32 with the
// 128-byte swizzle: the 16-byte word a lane reads from its row is XORed with row % 8, so the eight rows of a quarter warp
// hit eight different bank groups -- conflict-free LDS.128 without the padded pitch) and the chunk's arrival is an
// mbarrier transaction count instead of cp.async groups: no per-lane copy instructions, no bank-conflicted ring writes
// (a third of the shared-memory wavefronts of the cp.async ring's writes conflict).
// Rows / pixels outside the image are zero-filled by the TMA unit; the streamed runs never read them into a stored
// output (clipped windows are border outputs, gathered by the extra CTAs).
template <int S, int N, int NSLOT, int MINB, int BOXES = 2>
__global__ void __launch_bounds__(128, MINB) resize_h_tma_kernel(const StreamArgs a, const __grid_constant__ CUtensorMap tmap) {
  using T = Rot<S, N>;
  constexpr int kChunkPx = 8 * BOXES, kBoxBytes = 32 * 128, kSlotBytes = BOXES * kBoxBytes;
  constexpr int R = T::R, P = T::P, BODY = T::BODY;
  extern __shared__ __align__(1024) unsigned char ring_all[];
  __shared__ __align__(8) unsigned long long bars[4][NSLOT];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // the 128-byte swizzle is a function of the shared-memory ADDRESS: slots must start on 1024-byte boundaries
  const unsigned ring_base = (static_cast<unsigned>(__cvta_generic_to_shared(ring_all)) + 1023u) & ~1023u;
  const unsigned ring_s = ring_base + static_cast<unsigned>(warp) * NSLOT * kSlotBytes;
  const unsigned bar_s = static_cast<unsigned>(__cvta_generic_to_shared(&bars[warp][0]));
  const int row0 = blockIdx.y * 128 + warp * 32;
  if (row0 >= a.height) return;
  if (static_cast<int>(blockIdx.x) >= a.nstrips) {
    if (row0 + lane < a.height) border_output<0>(a, __ldg(a.border + (blockIdx.x - a.nstrips)), row0 + lane);
    return;
  }
  const Strip st = locate(a, blockIdx.x, S);
  double W[N];
#pragma unroll
  for (int j = 0; j < N; ++j) W[j] = __ldg(a.wsets + st.set * N + j);
  const int niter = (S * (st.nout - 1) + N + BODY - 1) / BODY;
  const int p0 = st.src0;
  const int c0 = p0 / kChunkPx;
  const int nchunks = (p0 + S * (st.nout - 1) + N + kChunkPx - 1) / kChunkPx - c0;
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < NSLOT; ++k) mbar_init(bar_s + 8 * k, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncwarp();
  auto issue = [&](int chunk_rel) {                 // elected lane: two boxes of 8 pixels x 32 rows into the chunk's slot
    if (lane == 0 && chunk_rel < nchunks) {
      const int k = chunk_rel % NSLOT;
      const unsigned slot = ring_s + static_cast<unsigned>(k) * kSlotBytes, bar = bar_s + 8 * k;
      const int x = (c0 + chunk_rel) * kChunkPx * 4;  // float index of the chunk's first pixel
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // the slot's last generic-proxy reads precede the refill
      mbar_expect_tx(bar, kSlotBytes);
      tma_load_2d(slot, &tmap, x, row0, bar);
      if (BOXES == 2) tma_load_2d(slot + kBoxBytes, &tmap, x + 32, row0, bar);
    }
  };
#pragma unroll
  for (int c = 0; c < NSLOT; ++c) issue(c);

  const int y = row0 + lane;
  const bool active = y < a.height;
  double acc[R][4];
#pragma unroll
  for (int q = 0; q < R; ++q) { acc[q][0] = acc[q][1] = acc[q][2] = acc[q][3] = 0.0; }
  int c = -R;
  float *outp = a.dst + (static_cast<ptrdiff_t>(active ? y : 0) * a.out_w + (st.o0 - (R - 1))) * 4;
  int chunk = 0;
  int px_in = p0 - c0 * kChunkPx;
  const unsigned row_off = lane * 128, swz = lane & 7;
  // address of pixel p (0..15) of this lane's row inside a slot: box p/8, 16-byte word (p%8) ^ (row%8)
  auto addr = [&](unsigned slot, int p) {
    return slot + static_cast<unsigned>(p >> 3) * kBoxBytes + row_off + ((static_cast<unsigned>(p & 7) ^ swz) << 4);
  };
  mbar_wait(bar_s, 0);
  unsigned slot_s = ring_s;
  float4 vnext;
  asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(vnext.x), "=f"(vnext.y), "=f"(vnext.z), "=f"(vnext.w) : "r"(addr(slot_s, px_in)));
#pragma unroll 1
  for (int t = 0; t < niter; ++t) {
#pragma unroll
    for (int b = 0; b < BODY; ++b) {
      const int m = b % P;
      const float4 v = vnext;
      if (++px_in == kChunkPx) {                    // warp-uniform: chunk exhausted
        px_in = 0;
        __syncwarp();                               // every lane is done reading the slot
        issue(chunk + NSLOT);                       // refill it
        ++chunk;
        const int k = chunk % NSLOT;
        if (chunk < nchunks) mbar_wait(bar_s + 8 * k, static_cast<unsigned>(chunk / NSLOT) & 1u);
        slot_s = ring_s + static_cast<unsigned>(k) * kSlotBytes;
      }
      asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(vnext.x), "=f"(vnext.y), "=f"(vnext.z), "=f"(vnext.w) : "r"(addr(slot_s, px_in)));
      feed<S, N>(acc, W, v, m);
      const int qd = done_slot<S, N>(m);
      if (qd >= 0) {
        ++c;
        if (c >= 0 && c < st.nout && active) *reinterpret_cast<float4 *>(outp) = finish_rgba(acc[qd]);
        outp += 4;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------ fused V + H
// ResizeImage with the SAME integer reduction on both axes (x_factor == y_factor: the reference filters vertically
// first, resize.c:3854-3861).  The two-pass form moves 36 B per input pixel through HBM (16 + 8 for the vertical pass,
// 8 + 4 for the horizontal one); here the vertically filtered intermediate of one output tile lives in shared memory --
// as float, i.e. with the reference's rounding between the passes -- and HBM sees the source once (plus tile halos,
// which the L2 absorbs) and the result: 20 B per input pixel (SURVEY 8d).
//   CTA = 128 threads, output tile TW x TH = (4*NW) x 31, both inside ONE run of bit-identical weights per axis.
//   phase A: thread = source column of the tile (S*(TW-1)+N <= 128 columns), the vertical kernel's streaming loop over
//            S*(TH-1)+N source rows (72 = 6 rotation periods for S=2, N=12): register prefetch ring, rotating FP64
//            accumulators, weights in registers; finished rows go to the shared tile [TH][128] float4 (row pitch
//            128*16+16 B: rows are read lane-wise in phase B, the odd pitch keeps LDS.128 conflict free);
//   phase B: lane = output row, warp w = output columns [NW*w, NW*w + NW): the horizontal kernel's streaming loop along
//            the shared tile (S*(NW-1)+N = 36 samples = 3 periods for NW = 13), 16-byte stores.
// Outputs outside the runs (clipped windows at the image border, very short low-binade runs) are produced by
// resize_border2d_kernel below from the reference's contribution lists.
struct Tile { int o0, nout, src0, set; };
struct FusedArgs {
  const float *src;
  float *dst;
  int width, height, out_w, out_h;
  const Tile *xt, *yt;          // tiles of the x / y runs (device)
  const double *wx, *wy;        // [run][N] weights
};

// Phase B of warp w reads the tile row from sample S*NW*w up to niter*BODY + 1 samples further: inside the 128 columns
// phase A filled for the last warp, whose source span S*(4*NW-1)+N must itself fit them.
template <int S, int N>
constexpr bool fused_fits(int nw) {
  return S * (4 * nw - 1) + N <= 128 &&
         S * 3 * nw + ((S * (nw - 1) + N + Rot<S, N>::BODY - 1) / Rot<S, N>::BODY) * Rot<S, N>::BODY + 1 <= 128;
}
template <int S, int N>
constexpr int fused_nw() {
  int nw = 13;
  while (nw > 1 && !fused_fits<S, N>(nw)) --nw;
  return nw;
}

template <int S, int N> struct FusedGeom {
  static constexpr int P = Rot<S, N>::P;
  static constexpr int TH = 31;                                  // S*(TH-1)+N = 72 = 6*P for S=2, N=12
  static constexpr int NW = fused_nw<S, N>();                    // output columns per warp in phase B
  static_assert(fused_fits<S, N>(NW), "no phase-B split fits the 128-column tile");
  static constexpr int TW = 4 * NW;
  // phase-A prefetch depth: the vertical kernel's, except (2,12), whose 12-deep ring spills at 168 registers (3 CTAs / SM);
  // 6 loads of 16 B per thread still keep ~36 KB per SM in flight
  static constexpr int PF = Rot<S, N>::PF == 12 ? 6 : Rot<S, N>::PF;
  static constexpr int kPitch = 128 * 16 + 16;                   // bytes per tile row
  static constexpr int kSmem = 32 * kPitch;
};

template <int S, int N>
__global__ void __launch_bounds__(128, 3) resize_fused_kernel(const FusedArgs a) {
  using T = Rot<S, N>;
  using G = FusedGeom<S, N>;
  constexpr int R = T::R, P = T::P, BODY = T::BODY, PF = G::PF;
  extern __shared__ __align__(16) unsigned char inter[];        // [TH][kPitch]
  const Tile xt = a.xt[blockIdx.x], yt = a.yt[blockIdx.y];
  double acc[R][4];
  {
    // ---- phase A: vertical filter of column xt.src0 + threadIdx.x over the tile's rows
    double W[N];
#pragma unroll
    for (int j = 0; j < N; ++j) W[j] = __ldg(a.wy + yt.set * N + j);
    const int x = min(xt.src0 + static_cast<int>(threadIdx.x), a.width - 1);
    const int niter = (S * (yt.nout - 1) + N + BODY - 1) / BODY;
    const size_t pitch = static_cast<size_t>(a.width) * 4;
    const float *col = a.src + static_cast<size_t>(x) * 4;
    const int last = min(a.height - 1, yt.src0 + S * (yt.nout - 1) + N - 1);
    int row = yt.src0;
    float4 pre[PF];
#pragma unroll
    for (int s = 0; s < PF; ++s, ++row)
      pre[s] = __ldg(reinterpret_cast<const float4 *>(col + static_cast<size_t>(min(row, last)) * pitch));
#pragma unroll
    for (int q = 0; q < R; ++q) { acc[q][0] = acc[q][1] = acc[q][2] = acc[q][3] = 0.0; }
    int c = -R;
    unsigned char *outp = inter + static_cast<ptrdiff_t>(-(R - 1)) * G::kPitch + threadIdx.x * 16;
#pragma unroll 1
    for (int t = 0; t < niter; ++t) {
#pragma unroll
      for (int b = 0; b < BODY; ++b) {
        const int m = b % P;
        const float4 v = pre[b % PF];
        pre[b % PF] = __ldg(reinterpret_cast<const float4 *>(col + static_cast<size_t>(min(row, last)) * pitch));
        ++row;
        feed<S, N>(acc, W, v, m);
        const int qd = done_slot<S, N>(m);
        if (qd >= 0) {
          ++c;
          if (c >= 0 && c < yt.nout) *reinterpret_cast<float4 *>(outp) = finish_rgba(acc[qd]);
          outp += G::kPitch;
        }
      }
    }
  }
  __syncthreads();
  {
    // ---- phase B: horizontal filter along the shared tile; lane = output row, warp = NW output columns
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int o_first = warp * G::NW;                          // first output column of this warp within the tile
    const int nout = min(G::NW, xt.nout - o_first);
    if (nout <= 0 || lane >= yt.nout) return;
    double W[N];
#pragma unroll
    for (int j = 0; j < N; ++j) W[j] = __ldg(a.wx + xt.set * N + j);
    const int niter = (S * (nout - 1) + N + BODY - 1) / BODY;   // the last warp never reads past the tile (fused_fits)
    const unsigned char *rd = inter + static_cast<size_t>(lane) * G::kPitch + static_cast<size_t>(S * o_first) * 16;
#pragma unroll
    for (int q = 0; q < R; ++q) { acc[q][0] = acc[q][1] = acc[q][2] = acc[q][3] = 0.0; }
    int c = -R;
    float *outp = a.dst + (static_cast<size_t>(yt.o0 + lane) * a.out_w + (xt.o0 + o_first - (R - 1))) * 4;
    float4 vnext = *reinterpret_cast<const float4 *>(rd);
#pragma unroll 1
    for (int t = 0; t < niter; ++t) {
#pragma unroll
      for (int b = 0; b < BODY; ++b) {
        const int m = b % P;
        const float4 v = vnext;
        rd += 16;
        vnext = *reinterpret_cast<const float4 *>(rd);
        feed<S, N>(acc, W, v, m);
        const int qd = done_slot<S, N>(m);
        if (qd >= 0) {
          ++c;
          if (c >= 0 && c < nout) *reinterpret_cast<float4 *>(outp) = finish_rgba(acc[qd]);
          outp += 4;
        }
      }
    }
  }
}

// Outputs whose row or column lies outside the streamed runs: thread = one output pixel, the reference's two passes on
// its own neighbourhood -- vertical contribution list per source column (rounded to float like the intermediate image,
// resize.c:3854), then the horizontal list over those values.
struct Border2dArgs {
  const float *src;
  float *dst;
  int width, height, out_w, out_h;
  const int *xstart, *xcount, *ystart, *ycount;
  const double *xweights, *yweights;     // tap-major [tap][out_n]
  const int *xborder, *yborder;          // output columns / rows outside the runs
  int nxborder, nyborder;
};

__device__ __forceinline__ float4 border2d_pixel(const Border2dArgs &a, int ox, int oy) {
  const int x0 = __ldg(a.xstart + ox), nx = __ldg(a.xcount + ox), y0 = __ldg(a.ystart + oy), ny = __ldg(a.ycount + oy);
  double hacc[4] = {0.0, 0.0, 0.0, 0.0};
  for (int i = 0; i < nx; ++i) {
    double vacc[4] = {0.0, 0.0, 0.0, 0.0};
    const float *p = a.src + (static_cast<size_t>(y0) * a.width + (x0 + i)) * 4;
    for (int j = 0; j < ny; ++j, p += static_cast<size_t>(a.width) * 4) {
      const double w = __ldg(a.yweights + static_cast<size_t>(j) * a.out_h + oy);
      const float4 v = __ldg(reinterpret_cast<const float4 *>(p));
      const double al = static_cast<double>(v.w);
      vacc[0] = fma(w, static_cast<double>(v.x) * al, vacc[0]);
      vacc[1] = fma(w, static_cast<double>(v.y) * al, vacc[1]);
      vacc[2] = fma(w, static_cast<double>(v.z) * al, vacc[2]);
      vacc[3] = fma(w, al, vacc[3]);
    }
    const float4 m = finish_rgba(vacc);                        // the intermediate image's float Quantum
    const double w = __ldg(a.xweights + static_cast<size_t>(i) * a.out_w + ox);
    const double al = static_cast<double>(m.w);
    hacc[0] = fma(w, static_cast<double>(m.x) * al, hacc[0]);
    hacc[1] = fma(w, static_cast<double>(m.y) * al, hacc[1]);
    hacc[2] = fma(w, static_cast<double>(m.z) * al, hacc[2]);
    hacc[3] = fma(w, al, hacc[3]);
  }
  return finish_rgba(hacc);
}

// grid.y = 0: border rows x all columns; grid.y = 1: border columns x the rows that are NOT border rows (no double work)
__global__ void __launch_bounds__(128) resize_border2d_kernel(const Border2dArgs a, const unsigned char *__restrict__ row_is_border) {
  const size_t i = static_cast<size_t>(blockIdx.x) * 128 + threadIdx.x;
  int ox, oy;
  if (blockIdx.y == 0) {
    if (i >= static_cast<size_t>(a.nyborder) * a.out_w) return;
    oy = __ldg(a.yborder + i / a.out_w);
    ox = static_cast<int>(i % a.out_w);
  } else {
    if (i >= static_cast<size_t>(a.nxborder) * a.out_h) return;
    ox = __ldg(a.xborder + i / a.out_h);
    oy = static_cast<int>(i % a.out_h);
    if (row_is_border[oy]) return;
  }
  if (__ldg(a.xcount + ox) <= 0 || __ldg(a.ycount + oy) <= 0) return;
  *reinterpret_cast<float4 *>(a.dst + (static_cast<size_t>(oy) * a.out_w + ox) * 4) = border2d_pixel(a, ox, oy);
}

template <int S, int N>
int launch_fused_sn(const FusedArgs &a, int nxt, int nyt, cudaStream_t s) {
  using G = FusedGeom<S, N>;
  cudaFuncSetAttribute(resize_fused_kernel<S, N>, cudaFuncAttributeMaxDynamicSharedMemorySize, G::kSmem);
  resize_fused_kernel<S, N><<<dim3(nxt, nyt), 128, G::kSmem, s>>>(a);
  return MB200_OK;
}

}  // namespace

// Tile geometry of the fused kernel for (stride, taps): outputs per tile along x / y; 0 = no fused kernel for this pair.
void resize_fused_tile(int stride, int taps, int *tw, int *th) {
  *tw = *th = 0;
  auto set = [&](auto geom) { *tw = decltype(geom)::TW; *th = decltype(geom)::TH; };
  if (stride == 2 && taps == 12) set(FusedGeom<2, 12>{});
  else if (stride == 2 && taps == 8) set(FusedGeom<2, 8>{});
  else if (stride == 2 && taps == 4) set(FusedGeom<2, 4>{});
  else if (stride == 3 && taps == 19) set(FusedGeom<3, 19>{});
  else if (stride == 4 && taps == 24) set(FusedGeom<4, 24>{});
  else if (stride == 4 && taps == 16) set(FusedGeom<4, 16>{});
}

// Fused vertical + horizontal pass: the tiles of both axes' runs, then the two-pass path's contribution and border lists
// for the outputs outside the runs.  MB200_EUNSUPPORTED => use two passes.
int launch_resize_fused(const float *src, size_t width, size_t height, float *dst, const ResizeAxis &x,
                        const ResizeAxis &y, void *stream) {
  const int stride = x.reg_stride, taps = x.reg_taps, nxt = x.ntiles_x, nyt = y.ntiles_y;
  if (y.reg_stride != stride || y.reg_taps != taps) return MB200_EUNSUPPORTED;
  if (width > 0x3fffffffull || height > 0x3fffffffull || nxt <= 0 || nyt <= 0 || nyt > 65535) return MB200_EUNSUPPORTED;
  const size_t out_w = x.out_n, out_h = y.out_n;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  FusedArgs a{};
  a.src = src; a.dst = dst;
  a.width = static_cast<int>(width); a.height = static_cast<int>(height);
  a.out_w = static_cast<int>(out_w); a.out_h = static_cast<int>(out_h);
  a.xt = reinterpret_cast<const Tile *>(x.d_tiles_x); a.yt = reinterpret_cast<const Tile *>(y.d_tiles_y);
  a.wx = x.d_wsets; a.wy = y.d_wsets;
  int rc = MB200_EUNSUPPORTED;
  if (stride == 2 && taps == 12) rc = launch_fused_sn<2, 12>(a, nxt, nyt, s);
  else if (stride == 2 && taps == 8) rc = launch_fused_sn<2, 8>(a, nxt, nyt, s);
  else if (stride == 2 && taps == 4) rc = launch_fused_sn<2, 4>(a, nxt, nyt, s);
  else if (stride == 3 && taps == 19) rc = launch_fused_sn<3, 19>(a, nxt, nyt, s);
  else if (stride == 4 && taps == 24) rc = launch_fused_sn<4, 24>(a, nxt, nyt, s);
  else if (stride == 4 && taps == 16) rc = launch_fused_sn<4, 16>(a, nxt, nyt, s);
  if (rc != MB200_OK) return rc;
  count_launch();
  count_family(kResizeFused);
  if (x.nborder > 0 || y.nborder > 0) {
    Border2dArgs b{};
    b.src = src; b.dst = dst; b.width = a.width; b.height = a.height; b.out_w = a.out_w; b.out_h = a.out_h;
    b.xstart = x.d_start; b.xcount = x.d_count; b.ystart = y.d_start; b.ycount = y.d_count;
    b.xweights = x.d_weights; b.yweights = y.d_weights;
    b.xborder = x.d_border; b.yborder = y.d_border; b.nxborder = x.nborder; b.nyborder = y.nborder;
    const size_t work = std::max(static_cast<size_t>(y.nborder) * out_w, static_cast<size_t>(x.nborder) * out_h);
    resize_border2d_kernel<<<dim3(static_cast<unsigned>((work + 127) / 128), 2), 128, 0, s>>>(b, y.d_is_border);
    count_launch();
  }
  return launch_status("fused resize launch", 0);
}

namespace {

template <int S, int N>
int launch_sn(StreamArgs a, int axis, cudaStream_t s) {
  // MB200_RESIZE_CHUNK: 16384^2 -> 8192^2: 2.02 ms with 128-byte chunks, 1.83 ms with 256-byte chunks (the default)
  const TuningKnobs knobs = tuning_knobs();
  const int lanes_blocks = axis == 1 ? (a.width + 127) / 128 : (a.height + 127) / 128;
  int total = 0;
  for (int k = 0; k < a.nseg; ++k) total += a.seg_n[k];
  // enough CTAs for ~8 waves of all SMs x 3 resident CTAs; strips no shorter than 24 outputs
  // (runs shorter than that are single strips)
  const int want = (8 * sm_count() * 3 + lanes_blocks - 1) / lanes_blocks;
  int strip = (total + want - 1) / want;
  if (strip < 24) strip = 24;
  if (knobs.resize_strip > 0) strip = knobs.resize_strip;
  a.strip = strip;
  int nstrips = 0;
  for (int k = 0; k < a.nseg; ++k) {
    a.seg_strip0[k] = nstrips;
    nstrips += (a.seg_n[k] + strip - 1) / strip;
  }
  a.nstrips = nstrips;
  nstrips += a.nborder;
  if (nstrips <= 0 || nstrips > 65535 || lanes_blocks > 65535) return MB200_EUNSUPPORTED;
  // default: the TMA-staged ring (110 instead of 168 registers, no bank-conflicted ring writes).  0 = the cp.async ring.
  const int tma = knobs.resize_tma, chunk = knobs.resize_chunk, slots = knobs.resize_slots;
  LaunchFamily family = kResizeHStream;
  CUtensorMap tmap;
  if (axis == 0 && tma != 0 && (reinterpret_cast<uintptr_t>(a.src) & 15) == 0 &&
      make_rgba_tensor_map(a.src, a.width, a.height, 32, 32, CU_TENSOR_MAP_SWIZZLE_128B,
                           CU_TENSOR_MAP_L2_PROMOTION_L2_256B, &tmap)) {
    // TMA-staged ring: 3 slots x 8 KB per warp, 2 CTAs / SM (tma == 2: 2 slots, 3 CTAs / SM)
    family = kResizeHTma;
    if (tma == 2) {
      constexpr int smem = 4 * 2 * 8192 + 1024;
      cudaFuncSetAttribute(resize_h_tma_kernel<S, N, 2, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
      resize_h_tma_kernel<S, N, 2, 3><<<dim3(nstrips, lanes_blocks), 128, smem, s>>>(a, tmap);
    } else {
      constexpr int smem = 4 * 3 * 8192 + 1024;
      cudaFuncSetAttribute(resize_h_tma_kernel<S, N, 3, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
      resize_h_tma_kernel<S, N, 3, 2><<<dim3(nstrips, lanes_blocks), 128, smem, s>>>(a, tmap);
    }
  } else if (axis == 1) {
    family = kResizeVStream;
    resize_v_stream_kernel<S, N><<<dim3(lanes_blocks, nstrips), 128, 0, s>>>(a);
  } else if (chunk == 16 && slots == 2) {  // experiment: 256-byte chunks, 2-slot rings, 3 CTAs / SM
    constexpr int smem = 4 * 2 * HRing<16>::kSlotBytes;
    cudaFuncSetAttribute(resize_h_stream_kernel<S, N, 2, 3, 16>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    resize_h_stream_kernel<S, N, 2, 3, 16><<<dim3(nstrips, lanes_blocks), 128, smem, s>>>(a);
  } else if (chunk == 16) {                    // 256-byte chunks, 3-slot rings, 2 CTAs / SM
    constexpr int smem = 4 * 3 * HRing<16>::kSlotBytes;
    cudaFuncSetAttribute(resize_h_stream_kernel<S, N, 3, 2, 16>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);   // per device; cheap
    resize_h_stream_kernel<S, N, 3, 2, 16><<<dim3(nstrips, lanes_blocks), 128, smem, s>>>(a);
  } else if (slots == 3) {                     // 4 CTAs / SM, 3-slot rings (221 KB of shared memory per SM)
    constexpr int smem = 4 * 3 * HRing<8>::kSlotBytes;
    cudaFuncSetAttribute(resize_h_stream_kernel<S, N, 3, 4, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    resize_h_stream_kernel<S, N, 3, 4, 8><<<dim3(nstrips, lanes_blocks), 128, smem, s>>>(a);
  } else {
    constexpr int smem = 4 * 4 * HRing<8>::kSlotBytes;
    cudaFuncSetAttribute(resize_h_stream_kernel<S, N, 4, 3, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    resize_h_stream_kernel<S, N, 4, 3, 8><<<dim3(nstrips, lanes_blocks), 128, smem, s>>>(a);
  }
  count_family(family);
  return MB200_OK;
}

}  // namespace

// Streams the uniform runs of one axis (RGBA only) and gathers the remaining outputs in the same launch.
// MB200_EUNSUPPORTED => the caller uses the kernels of resize.cu for the whole axis.
int launch_resize_stream(const float *src, size_t width, size_t height, float *dst, int axis, const ResizeAxis &t,
                         void *stream) {
  const size_t out_n = t.out_n;
  const int stride = t.reg_stride, taps = t.reg_taps;
  if (t.d_wsets == nullptr || t.nseg <= 0 || t.nseg > kMaxSegments) return MB200_EUNSUPPORTED;
  if (width > 0x3fffffffull || height > 0x3fffffffull || out_n > 0x3fffffffull) return MB200_EUNSUPPORTED;
  StreamArgs a{};
  a.src = src; a.dst = dst;
  a.width = static_cast<int>(width); a.height = static_cast<int>(height);
  if (axis == 1) { a.out_w = a.width; a.out_h = static_cast<int>(out_n); a.in_n = a.height; }
  else { a.out_w = static_cast<int>(out_n); a.out_h = a.height; a.in_n = a.width; }
  a.nseg = t.nseg;
  for (int k = 0; k < t.nseg; ++k) { a.seg_o[k] = t.seg_o[k]; a.seg_n[k] = t.seg_n[k]; a.seg_src[k] = t.seg_src[k]; }
  a.wsets = t.d_wsets;
  a.nborder = t.nborder; a.border = t.d_border; a.out_n = static_cast<int>(out_n);
  a.start = t.d_start; a.count = t.d_count; a.weights = t.d_weights;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  int rc = MB200_EUNSUPPORTED;
  if (stride == 2 && taps == 12) rc = launch_sn<2, 12>(a, axis, s);        // 3-lobe filters, 2x
  else if (stride == 2 && taps == 8) rc = launch_sn<2, 8>(a, axis, s);     // 2-lobe / cubic filters, 2x
  else if (stride == 2 && taps == 4) rc = launch_sn<2, 4>(a, axis, s);     // triangle, 2x
  else if (stride == 3 && taps == 19) rc = launch_sn<3, 19>(a, axis, s);   // 3-lobe, 3x
  else if (stride == 4 && taps == 24) rc = launch_sn<4, 24>(a, axis, s);   // 3-lobe, 4x
  else if (stride == 4 && taps == 16) rc = launch_sn<4, 16>(a, axis, s);   // 2-lobe / cubic, 4x
  if (rc != MB200_OK) return rc;
  return launch_status("resize stream launch");
}

}  // namespace mb200
