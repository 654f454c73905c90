// morph_direct.cu -- the directly applied morphology methods, Distance (21) and Voronoi (22): MorphologyApply's special
// branch (MagickCore/morphology.c:3736-3776) around MorphologyPrimitiveDirect (:3242-3623).
//
// The reference sweeps the image twice in place, each output reading outputs of the same pass that were already rounded
// to float, so neither pass is a parallel prefix.  Per channel:
//   pixel = QuantumRange; pixel = min(pixel, (double) sample + k) over the non-NaN kernel cells (strictly less replaces,
//   so NaN terms never win); q = (float) pixel.
// Forward (rows down, columns right; ox = kw-kx-1, oy = kh-ky-1): the virtual region of rows y-oy .. y (Voronoi: .. y-1)
// at columns x-ox .. x+kx (edge clamped; its row y is the row before the pass, the rows above final), then the updated
// values of the ox pixels to the left.  Reverse (rows up, columns left): rows y .. y+ky of the forward result (row y
// before the pass, the rows below final) at columns x-ox .. x+kx, then the updated values of the kx pixels to the right.
//
// Both passes are one kernel, launched out of place (forward: src -> a pool temporary, reverse: temporary -> dst), so
// "the row before the pass" is simply the pass's input.  The reverse pass runs in mirrored coordinates (logical row
// Y = h-1-y, column X = w-1-x), which makes both passes the same recurrence: a row reads A rows above it up to Rr columns
// to its right (Rr = kx forward, ox reverse) and its own updated values L columns to its left.
//
// Wavefront.  A CTA is one warp and owns a band of 32 rows of one channel, one lane per row; lane r works on column
// X = t - r*s at step t, s = Rr + 1 (0 when A = 0: rows are then independent).  At step t the lane above has finished
// column X + Rr, so the rows above are final as far right as the lane reads.  The in-row recurrence stays sequential in
// the lane, in the reference's term order.  The band's rows (and the A rows above it) live in a shared-memory ring of
// RING columns per row; the input rows in a second ring.  Every 32 steps the warp loads the next 32 columns of its input
// rows (each row its own skewed window, one coalesced row at a time) and stores the 32 columns it finished, likewise.
//
// Bands chain across CTAs.  Band b reads the last A rows of band b-1 (of the same pass and channel) from global memory
// once band b-1 has published that its last row is flushed far enough (release store after a fence; acquire load,
// then L1-bypassing loads).  The band a CTA works on is taken from a per-launch atomic ticket, zeroed on the stream
// before the launch, with the band index growing with the ticket: a CTA only ever waits on a band claimed by a CTA that
// is already running, which never waits on anything but a smaller ticket, so the wait chain ends at ticket 0.  No CTA
// waits on anything else; there is no co-residency assumption and no cooperative launch.  Every wait is for a band
// that moves forward, by construction, so none retries or times out.
//
// Voronoi on an image with alpha skips the alpha sweep; the reverse launch writes the epilogue instead (SetImageAlpha-
// Channel(Deactivate), CompositeImage(CopyAlpha), Deactivate): alpha = ClampPixel(QuantumRange*(QuantumScale*a)) of the
// source, every swept channel ClampPixel(value) (composite.c:2606-2612, :2708, :2860-2863, :3562).
#include "launch.cuh"

#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <mutex>
#include <vector>

namespace mb200 {
namespace {

constexpr int kBand = 32;                               // rows per band = lanes per CTA
constexpr double kQuantumRange = 65535.0;

constexpr int kMaxTerms = 1024;                         // kernel cells per pass carried in the launch parameters

struct Term {                                           // one kernel cell: value, logical row / column offset, source
  double k;
  short dv, d;                                          // dv <= 0 rows above; d columns (negative: left)
  int live;                                             // 1: this pass's updated value of the own row (guarded, no clamp)
};

// The launch parameters, term list included (16 KB at most: parameters up to 32 KB need CUDA 12.1, which sm_90a code
// needs anyway), so a call uploads nothing and never waits for the host.
struct DirectArgs {
  const float *in;                                      // this pass's input (forward: src; reverse: the temporary)
  float *out;
  const float *alpha_src;                               // Voronoi epilogue: the source (reverse launch only)
  int nterms;
  int w, h, ch;
  int A, Rr, s;                                         // rows above, reach right, skew
  int ring_out, ring_in;                                // ring columns (powers of two)
  int nbands, nswept, epilogue;                         // epilogue: Voronoi alpha (the last channel) written here
  unsigned *ticket;
  int *progress;                                        // [nswept * nbands]: columns flushed by the band's last row
  Term terms[kMaxTerms];
};

__device__ __forceinline__ int ld_acquire(const int *p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release(int *p, int v) {
  asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

__device__ __forceinline__ float clamp_pixel(float v) {  // ClampPixel (NaN passes)
  return v < 0.0f ? 0.0f : (v >= 65535.0f ? 65535.0f : v);
}

// REV: the reverse pass (mirrored coordinates).
template <bool REV>
__global__ void __launch_bounds__(kBand) direct_sweep_kernel(const __grid_constant__ DirectArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  Term *s_terms = reinterpret_cast<Term *>(smem);
  float *out_ring = reinterpret_cast<float *>(s_terms + a.nterms);   // (A + 32) rows: A halo rows, then the band
  float *in_ring = out_ring + static_cast<size_t>(a.A + kBand) * a.ring_out;
  __shared__ unsigned s_ticket;
  const int lane = threadIdx.x;
  if (lane == 0) s_ticket = atomicAdd(a.ticket, 1u);
  __syncwarp();
  const unsigned ticket = s_ticket;
  const int w = a.w, h = a.h, ch = a.ch, mask = a.ring_out - 1, mask_in = a.ring_in - 1;
  auto gidx = [&](int Y, int X, int c) -> size_t {      // logical (Y, X) -> interleaved physical index
    const int y = REV ? h - 1 - Y : Y, x = REV ? w - 1 - X : X;
    return (static_cast<size_t>(y) * w + x) * ch + c;
  };

  const unsigned swept = static_cast<unsigned>(a.nswept) * a.nbands;
  if (ticket >= swept) {                                // Voronoi alpha epilogue of one band
    const int band = static_cast<int>(ticket - swept), c = ch - 1;
    for (int r = 0; r < kBand; ++r) {
      const int Y = band * kBand + r;
      if (Y >= h) break;
      for (int X = lane; X < w; X += kBand) {
        const double v = kQuantumRange * ((1.0 / 65535.0) * static_cast<double>(a.alpha_src[gidx(Y, X, c)]));
        a.out[gidx(Y, X, c)] = clamp_pixel(static_cast<float>(v));
      }
    }
    return;
  }
  const int c = static_cast<int>(ticket % a.nswept), band = static_cast<int>(ticket / a.nswept);
  const int Y0 = band * kBand, Y = Y0 + lane;
  const int A = a.A, Rr = a.Rr, s = a.s;
  const bool clamp_out = a.epilogue != 0;               // Voronoi reverse: ClampPixel on the stored colour channels
  for (int i = lane; i < a.nterms; i += kBand) s_terms[i] = a.terms[i];
  const int *pred = band > 0 && A > 0 ? a.progress + (ticket - a.nswept) : nullptr;
  int *mine = a.progress + ticket;
  const int last_row = min(kBand, h - Y0) - 1;          // the band's last valid row
  const int blocks = (w + last_row * s + kBand - 1) / kBand;
  int halo_loaded = 0;                                  // halo columns [0, halo_loaded) are in the ring
  __syncwarp();

  for (int k = 0; k < blocks; ++k) {
    // 1. halo: the last A rows of the band above, as far as lane 0 reads in this block
    if (pred) {
      const int need = min(w, kBand * k + kBand + Rr);
      while (halo_loaded < need) {
        const int upto = min(need, halo_loaded + kBand);
        if (lane == 0)
          while (ld_acquire(pred) < upto) __nanosleep(64);
        __syncwarp();
        const int X = halo_loaded + lane;
        if (X < upto)
          for (int j = 1; j <= A; ++j) out_ring[(A - j) * a.ring_out + (X & mask)] = __ldcg(a.out + gidx(Y0 - j, X, c));
        halo_loaded = upto;
      }
    }
    // 2. input rows: row r gets its columns up to 32k + 31 - r*s + Rr (each row a coalesced load)
    for (int r = 0; r <= last_row; ++r) {
      const int to = min(w, kBand * k + kBand - r * s + Rr);
      const int from = k == 0 ? 0 : max(0, to - kBand);
      for (int X = from + lane; X < to; X += kBand) in_ring[r * a.ring_in + (X & mask_in)] = __ldg(a.in + gidx(Y0 + r, X, c));
    }
    __syncwarp();
    // 3. 32 wavefront steps
    for (int t = kBand * k; t < kBand * k + kBand; ++t) {
      const int X = t - lane * s;
      if (lane <= last_row && X >= 0 && X < w) {
        double pixel = kQuantumRange;
        float *own = out_ring + (A + lane) * a.ring_out;
#pragma unroll 4
        for (int i = 0; i < a.nterms; ++i) {
          const Term tm = s_terms[i];
          int col = X + tm.d;
          float sample;
          if (tm.live) {
            if (col < 0) continue;
            sample = own[col & mask];
          } else {
            col = min(max(col, 0), w - 1);
            const int yy = max(Y + tm.dv, 0);
            sample = yy == Y ? in_ring[lane * a.ring_in + (col & mask_in)] : out_ring[(A + yy - Y0) * a.ring_out + (col & mask)];
          }
          const double v = static_cast<double>(sample) + tm.k;
          if (v < pixel) pixel = v;
        }
        own[X & mask] = __double2float_rn(pixel);
      }
      __syncwarp();
    }
    // 4. store the 32 columns each row finished in this block, then publish the last row's progress
    for (int r = 0; r <= last_row; ++r) {
      const int X = max(0, kBand * k - r * s) + lane, to = min(w, kBand * k + kBand - r * s);
      if (X < to) {
        const float v = out_ring[(A + r) * a.ring_out + (X & mask)];
        a.out[gidx(Y0 + r, X, c)] = clamp_out ? clamp_pixel(v) : v;
      }
    }
    __threadfence();
    __syncwarp();
    if (lane == 0) st_release(mine, max(0, min(w, kBand * k + kBand - last_row * s)));
  }
  if (lane == 0) st_release(mine, w);
}

// Power of two >= n
int pow2_at_least(int n) {
  int p = 1;
  while (p < n) p <<= 1;
  return p;
}

}  // namespace

// The term list of one pass in the reference's order (logical coordinates), and its geometry.
struct DirectPass {
  std::vector<Term> terms;
  int A, Rr, s, ring_out, ring_in;
  size_t smem;
};

static DirectPass plan_pass(const mb200_kernel_info *k, bool voronoi, bool reverse) {
  const long kw = static_cast<long>(k->width), kh = static_cast<long>(k->height), kx = k->x, ky = k->y;
  const long ox = kw - kx - 1, oy = kh - ky - 1;
  DirectPass p;
  auto add = [&](long idx, long dv, long d, int live) {
    const double v = k->values[idx];
    if (!std::isnan(v)) p.terms.push_back(Term{v, static_cast<short>(dv), static_cast<short>(d), live});
  };
  if (!reverse) {                                                   // :3368-3397, Voronoi :3399-3428
    const long rows = voronoi ? oy : oy + 1;
    for (long v = 0; v < rows; ++v)
      for (long u = 0; u < kw; ++u) add(kw * kh - 1 - (v * kw + u), v - oy, u - ox, 0);
    for (long u = 0; u < ox; ++u) add(kw * (ky + 1) - 1 - u, 0, u - ox, 1);
    p.A = static_cast<int>(oy); p.Rr = static_cast<int>(kx);
  } else {                                                          // :3532-3561, Voronoi :3563-3592 (mirrored)
    for (long r = 0; r <= ky; ++r)
      for (long u = 0; u < kw; ++u) add(kw * (ky + 1) - 1 - (r * kw + u), -r, ox - u, 0);
    for (long j = 1; j <= kx; ++j) add(voronoi ? kw * (ky + 1) - j : kw * ky + kx - j, 0, -j, 1);
    p.A = static_cast<int>(ky); p.Rr = static_cast<int>(ox);
  }
  p.s = p.A > 0 ? p.Rr + 1 : 0;
  // Ring spans: the rows above are read from L columns left of a lane's column to the newest column written or loaded
  // (at most A*s + kw + 31 columns); an input row from L left to Rr right plus the 32 columns loaded ahead (kw + 31).
  const long span_out = static_cast<long>(p.A) * p.s + kw + kBand, span_in = kw + kBand;
  p.ring_out = span_out > (1 << 20) ? (1 << 21) : pow2_at_least(static_cast<int>(span_out));
  p.ring_in = span_in > (1 << 20) ? (1 << 21) : pow2_at_least(static_cast<int>(span_in));
  p.smem = p.terms.size() * sizeof(Term) +
           (static_cast<size_t>(p.A + kBand) * p.ring_out + static_cast<size_t>(kBand) * p.ring_in) * sizeof(float);
  return p;
}

int morphology_direct_check(int channels, int method, const mb200_kernel_info *kernel) {
  if (method != MB200_DistanceMorphology && method != MB200_VoronoiMorphology)
    return fail(MB200_EINVAL, "morphology direct: method %d is neither Distance nor Voronoi", method);
  if (!kernel || !kernel->values || kernel->width == 0 || kernel->height == 0 || kernel->x < 0 || kernel->y < 0 ||
      static_cast<size_t>(kernel->x) >= kernel->width || static_cast<size_t>(kernel->y) >= kernel->height)
    return fail(MB200_EINVAL, "morphology direct: no kernel, or its origin lies outside it");
  if (method == MB200_VoronoiMorphology && !has_alpha(channels))
    return fail(MB200_EUNSUPPORTED, "morphology direct: Voronoi adds an alpha channel to an image without one");
  static const size_t kMaxSmem = 227 * 1024 - 1024;
  for (int rev = 0; rev < 2; ++rev) {
    const DirectPass p = plan_pass(kernel, method == MB200_VoronoiMorphology, rev != 0);
    if (p.A > kBand || p.smem > kMaxSmem || p.terms.size() > static_cast<size_t>(kMaxTerms))
      return fail(MB200_EUNSUPPORTED,
                  "morphology direct: a %zux%zu kernel does not fit the wavefront (cells, rows or shared memory)",
                  kernel->width, kernel->height);
  }
  return MB200_OK;
}

int launch_morphology_direct(const float *src, float *tmp, float *dst, size_t width, size_t height, int channels,
                             int method, const mb200_kernel_info *kernel, void *stream) {
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const bool voronoi = method == MB200_VoronoiMorphology;
  const int nbands = static_cast<int>((height + kBand - 1) / kBand);
  const int nswept = voronoi ? channels - 1 : channels;
  const DirectPass passes[2] = {plan_pass(kernel, voronoi, false), plan_pass(kernel, voronoi, true)};
  // one device block, zeroed on the stream before the launches: [tickets 2][progress 2 * nswept * nbands]
  const size_t nprog = static_cast<size_t>(nswept) * nbands;
  const size_t sync_bytes = (2 + 2 * nprog) * sizeof(int);
  StreamAlloc block(s);
  int rc = block.alloc(sync_bytes, "morphology direct: allocation");
  if (rc) return rc;
  unsigned char *base = block.as<unsigned char>();
  cudaError_t e = cudaMemsetAsync(base, 0, sync_bytes, s);
  if (e != cudaSuccess) rc = cuda_fail(e, "morphology direct: memset");
  static DirectArgs args[2];                            // 16 KB each: kept off the stack
  static std::mutex args_lock;
  std::lock_guard<std::mutex> lock(args_lock);          // the launch copies the parameters; the lock covers the staging
  for (int rev = 0; rev < 2 && rc == MB200_OK; ++rev) {
    const DirectPass &p = passes[rev];
    DirectArgs &a = args[rev];
    a = DirectArgs{};
    a.in = rev ? tmp : src;
    a.out = rev ? dst : tmp;
    a.alpha_src = src;
    std::copy(p.terms.begin(), p.terms.end(), a.terms);
    a.nterms = static_cast<int>(p.terms.size());
    a.w = static_cast<int>(width); a.h = static_cast<int>(height); a.ch = channels;
    a.A = p.A; a.Rr = p.Rr; a.s = p.s; a.ring_out = p.ring_out; a.ring_in = p.ring_in;
    a.nbands = nbands; a.nswept = nswept;
    a.epilogue = rev && voronoi;
    a.ticket = reinterpret_cast<unsigned *>(base) + rev;
    a.progress = reinterpret_cast<int *>(base) + 2 + rev * nprog;
    const void *fn = rev ? reinterpret_cast<const void *>(direct_sweep_kernel<true>)
                         : reinterpret_cast<const void *>(direct_sweep_kernel<false>);
    e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(p.smem));
    if (e != cudaSuccess) { rc = cuda_fail(e, "morphology direct: shared memory"); break; }
    const unsigned grid = static_cast<unsigned>(nprog + (a.epilogue ? nbands : 0));
    if (rev) direct_sweep_kernel<true><<<grid, kBand, p.smem, s>>>(a);
    else direct_sweep_kernel<false><<<grid, kBand, p.smem, s>>>(a);
    if ((rc = launch_status("morphology direct: launch", 0))) break;
    count_launch();                                     // counted once the launch is known to have been accepted
    count_family(kMorphDirect);
  }
  return rc;
}

}  // namespace mb200
