// equalize.cuh -- the histogram and table-apply kernels of EqualizeImage and of the histogram-driven level operators
// (level.cu: ContrastStretchImage, LinearStretchImage, GammaImage), which run the same two passes with a table built on
// the host in between; AutoThresholdImage takes the histogram pass alone.
#pragma once

#include <cuda_runtime.h>

namespace mb200 {
namespace {

constexpr unsigned kBins = 65536;

// quantum-private.h:504-514 (HDRI)
__device__ __forceinline__ unsigned scale_quantum_to_map(float q) {
  if (q >= 65535.0f) return 65535u;
  if (!(q > 0.0f)) return 0u;                       // NaN or <= 0
  return static_cast<unsigned>(q + 0.5f);
}

// quantum.h:113-124 ScaleQuantumToChar (Q16, HDRI): float division and addition, as the reference evaluates them
__device__ __forceinline__ unsigned scale_quantum_to_char(float q) {
  if (!(q > 0.0f)) return 0u;                       // NaN or <= 0
  const float d = __fdiv_rn(q, 257.0f);
  if (d >= 255.0f) return 255u;
  return static_cast<unsigned>(__fadd_rn(d, 0.5f));
}

// One histogram per channel (sync == 0) or one shared, intensity-driven histogram (sync != 0): counts[c][bin].
// CHAR_BINS: the intensity histogram of AutoThresholdImage (threshold.c:731), 256 bins of ScaleQuantumToChar.
// Lanes of a warp that hit the same bin are merged before the atomic (images have long runs of equal values).
template <int CH, bool CHAR_BINS = false>
__global__ void __launch_bounds__(256) histogram_kernel(const float *__restrict__ buf, size_t npixels, int sync,
                                                        unsigned *__restrict__ counts) {
  const size_t i = static_cast<size_t>(blockIdx.x) * 256 + threadIdx.x;
  const bool live = i < npixels;
  float v[CH];
#pragma unroll
  for (int c = 0; c < CH; ++c) v[c] = live ? __ldg(buf + i * CH + c) : 0.0f;
  auto add = [&](unsigned *hist, unsigned bin) {
    const unsigned active = __ballot_sync(0xffffffffu, live);
    if (!live) return;
    const unsigned peers = __match_any_sync(active, bin);
    if ((threadIdx.x & 31) == static_cast<unsigned>(__ffs(peers) - 1)) atomicAdd(hist + bin, static_cast<unsigned>(__popc(peers)));
  };
  if (sync) {
    const double red = static_cast<double>(v[0]);
    double pixel = red;                                                  // pixel.c:2356 GetPixelIntensity, Rec709Luma
    if (CH > 1)          // Gray+Alpha: the green / blue accessors resolve to the gray sample (same expression on g,g,g)
      pixel = __dadd_rn(__dadd_rn(__dmul_rn(0.212656, red), __dmul_rn(0.715158, static_cast<double>(v[CH >= 3 ? 1 : 0]))),
                        __dmul_rn(0.072186, static_cast<double>(v[CH >= 3 ? 2 : 0])));
    const float quantum = static_cast<float>(pixel);                     // ClampToQuantum (HDRI) == the float cast
    add(counts, CHAR_BINS ? scale_quantum_to_char(quantum) : scale_quantum_to_map(quantum));
  } else {
#pragma unroll
    for (int c = 0; c < CH; ++c) add(counts + static_cast<size_t>(c) * kBins, scale_quantum_to_map(v[c]));
  }
}

// table[c][bin] (float Quantum); enabled bit c: the channel is rewritten (Equalize: black[c] != white[c])
template <int CH>
__global__ void __launch_bounds__(256) equalize_apply_kernel(float *__restrict__ buf, size_t npixels,
                                                             const float *__restrict__ table, unsigned enabled) {
  const size_t i = static_cast<size_t>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= npixels) return;
#pragma unroll
  for (int c = 0; c < CH; ++c) {
    if (!(enabled >> c & 1u)) continue;
    const float q = buf[i * CH + c];
    buf[i * CH + c] = __ldg(table + static_cast<size_t>(c) * kBins + scale_quantum_to_map(q));
  }
}

}  // namespace
}  // namespace mb200
