// equalize.cu -- EqualizeImage (MagickCore/enhance.c:2040-2290), the second half of EmbossImage (effect.c:1600-1681:
// ConvolveImage with an anti-diagonal kernel, then EqualizeImage on the result).
//
// Reference algorithm (Q16-HDRI, MaxMap = 65535):
//   1. histogram[bin][i]++ for every channel i of every pixel, bin = ScaleQuantumToMap(ClampToQuantum(intensity)) where
//      intensity is the pixel's GetPixelIntensity (Rec709 luma; the gray sample of gray images) when the channel mask
//      carries SyncChannels -- which the default mask (AllChannels) does -- and the channel's own value otherwise (:2125-2129);
//   2. map = running sum of the histogram; black = map[0], white = map[MaxMap];
//      equalize_map[j] = ScaleMapToQuantum(MaxMap * (map[j] - black) / (white - black))              (:2138-2169)
//   3. every Update channel with black != white: q = equalize_map[ScaleQuantumToMap(q)]                (:2229-2260)
// Step 1 and 3 run on the device (integer counts: exact; table lookup: exact), step 2 -- 65 536 doubles per channel in
// the reference's own order -- on the host between them, so the result is bit-identical to the reference's.
#include "mb200_internal.h"
#include "equalize.cuh"

#include <cuda_runtime.h>

#include <vector>

namespace mb200 {

int launch_equalize(float *buf, size_t npixels, int channels, int sync_channels, void *stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (channels < 1 || channels > 4) return fail(MB200_EINVAL, "equalize: 1..4 channels");
  const size_t blocks = (npixels + 255) / 256;
  if (blocks == 0 || blocks > 0x7fffffffull) return fail(MB200_EINVAL, "equalize: bad image size");
  const unsigned grid = static_cast<unsigned>(blocks);
  const int nhist = sync_channels ? 1 : channels;
  unsigned *d_counts = nullptr;
  float *d_table = nullptr;
  cudaError_t e = cudaMallocAsync(reinterpret_cast<void **>(&d_counts), sizeof(unsigned) * kBins * nhist, temp_pool(), s);
  if (e == cudaSuccess) e = cudaMallocAsync(reinterpret_cast<void **>(&d_table), sizeof(float) * kBins * channels, temp_pool(), s);
  if (e != cudaSuccess) { if (d_counts) cudaFreeAsync(d_counts, s); return cuda_fail(e, "equalize: allocation"); }
  cudaMemsetAsync(d_counts, 0, sizeof(unsigned) * kBins * nhist, s);
  switch (channels) {
    case 1: histogram_kernel<1><<<grid, 256, 0, s>>>(buf, npixels, sync_channels, d_counts); break;
    case 2: histogram_kernel<2><<<grid, 256, 0, s>>>(buf, npixels, sync_channels, d_counts); break;
    case 3: histogram_kernel<3><<<grid, 256, 0, s>>>(buf, npixels, sync_channels, d_counts); break;
    default: histogram_kernel<4><<<grid, 256, 0, s>>>(buf, npixels, sync_channels, d_counts); break;
  }
  count_launch();
  std::vector<unsigned> counts(static_cast<size_t>(kBins) * nhist);
  e = cudaMemcpyAsync(counts.data(), d_counts, counts.size() * sizeof(unsigned), cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) { cudaFreeAsync(d_counts, s); cudaFreeAsync(d_table, s); return cuda_fail(e, "equalize: histogram readback"); }
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
    for (unsigned j = 0; j < kBins; ++j) {
      const double value = (65535.0 * (map[j] - black)) / (white - black);
      // ScaleMapToQuantum (quantum-private.h:464-475, HDRI)
      table[static_cast<size_t>(c) * kBins + j] = value <= 0.0 ? 0.0f : value >= 65535.0 ? 65535.0f : static_cast<float>(value);
    }
  }
  int rc = MB200_OK;
  if (enabled) {
    e = cudaMemcpyAsync(d_table, table.data(), table.size() * sizeof(float), cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) {
      switch (channels) {
        case 1: equalize_apply_kernel<1><<<grid, 256, 0, s>>>(buf, npixels, d_table, enabled); break;
        case 2: equalize_apply_kernel<2><<<grid, 256, 0, s>>>(buf, npixels, d_table, enabled); break;
        case 3: equalize_apply_kernel<3><<<grid, 256, 0, s>>>(buf, npixels, d_table, enabled); break;
        default: equalize_apply_kernel<4><<<grid, 256, 0, s>>>(buf, npixels, d_table, enabled); break;
      }
      count_launch();
      e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);         // `table` (pageable) must outlive the copy
    if (e != cudaSuccess) rc = cuda_fail(e, "equalize: apply");
  }
  cudaFreeAsync(d_counts, s);
  cudaFreeAsync(d_table, s);
  return rc;
}

}  // namespace mb200
