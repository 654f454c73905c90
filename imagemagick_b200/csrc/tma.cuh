// tma.cuh -- the Hopper tensor-memory-accelerator pieces shared by the staging rings of resize_stream.cu and
// conv_mma.cu: mbarrier transaction counts, one 2-D cp.async.bulk.tensor load, and the tensor map of an RGBA float
// image seen as a 2-D array of floats (4 * width x height).
#pragma once

#include <cuda.h>                 // CUtensorMap (types only: the encoder is fetched through cudaGetDriverEntryPoint)
#include <cudaTypedefs.h>
#include <cuda_runtime.h>

namespace mb200 {

__device__ __forceinline__ void mbar_init(unsigned bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(unsigned bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned bar, unsigned parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "MB200_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra MB200_DONE;\n"
      "bra MB200_WAIT;\n"
      "MB200_DONE:\n"
      "}\n" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_2d(unsigned dst, const CUtensorMap *map, int c0, int c1, unsigned bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
               ::"r"(dst), "l"(map), "r"(c0), "r"(c1), "r"(bar) : "memory");
}

// Tensor map of an RGBA float image as a 2-D array of floats (4 * width x height rows), box = box_floats x box_rows, with the given
// swizzle and L2 promotion.
// Boxes that reach past the image are zero-filled.  The encoder is a driver entry point; the library links the runtime
// only, so it is fetched by name.
inline bool make_rgba_tensor_map(const float *src, int width, int height, unsigned box_floats, unsigned box_rows,
                                 CUtensorMapSwizzle swizzle, CUtensorMapL2promotion promotion, CUtensorMap *map) {
  static PFN_cuTensorMapEncodeTiled encode = [] {
    void *fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      fn = nullptr;
    return reinterpret_cast<PFN_cuTensorMapEncodeTiled>(fn);
  }();
  if (encode == nullptr) return false;
  const cuuint64_t dims[2] = {static_cast<cuuint64_t>(width) * 4, static_cast<cuuint64_t>(height)};
  const cuuint64_t strides[1] = {static_cast<cuuint64_t>(width) * 16};
  const cuuint32_t box[2] = {box_floats, box_rows}, estr[2] = {1, 1};
  return encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float *>(src), dims, strides, box, estr,
                CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, promotion,
                CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace mb200
