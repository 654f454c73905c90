// launch.cuh -- the host side shared by the .cu launchers: channel dispatch, the check after a launch, the 1-D grid size
// and stream-ordered temporaries from the library's pool.
#pragma once

#include "mb200_internal.h"

#include <cuda_runtime.h>

#include <cstdint>
#include <type_traits>

namespace mb200 {

// f(std::integral_constant<int, C>{}) for C = channels in 1..4, so that a site reads kernel<ch()><<<...>>>; any other
// channel count is declined.  Returns what f returns.
template <typename F>
int with_channels(int channels, const char *what, F &&f) {
  switch (channels) {
    case 1: return f(std::integral_constant<int, 1>{});
    case 2: return f(std::integral_constant<int, 2>{});
    case 3: return f(std::integral_constant<int, 3>{});
    case 4: return f(std::integral_constant<int, 4>{});
    default: return fail(MB200_EINVAL, "%s: 1..4 channels", what);
  }
}

// The same with the float4 form of RGBA: f(ch, vec) with vec = std::bool_constant, true only for 4 channels when `vec4`
// (the caller's 16-byte alignment test), so only <1..4, false> and <4, true> are instantiated.
template <typename F>
int with_channels(int channels, bool vec4, const char *what, F &&f) {
  if (channels == 4 && vec4) return f(std::integral_constant<int, 4>{}, std::true_type{});
  return with_channels(channels, what, [&](auto ch) { return f(ch, std::false_type{}); });
}

// Counts `launches` kernel launches (0 where the site counts them itself), then reports a failed launch.
inline int launch_status(const char *what, unsigned launches = 1) {
  count_launch(launches);
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? MB200_OK : cuda_fail(e, what);
}

// Blocks of `block` threads covering n items, declined when n is 0 or the grid exceeds the 1-D limit.
inline int grid_of(size_t n, unsigned block, unsigned *grid, const char *what) {
  const size_t blocks = (n + block - 1) / block;
  if (blocks == 0 || blocks > 0x7fffffffull) return fail(MB200_EINVAL, "%s: bad image size", what);
  *grid = static_cast<unsigned>(blocks);
  return MB200_OK;
}

// Both pointers on a 16-byte boundary (float4 access to RGBA pixels).
inline bool aligned16(const void *p, const void *q = nullptr) {
  return ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(q)) & 15) == 0;
}

// A stream-ordered temporary from the library's pool (temp_pool()), freed stream-ordered when it goes out of scope, so
// work queued on the stream before the free may still read it.
struct StreamAlloc {
  void *ptr = nullptr;
  cudaStream_t s;
  explicit StreamAlloc(cudaStream_t stream) : s(stream) {}
  ~StreamAlloc() { if (ptr) cudaFreeAsync(ptr, s); }
  StreamAlloc(const StreamAlloc &) = delete;
  StreamAlloc &operator=(const StreamAlloc &) = delete;

  int alloc(size_t bytes, const char *what = "temporary allocation") {
    const cudaError_t e = cudaMallocAsync(&ptr, bytes ? bytes : 1, temp_pool(), s);
    if (e != cudaSuccess) { ptr = nullptr; return cuda_fail(e, what); }
    return MB200_OK;
  }
  // alloc, then an asynchronous copy of a host table: from pageable memory the runtime has staged the table when the
  // call returns, so `host` may go away right after.
  int upload(const void *host, size_t bytes, const char *what) {
    int rc = alloc(bytes, what);
    if (rc) return rc;
    const cudaError_t e = cudaMemcpyAsync(ptr, host, bytes, cudaMemcpyHostToDevice, s);
    return e == cudaSuccess ? MB200_OK : cuda_fail(e, what);
  }
  template <typename T> T *as() const { return static_cast<T *>(ptr); }
};

}  // namespace mb200
