// geometry.cu -- the orientation and crop operators of MagickCore/transform.c and shear.c (CropImage, ShaveImage,
// FlipImage, FlopImage, TransposeImage, TransverseImage, IntegralRotateImage, RollImage): out(x, y) = in(map(x, y)) for
// a plan of geometry_plan.cpp.
//
// Pure data movement, so samples travel as 32-bit words: NaN payloads, -0 and denormals keep their bits.  Two kernels:
//   - maps that keep the axes (crop, flip, flop, 180 degrees, roll): one CTA row loop per output row, consecutive
//     threads on consecutive output pixels, so the reads run forwards or backwards along one source row.  A pixel of
//     1, 2 or 4 channels is one 4-, 8- or 16-byte access when both buffers are aligned to it; 3 and 5 channels (and
//     unaligned buffers) copy word by word.
//   - maps that swap the axes (transpose, transverse, 90 and 270 degrees): 32 x 32 pixel tiles staged in shared memory,
//     read along source rows and written along output rows, so both sides coalesce.  A tile row is 33 * CH words: the
//     pad makes the column-wise read of the store phase conflict-free for every channel count.
// Offsets are 64-bit and every loop is grid-stride, so no dimension is limited.
#include "mb200_internal.h"

#include <cuda_runtime.h>

namespace mb200 {
namespace {

constexpr int kTile = 32;
constexpr int kRowThreads = 256;
constexpr int kTileThreads = 256;        // 8 warps per 32 x 32 tile

struct Map {
  const unsigned *src;
  unsigned *dst;
  long long sw;                          // source row length in pixels
  long long ow, oh;                      // output
  long long rw, rh;                      // the source rectangle (ow x oh, swapped for transposing maps)
  long long sx, sy;                      // its origin
  long long roll_x, roll_y;
  int flop, flip;
};

// source column / row of the rectangle for output coordinate c along an axis that is not swapped
__device__ __forceinline__ long long axis_src(long long c, long long roll, long long n, int mirror) {
  long long u = c - roll;
  if (u < 0) u += n;
  return mirror ? n - 1 - u : u;
}

// Maps that keep the axes, one pixel of type P (CH words) per access.
template <typename P>
__global__ void __launch_bounds__(kRowThreads) geometry_rows_pixels(const __grid_constant__ Map m) {
  const P *src = reinterpret_cast<const P *>(m.src);
  P *dst = reinterpret_cast<P *>(m.dst);
  for (long long y = blockIdx.y; y < m.oh; y += gridDim.y) {
    const long long v = axis_src(y, m.roll_y, m.rh, m.flip);
    const P *row = src + (m.sy + v) * m.sw + m.sx;
    P *out = dst + y * m.ow;
    for (long long x = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; x < m.ow;
         x += static_cast<long long>(gridDim.x) * blockDim.x)
      out[x] = __ldg(row + axis_src(x, m.roll_x, m.rw, m.flop));
  }
}

// The same, word by word: consecutive threads take consecutive words of the output row.
template <int CH>
__global__ void __launch_bounds__(kRowThreads) geometry_rows_words(const __grid_constant__ Map m) {
  const long long n = m.ow * CH;
  for (long long y = blockIdx.y; y < m.oh; y += gridDim.y) {
    const long long v = axis_src(y, m.roll_y, m.rh, m.flip);
    const unsigned *row = m.src + ((m.sy + v) * m.sw + m.sx) * CH;
    unsigned *out = m.dst + y * n;
    for (long long w = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; w < n;
         w += static_cast<long long>(gridDim.x) * blockDim.x) {
      const long long x = w / CH;
      const int k = static_cast<int>(w - x * CH);
      out[w] = __ldg(row + axis_src(x, m.roll_x, m.rw, m.flop) * CH + k);
    }
  }
}

// Maps that swap the axes: output (x, y) reads the rectangle's column y and row x (each mirrored by its bit).
template <int CH>
__global__ void __launch_bounds__(kTileThreads) geometry_tiles(const __grid_constant__ Map m) {
  constexpr int kStride = (kTile + 1) * CH;
  __shared__ unsigned tile[kTile * kStride];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long tiles_x = (m.ow + kTile - 1) / kTile, tiles_y = (m.oh + kTile - 1) / kTile;
  for (long long t = blockIdx.x; t < tiles_x * tiles_y; t += gridDim.x) {
    const long long ox0 = (t % tiles_x) * kTile, oy0 = (t / tiles_x) * kTile;
    const int nx = static_cast<int>(min(static_cast<long long>(kTile), m.ow - ox0));
    const int ny = static_cast<int>(min(static_cast<long long>(kTile), m.oh - oy0));
    // the tile's source columns (output rows oy0 .. oy0 + ny - 1), in memory order from umin
    const long long umin = m.flop ? m.rw - oy0 - ny : oy0;
    const unsigned *base = m.src + (m.sy * m.sw + m.sx + umin) * CH;
    // load: tile row i holds the source row of output column ox0 + i, words of the ny pixels in memory order
    for (int i = warp; i < nx; i += kTileThreads / 32) {
      const long long v = m.flip ? m.rh - 1 - (ox0 + i) : ox0 + i;
      const unsigned *row = base + v * m.sw * CH;
      for (int w = lane; w < ny * CH; w += 32) tile[i * kStride + w] = __ldg(row + w);
    }
    __syncthreads();
    // store: output row oy0 + j, words of the nx pixels from tile column m_j
    for (int j = warp; j < ny; j += kTileThreads / 32) {
      const int mj = m.flop ? ny - 1 - j : j;
      unsigned *out = m.dst + ((oy0 + j) * m.ow + ox0) * CH;
      for (int w = lane; w < nx * CH; w += 32) {
        const int i = w / CH, k = w - i * CH;
        out[w] = tile[i * kStride + mj * CH + k];
      }
    }
    __syncthreads();
  }
}

template <typename P>
bool aligned(const void *a, const void *b) {
  return reinterpret_cast<uintptr_t>(a) % sizeof(P) == 0 && reinterpret_cast<uintptr_t>(b) % sizeof(P) == 0;
}

template <int CH>
cudaError_t launch_words(const Map &m, cudaStream_t s) {
  const long long n = m.ow * CH;
  const dim3 grid(static_cast<unsigned>(min((n + kRowThreads - 1) / kRowThreads, 1024LL)),
                  static_cast<unsigned>(min(m.oh, 65535LL)));
  geometry_rows_words<CH><<<grid, kRowThreads, 0, s>>>(m);
  return cudaGetLastError();
}

template <typename P>
cudaError_t launch_pixels(const Map &m, cudaStream_t s) {
  const dim3 grid(static_cast<unsigned>(min((m.ow + kRowThreads - 1) / kRowThreads, 1024LL)),
                  static_cast<unsigned>(min(m.oh, 65535LL)));
  geometry_rows_pixels<P><<<grid, kRowThreads, 0, s>>>(m);
  return cudaGetLastError();
}

template <int CH>
cudaError_t launch_tiles(const Map &m, cudaStream_t s) {
  const long long tiles = ((m.ow + kTile - 1) / kTile) * ((m.oh + kTile - 1) / kTile);
  const unsigned grid = static_cast<unsigned>(min(tiles, static_cast<long long>(sm_count()) * 16));
  geometry_tiles<CH><<<grid, kTileThreads, 0, s>>>(m);
  return cudaGetLastError();
}

}  // namespace

int geometry_check(size_t width, size_t height, int channels, const mb200_geometry_params *plan) {
  if (!plan || width == 0 || height == 0 || channels < 1 || channels > 5 || plan->map < 0 || plan->map > 7 ||
      plan->columns == 0 || plan->rows == 0)
    return fail(MB200_EINVAL, "geometry: bad arguments");
  const bool swap = (plan->map & 4) != 0;
  const size_t rw = swap ? plan->rows : plan->columns, rh = swap ? plan->columns : plan->rows;
  if (plan->src_x < 0 || plan->src_y < 0 || rw > width || rh > height ||
      static_cast<size_t>(plan->src_x) > width - rw || static_cast<size_t>(plan->src_y) > height - rh ||
      plan->roll_x < 0 || plan->roll_y < 0 || static_cast<size_t>(plan->roll_x) >= rw ||
      static_cast<size_t>(plan->roll_y) >= rh || (swap && (plan->roll_x || plan->roll_y)))
    return fail(MB200_EINVAL, "geometry: the plan's source rectangle does not fit the image");
  return MB200_OK;
}

int launch_geometry(const float *src, size_t width, size_t height, int channels, float *dst,
                    const mb200_geometry_params *plan, void *stream) {
  (void) height;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  Map m;
  m.src = reinterpret_cast<const unsigned *>(src);
  m.dst = reinterpret_cast<unsigned *>(dst);
  m.sw = static_cast<long long>(width);
  m.ow = static_cast<long long>(plan->columns);
  m.oh = static_cast<long long>(plan->rows);
  const bool swap = (plan->map & 4) != 0;
  m.rw = swap ? m.oh : m.ow;
  m.rh = swap ? m.ow : m.oh;
  m.sx = plan->src_x;
  m.sy = plan->src_y;
  m.roll_x = plan->roll_x;
  m.roll_y = plan->roll_y;
  m.flop = plan->map & 1;
  m.flip = (plan->map >> 1) & 1;
  cudaError_t e;
  if (swap) {
    switch (channels) {
      case 1: e = launch_tiles<1>(m, s); break;
      case 2: e = launch_tiles<2>(m, s); break;
      case 3: e = launch_tiles<3>(m, s); break;
      case 4: e = launch_tiles<4>(m, s); break;
      default: e = launch_tiles<5>(m, s); break;
    }
  } else {
    switch (channels) {
      case 1: e = launch_pixels<unsigned>(m, s); break;
      case 2: e = aligned<uint2>(src, dst) ? launch_pixels<uint2>(m, s) : launch_words<2>(m, s); break;
      case 3: e = launch_words<3>(m, s); break;
      case 4: e = aligned<uint4>(src, dst) ? launch_pixels<uint4>(m, s) : launch_words<4>(m, s); break;
      default: e = launch_words<5>(m, s); break;
    }
  }
  if (e != cudaSuccess) return cuda_fail(e, "geometry launch");
  count_family(kGeometry);
  count_launch();
  return MB200_OK;
}

}  // namespace mb200
