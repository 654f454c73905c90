// runtime.cu -- device selection, error reporting, staging buffers.
//
// The CUDA analogue of the reference's OpenCL environment plumbing
// (MagickCore/opencl.c: GetCurrentOpenCLEnv, RequestOpenCLDevice :2578, AcquireMagickCLCacheInfo
// :528) reduced to what the hot path needs: one stream and a few grow-only scratch
// buffers per device, guarded by a mutex (cf. openCL_lock, opencl.c:538).
#include "mb200_internal.h"

#include <cuda_runtime.h>

#include <atomic>
#include <cctype>
#include <climits>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>

namespace mb200 {

namespace {
thread_local char t_error[512] = "";
std::atomic<unsigned long long> g_launches{0};

constexpr int kMaxDevices = 16;
constexpr int kScratchSlots = 8;

struct DeviceStateImpl {
  bool ready = false;
  cudaStream_t stream = nullptr;
  cudaMemPool_t pool = nullptr;      // private pool of the operators' temporaries
  int sms = 0;
  int l2_bytes = 0;
  void *scratch[kScratchSlots] = {nullptr};
  size_t scratch_bytes[kScratchSlots] = {0};
};
DeviceStateImpl g_dev[kMaxDevices];
std::mutex g_mutex;
}  // namespace

int fail(int code, const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(t_error, sizeof(t_error), fmt, ap);
  va_end(ap);
  return code;
}

int cuda_fail(int e, const char *what) {
  const cudaError_t err = static_cast<cudaError_t>(e);
  if (err == cudaErrorNoDevice || err == cudaErrorInsufficientDriver)
    return fail(MB200_ENODEVICE, "%s: %s", what, cudaGetErrorString(err));
  if (err == cudaErrorMemoryAllocation) return fail(MB200_ENOMEM, "%s: %s", what, cudaGetErrorString(err));
  return fail(MB200_ECUDA, "%s: %s", what, cudaGetErrorString(err));
}

void count_launch(unsigned n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

namespace {
// One row per option: the option name (the environment variable is MB200_ + its upper-case form unless the row names
// another), the default, the accepted values and how a value is read.  The upper bounds keep the strip arithmetic of
// the launchers inside int.
constexpr int kKnobMax = 1 << 20;
enum KnobKind {
  kInteger,     // a decimal int inside the accepted values
  kSwitch,      // on for any value other than 0; in the environment, for any non-empty value not starting with '0'
};
struct KnobSpec {
  const char *name;
  int TuningKnobs::*field;
  int fallback;
  bool (*valid)(int);
  KnobKind kind;
  const char *env;
};
bool any_value(int) { return true; }
const KnobSpec kKnobs[] = {
    {"mma_strip", &TuningKnobs::mma_strip, 512, [](int v) { return v >= 8 && v <= kKnobMax; }},   // rounded up to 8
    {"mma_minb", &TuningKnobs::mma_minb, 4, [](int v) { return v == 3 || v == 4; }},
    {"mma_l2pf", &TuningKnobs::mma_l2pf, -1, [](int v) { return v >= -1 && v <= 1; }},    // -1: windows of <= 9 taps
    // matrix path of the separable convolution: -1 automatic (float in / float out passes), 0 never, 1 whenever possible
    {"conv_mma", &TuningKnobs::conv_mma, -1, [](int v) { return v >= -1 && v <= 1; }, kInteger, "MB200_MMA"},
    // DMMA.16x8x16 tiles on the matrix path: -1 automatic (windows of 18-33 taps), 0 never, 1 every float-in pass
    {"mma_wide", &TuningKnobs::mma_wide, -1, [](int v) { return v >= -1 && v <= 1; }},
    {"pair", &TuningKnobs::pair, 1, [](int v) { return v == 0 || v == 1; }},
    {"pair_async", &TuningKnobs::pair_async, 1, [](int v) { return v == 0 || v == 1; }},
    {"pair_async_col", &TuningKnobs::pair_async_col, -1, [](int v) { return v >= -1 && v <= 1; }},   // -1: < 33 taps
    {"col_rot", &TuningKnobs::col_rot, 16, [](int v) { return v >= 1 && v <= kKnobMax; }},
    {"row_pair_rot", &TuningKnobs::row_pair_rot, 16, [](int v) { return v >= 1 && v <= kKnobMax; }},
    {"row_rot", &TuningKnobs::row_rot, 0, [](int v) { return v >= 0 && v <= kKnobMax; }},      // 0: >= 64 outputs
    {"resize_tma", &TuningKnobs::resize_tma, 1, [](int v) { return v >= 0 && v <= 2; }},
    {"resize_chunk", &TuningKnobs::resize_chunk, 16, [](int v) { return v == 8 || v == 16; }},
    {"resize_slots", &TuningKnobs::resize_slots, 0, [](int v) { return v == 0 || v == 2 || v == 3; }},
    {"resize_strip", &TuningKnobs::resize_strip, 0, [](int v) { return v >= 0 && v <= kKnobMax; }},  // 0: automatic
    // output rows per thread of the dense 2-D convolution: 0 automatic, 8 / 4 / 2 forced where that tile fits
    {"conv2d_rows", &TuningKnobs::conv2d_rows, 0, [](int v) { return v == 0 || v == 2 || v == 4 || v == 8; }},
    // switches that force the generic kernels, so that tests can compare them with the specialised ones
    {"no_rank1", &TuningKnobs::no_rank1, 0, any_value, kSwitch},
    {"no_morph_stream", &TuningKnobs::no_morph_stream, 0, any_value, kSwitch},
    {"no_resize_stream", &TuningKnobs::no_resize_stream, 0, any_value, kSwitch},
    {"no_fused_unsharp", &TuningKnobs::no_fused_unsharp, 0, any_value, kSwitch},
    {"no_resize_fused", &TuningKnobs::no_resize_fused, 0, any_value, kSwitch},
    {"no_adaptive_tile", &TuningKnobs::no_adaptive_tile, 0, any_value, kSwitch},
    // opt-in path that measured slower than the default
    {"resize_regular_h", &TuningKnobs::resize_regular_h, 0, any_value, kSwitch},
    // the fused ResizeImage wherever it applies, also below the automatic size threshold
    {"resize_fused", &TuningKnobs::resize_fused, 0, any_value, kSwitch},
};
constexpr size_t kNumKnobs = sizeof(kKnobs) / sizeof(kKnobs[0]);

int parse_env(const KnobSpec &k, const char *s) {
  if (!s || !*s) return k.fallback;
  if (k.kind == kSwitch) return *s != '0';
  char *end = nullptr;
  const long parsed = std::strtol(s, &end, 10);
  if (*end == '\0' && parsed >= INT_MIN && parsed <= INT_MAX && k.valid(static_cast<int>(parsed)))
    return static_cast<int>(parsed);
  return k.fallback;
}

struct KnobStore {
  std::atomic<int> value[kNumKnobs];
  KnobStore() {
    for (size_t i = 0; i < kNumKnobs; ++i) {
      char env[64] = "MB200_";
      for (size_t j = 0; kKnobs[i].name[j] && j + 7 < sizeof(env); ++j)
        env[6 + j] = static_cast<char>(std::toupper(static_cast<unsigned char>(kKnobs[i].name[j])));
      value[i].store(parse_env(kKnobs[i], std::getenv(kKnobs[i].env ? kKnobs[i].env : env)), std::memory_order_relaxed);
    }
  }
};
KnobStore &knob_store() {
  static KnobStore s;
  return s;
}
int knob_index(const char *name) {
  for (size_t i = 0; i < kNumKnobs; ++i)
    if (std::strcmp(kKnobs[i].name, name) == 0) return static_cast<int>(i);
  return -1;
}

const char *const kFamilyNames[kLaunchFamilies] = {
    "conv_mma_launches", "conv_mma_wide_launches", "conv_pair_launches", "conv_pair_async_launches", "conv_generic_launches",
    "resize_v_stream_launches", "resize_h_tma_launches", "resize_h_stream_launches", "resize_fused_launches",
    "resize_regular_launches", "resize_gather_launches", "conv2d_dense_r8_launches", "conv2d_dense_r4_launches",
    "conv2d_dense_r2_launches", "morph2d_launches", "minmax2d_launches", "morph_stream_launches", "morph_direct_launches",
    "distort_launches", "geometry_launches", "adaptive_threshold_tile_launches", "adaptive_threshold_direct_launches",
    "bounding_box_launches"};
std::atomic<unsigned long long> g_family_launches[kLaunchFamilies];
int family_index(const char *name) {
  for (int f = 0; f < kLaunchFamilies; ++f)
    if (std::strcmp(kFamilyNames[f], name) == 0) return f;
  return -1;
}
}  // namespace

TuningKnobs tuning_knobs() {
  TuningKnobs t;
  KnobStore &s = knob_store();
  for (size_t i = 0; i < kNumKnobs; ++i) t.*kKnobs[i].field = s.value[i].load(std::memory_order_relaxed);
  return t;
}

void count_family(LaunchFamily family) { g_family_launches[family].fetch_add(1, std::memory_order_relaxed); }

int ensure_device() {
  int dev = -1;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) { cudaGetLastError(); return cuda_fail(e, "cudaGetDevice"); }
  if (dev < 0 || dev >= kMaxDevices) return fail(MB200_ENODEVICE, "device index %d out of range", dev);
  std::lock_guard<std::mutex> lock(g_mutex);
  DeviceStateImpl &d = g_dev[dev];
  if (d.ready) return MB200_OK;
  cudaDeviceProp prop;
  e = cudaGetDeviceProperties(&prop, dev);
  if (e != cudaSuccess) return cuda_fail(e, "cudaGetDeviceProperties");
  if (prop.major != 9 || prop.minor != 0)
    return fail(MB200_ENODEVICE, "device %d is sm_%d%d; libmagickb200 carries sm_90a code only", dev,
                prop.major, prop.minor);
  d.sms = prop.multiProcessorCount;
  e = cudaDeviceGetAttribute(&d.l2_bytes, cudaDevAttrL2CacheSize, dev);
  if (e != cudaSuccess) return cuda_fail(e, "cudaDeviceGetAttribute(L2 size)");
  e = cudaStreamCreateWithFlags(&d.stream, cudaStreamNonBlocking);
  if (e != cudaSuccess) return cuda_fail(e, "cudaStreamCreate");
  {
    // Temporaries come from a pool of our own: freed blocks stay cached for the next call (an 8192^2 blur needs a
    // 1 GiB intermediate per call; re-creating it costs ~130 ms, reusing it 3 us -- tools/micro/staging.cu) without
    // touching the release threshold of the host application's default pool.  mb200_trim() returns the memory.
    cudaMemPoolProps props = {};
    props.allocType = cudaMemAllocationTypePinned;
    props.handleTypes = cudaMemHandleTypeNone;
    props.location.type = cudaMemLocationTypeDevice;
    props.location.id = dev;
    e = cudaMemPoolCreate(&d.pool, &props);
    if (e != cudaSuccess) return cuda_fail(e, "cudaMemPoolCreate");
    unsigned long long threshold = ~0ull;
    cudaMemPoolSetAttribute(d.pool, cudaMemPoolAttrReleaseThreshold, &threshold);
  }
  d.ready = true;
  return MB200_OK;
}

static DeviceStateImpl *current() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) return nullptr;
  return &g_dev[dev];
}

// The library stream of the CALLING THREAD on the current device: host-buffer calls made from different application
// threads (MagickWand users, `-concurrent`) run on different streams and overlap -- one thread's upload with another's
// kernels and download -- while the calls of one thread stay ordered.  (SURVEY 8b "Threading": re-entrant, per-call stream.)
void *default_stream() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) return nullptr;
  thread_local cudaStream_t streams[kMaxDevices] = {nullptr};
  if (!streams[dev] && cudaStreamCreateWithFlags(&streams[dev], cudaStreamNonBlocking) != cudaSuccess) {
    cudaGetLastError();
    return g_dev[dev].stream;            // the per-device stream created by ensure_device()
  }
  return streams[dev];
}

::CUmemPoolHandle_st *temp_pool() {
  DeviceStateImpl *d = current();
  return d ? d->pool : nullptr;
}

int sm_count() {
  DeviceStateImpl *d = current();
  return d && d->sms ? d->sms : 132;
}

size_t l2_bytes() {
  DeviceStateImpl *d = current();
  return d && d->l2_bytes > 0 ? static_cast<size_t>(d->l2_bytes) : size_t{50} << 20;
}

int scratch(void **ptr, size_t bytes, int slot) {
  DeviceStateImpl *d = current();
  if (!d || slot < 0 || slot >= kScratchSlots) return fail(MB200_EINVAL, "bad scratch slot");
  std::lock_guard<std::mutex> lock(g_mutex);
  if (d->scratch_bytes[slot] < bytes) {
    if (d->scratch[slot]) {
      cudaDeviceSynchronize();
      cudaFree(d->scratch[slot]);
      d->scratch[slot] = nullptr;
      d->scratch_bytes[slot] = 0;
    }
    cudaError_t e = cudaMalloc(&d->scratch[slot], bytes);
    if (e != cudaSuccess) return cuda_fail(e, "cudaMalloc(scratch)");
    d->scratch_bytes[slot] = bytes;
  }
  *ptr = d->scratch[slot];
  return MB200_OK;
}

// FP64 FMA issue-rate probe (the co-limit of the convolution kernels, SURVEY 8d): 16 independent DFMA chains per
// thread, 1024 threads per SM.
__global__ void __launch_bounds__(1024) fp64_probe_kernel(double *out, double a, double b, int iters) {
  double acc[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) acc[i] = threadIdx.x + i;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[i] = fma(acc[i], a, b);
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < 16; ++i) s += acc[i];
  if (s == 123.456) out[0] = s;
}

}  // namespace mb200

using namespace mb200;

extern "C" {

int mb200_device_count(void) {
  // probed once per process: cudaGetDeviceProperties costs milliseconds per device on a multi-GPU host
  static std::once_flag once;
  static int usable = 0;
  std::call_once(once, [] {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return; }
    for (int i = 0; i < n; ++i) {
      int major = 0, minor = 0;
      if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, i) == cudaSuccess &&
          cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, i) == cudaSuccess && major == 9 && minor == 0)
        ++usable;
    }
  });
  return usable;
}

int mb200_trim(size_t keep_bytes) {
  int rc = ensure_device();
  if (rc) return rc;
  cudaDeviceSynchronize();
  cudaError_t e = cudaMemPoolTrimTo(temp_pool(), keep_bytes);
  if (e != cudaSuccess) return cuda_fail(e, "cudaMemPoolTrimTo");
  return MB200_OK;
}

int mb200_set_device(int device) {
  cudaError_t e = cudaSetDevice(device);
  if (e != cudaSuccess) { cudaGetLastError(); return cuda_fail(e, "cudaSetDevice"); }
  return ensure_device();
}

// Test / developer hook: the options of kKnobs (initialised from the environment) can be changed at run time, e.g. to
// compare a specialised kernel with the generic one in one process.  mb200_get_option also reads the launch counters.
int mb200_set_option(const char *name, int value) {
  if (!name) return fail(MB200_EINVAL, "set_option: null name");
  const int i = knob_index(name);
  if (i < 0) return fail(MB200_EINVAL, "set_option: unknown option '%s'", name);
  const KnobSpec &k = kKnobs[i];
  if (!k.valid(value)) return fail(MB200_EINVAL, "set_option: %d is not a valid value of '%s'", value, name);
  knob_store().value[i].store(k.kind == kSwitch ? value != 0 : value, std::memory_order_relaxed);
  return MB200_OK;
}

int mb200_get_option(const char *name, int *value) {
  if (!name || !value) return fail(MB200_EINVAL, "get_option: null argument");
  const int i = knob_index(name), f = family_index(name);
  if (i >= 0) *value = knob_store().value[i].load(std::memory_order_relaxed);
  else if (f >= 0) *value = static_cast<int>(g_family_launches[f].load(std::memory_order_relaxed) & 0x7fffffff);
  else return fail(MB200_EINVAL, "get_option: unknown option '%s'", name);
  return MB200_OK;
}

const char *mb200_last_error(void) { return t_error; }
const char *mb200_version(void) { return "magick-b200 0.1 (sm_90a; ImageMagick 7.1.1-45 Q16-HDRI semantics)"; }
unsigned long long mb200_launch_count(void) { return g_launches.load(); }

int mb200_synchronize(void *stream) {
  int rc = ensure_device();
  if (rc) return rc;
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : static_cast<cudaStream_t>(default_stream());
  cudaError_t e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) return cuda_fail(e, "cudaStreamSynchronize");
  return MB200_OK;
}

int mb200_probe_fp64_fma_rate(double *fma_per_second) {
  if (!fma_per_second) return fail(MB200_EINVAL, "probe: null result");
  int rc = ensure_device();
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(default_stream());
  void *buf = nullptr;
  rc = scratch(&buf, 64, 7);
  if (rc) return rc;
  cudaEvent_t a, b;
  cudaEventCreate(&a); cudaEventCreate(&b);
  const int iters = 8192, blocks = sm_count() * 2;
  double best = 0.0;
  for (int rep = 0; rep < 4; ++rep) {
    cudaEventRecord(a, s);
    fp64_probe_kernel<<<blocks, 1024, 0, s>>>(static_cast<double *>(buf), 1.0000001, 1e-9, iters);
    cudaEventRecord(b, s);
    cudaError_t e = cudaEventSynchronize(b);
    if (e != cudaSuccess) { cudaEventDestroy(a); cudaEventDestroy(b); return cuda_fail(e, "fp64 probe"); }
    float ms = 0;
    cudaEventElapsedTime(&ms, a, b);
    const double rate = static_cast<double>(blocks) * 1024.0 * 16.0 * iters / (ms * 1e-3);
    if (rep > 0 && rate > best) best = rate;
  }
  cudaEventDestroy(a); cudaEventDestroy(b);
  count_launch(4);
  *fma_per_second = best;
  return MB200_OK;
}

int mb200_malloc(void **dev_ptr, size_t bytes) {
  int rc = ensure_device();
  if (rc) return rc;
  cudaError_t e = cudaMalloc(dev_ptr, bytes ? bytes : 1);
  if (e != cudaSuccess) return cuda_fail(e, "cudaMalloc");
  return MB200_OK;
}

int mb200_free(void *dev_ptr) {
  cudaError_t e = cudaFree(dev_ptr);
  if (e != cudaSuccess) return cuda_fail(e, "cudaFree");
  return MB200_OK;
}

int mb200_malloc_host(void **host_ptr, size_t bytes) {
  int rc = ensure_device();
  if (rc) return rc;
  cudaError_t e = cudaMallocHost(host_ptr, bytes ? bytes : 1);
  if (e != cudaSuccess) return cuda_fail(e, "cudaMallocHost");
  return MB200_OK;
}

int mb200_free_host(void *host_ptr) {
  cudaError_t e = cudaFreeHost(host_ptr);
  if (e != cudaSuccess) return cuda_fail(e, "cudaFreeHost");
  return MB200_OK;
}

int mb200_upload(void *dev_dst, const void *host_src, size_t bytes, void *stream) {
  int rc = ensure_device();
  if (rc) return rc;
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : static_cast<cudaStream_t>(default_stream());
  return copy_h2d(dev_dst, host_src, bytes, s);
}

int mb200_download(void *host_dst, const void *dev_src, size_t bytes, void *stream) {
  int rc = ensure_device();
  if (rc) return rc;
  cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : static_cast<cudaStream_t>(default_stream());
  cudaPointerAttributes attr;
  if (cudaPointerGetAttributes(&attr, host_dst) == cudaSuccess &&
      (attr.type == cudaMemoryTypeHost || attr.type == cudaMemoryTypeManaged)) {       // pinned: stays asynchronous
    cudaError_t e = cudaMemcpyAsync(host_dst, dev_src, bytes, cudaMemcpyDeviceToHost, s);
    return e == cudaSuccess ? MB200_OK : cuda_fail(e, "cudaMemcpyAsync(D2H)");
  }
  cudaGetLastError();
  return copy_d2h(host_dst, dev_src, bytes, s);
}

}  // extern "C"
