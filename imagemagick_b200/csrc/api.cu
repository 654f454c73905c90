// api.cu -- the C-ABI operators (include/magick_b200.h): the host-side control flow of
// the hot path around the CUDA kernels.
//
// Mirrors the drivers in the reference (behaviour, not code):
//   MorphologyImage / MorphologyApply  MagickCore/morphology.c:4129, :3634  (kernel lists are
//     re-iterated, compound Open/Close/Smooth staging :3813-3893, `changed`-driven iteration :3919)
//   BlurImage :765, ConvolveImage :1170, GaussianBlurImage :1709, UnsharpMaskImage :4256
//     (MagickCore/effect.c)
//   ResizeImage MagickCore/resize.c:3761 (pass order :3846-3861, default filter :3806-3816)
//   TransformImageColorspace MagickCore/colorspace.c:1751
// Intermediates live in HBM as float Quantum, exactly like the reference's intermediate
// images (the rounding between passes is part of the semantics).
#include "mb200_internal.h"

#include <cuda_runtime.h>

#include <cmath>
#include <cstdlib>
#include <memory>
#include <vector>

using namespace mb200;

namespace {

struct StreamAlloc {           // stream-ordered temporary; freed (stream-ordered) on scope exit
  void *ptr = nullptr;
  cudaStream_t s;
  explicit StreamAlloc(cudaStream_t stream) : s(stream) {}
  int alloc(size_t bytes) {
    cudaError_t e = cudaMallocAsync(&ptr, bytes ? bytes : 1, temp_pool(), s);      // the library's private pool
    if (e != cudaSuccess) { ptr = nullptr; return cuda_fail(e, "cudaMallocAsync"); }
    return MB200_OK;
  }
  ~StreamAlloc() { if (ptr) cudaFreeAsync(ptr, s); }
  StreamAlloc(const StreamAlloc &) = delete;
  StreamAlloc &operator=(const StreamAlloc &) = delete;
};

int prepare(void *stream, cudaStream_t *out) {
  int rc = ensure_device();
  if (rc) return rc;
  *out = stream ? static_cast<cudaStream_t>(stream) : static_cast<cudaStream_t>(default_stream());
  return MB200_OK;
}

bool valid_image(size_t w, size_t h, int ch) { return w > 0 && h > 0 && ch >= 1 && ch <= 4; }

size_t image_bytes(size_t w, size_t h, int ch) { return w * h * static_cast<size_t>(ch) * sizeof(float); }

// Argument check of a device operator (`op` names it in the message; an operator with an output geometry also rejects an
// empty one, the reference's NegativeOrZeroImageSize), then the device state and the call's stream.
int prepare_dev(bool args_ok, const char *op, void *stream, cudaStream_t *s, size_t out_w = 1, size_t out_h = 1) {
  if (!args_ok) return fail(MB200_EINVAL, "%s: bad arguments", op);
  if (out_w == 0 || out_h == 0) return fail(MB200_EINVAL, "NegativeOrZeroImageSize");
  return prepare(stream, s);
}

// The reference's CloneImage when the output geometry equals the input's.
int clone_image(const float *src, float *dst, size_t w, size_t h, int ch, const char *what, cudaStream_t s) {
  const cudaError_t e = cudaMemcpyAsync(dst, src, image_bytes(w, h, ch), cudaMemcpyDeviceToDevice, s);
  return e == cudaSuccess ? MB200_OK : cuda_fail(e, what);
}

// One MorphologyPrimitive launch.  d_counter may be null.
int primitive(const float *src, float *dst, size_t w, size_t h, int ch, int method,
              const mb200_kernel_info *k, double bias, unsigned long long *d_counter, cudaStream_t s,
              const UnsharpEpilogue *epilogue = nullptr, bool *epilogue_fused = nullptr) {
  const TuningKnobs knobs = tuning_knobs();
  const int kw = static_cast<int>(k->width), kh = static_cast<int>(k->height);
  const size_t n = k->width * k->height;
  std::vector<double> win(n);
  int ox, oy;
  bool has_nan = false;
  if (method == MB200_ConvolveMorphology || method == MB200_DilateMorphology || method == MB200_DilateIntensityMorphology ||
      method == MB200_IterativeDistanceMorphology) {                              // reflected, :2612-2626
    for (size_t i = 0; i < n; ++i) win[i] = k->values[n - 1 - i];
    ox = kw - static_cast<int>(k->x) - 1;
    oy = kh - static_cast<int>(k->y) - 1;
  } else if (method == MB200_ErodeMorphology || method == MB200_ErodeIntensityMorphology ||
             method == MB200_HitAndMissMorphology || method == MB200_ThinningMorphology ||
             method == MB200_ThickenMorphology) {
    for (size_t i = 0; i < n; ++i) win[i] = k->values[i];
    ox = static_cast<int>(k->x);
    oy = static_cast<int>(k->y);
  } else {
    return fail(MB200_EUNSUPPORTED, "morphology primitive %d is not implemented on the GPU path", method);
  }
  for (double v : win) if (std::isnan(v)) has_nan = true;
  if (ox < 0 || oy < 0 || ox >= kw || oy >= kh) return fail(MB200_EINVAL, "kernel origin outside the kernel");
  if (method == MB200_ConvolveMorphology && !has_nan && (kw == 1 || kh == 1)) {
    // width-1 kernels take the reference's column path (:2654); for all-finite taps its extra
    // gamma*(height/count) factor is exactly 1.
    const int axis = (kw == 1) ? 1 : 0;
    const int rc = launch_conv1d(src, dst, w, h, ch, axis, win.data(), axis == 1 ? kh : kw, axis == 1 ? oy : ox,
                                 bias, 1.0, d_counter, s, 0, epilogue, epilogue_fused);
    if (rc != MB200_EUNSUPPORTED) return rc;
  }
  if (method == MB200_ConvolveMorphology && !has_nan && kw > 1 && kh > 1 && kw <= 33 && kh <= 33 && ch == 4 &&
      bias == 0.0 && d_counter == nullptr && !knobs.no_rank1) {
    // Rank-1 kernels with non-negative taps ("gaussian:RxS", "binomial", "square" ...): K[v][u] = a[v] * b[u]
    // to 1e-14, so the kw*kh-tap sum is evaluated as a row pass that keeps RAW double sums and a column
    // pass that normalises -- same double accumulation as MorphologyPrimitive's inner loop
    // (morphology.c:2837-2871) without the float rounding a two-kernel list would add between passes.
    size_t pivot = 0;
    bool nonneg = true;
    for (size_t i = 0; i < n; ++i) {
      if (win[i] < 0.0) nonneg = false;
      if (win[i] > win[pivot]) pivot = i;
    }
    if (nonneg && win[pivot] > 0.0) {
      const int pv = static_cast<int>(pivot) / kw, pu = static_cast<int>(pivot) % kw;
      std::vector<double> colf(kh), rowf(kw);
      for (int v = 0; v < kh; ++v) colf[v] = win[static_cast<size_t>(v) * kw + pu];
      for (int u = 0; u < kw; ++u) rowf[u] = win[static_cast<size_t>(pv) * kw + u] / win[pivot];
      bool rank1 = true;
      for (int v = 0; v < kh && rank1; ++v)
        for (int u = 0; u < kw; ++u)
          if (std::fabs(win[static_cast<size_t>(v) * kw + u] - colf[v] * rowf[u]) > 1.0e-14 * win[pivot]) { rank1 = false; break; }
      if (rank1) {
        StreamAlloc sums(s);
        int rc = sums.alloc(w * h * 4 * sizeof(double));
        if (rc == MB200_OK) {
          rc = launch_conv1d(src, static_cast<float *>(sums.ptr), w, h, ch, 0, rowf.data(), kw, ox, 0.0, 1.0, nullptr, s, 1);
          if (rc == MB200_OK)
            rc = launch_conv1d(static_cast<const float *>(sums.ptr), dst, w, h, ch, 1, colf.data(), kh, oy, 0.0, 1.0,
                               nullptr, s, 2);
          if (rc != MB200_EUNSUPPORTED) return rc;
        }
        // allocation failure / unsupported geometry: fall through to the direct 2-D kernel
      }
    }
  }
  if ((method == MB200_ErodeMorphology || method == MB200_DilateMorphology) && d_counter == nullptr &&
      !knobs.no_morph_stream) {                            // register-streaming kernel for the built-in shapes
    const int rc = launch_morph_stream(src, dst, w, h, ch, method, win.data(), kw, kh, ox, oy, s);
    if (rc != MB200_EUNSUPPORTED) return rc;
  }
  double gamma_scale = 1.0;
  if (method == MB200_ConvolveMorphology && kw == 1) {
    size_t count = 0;
    for (double v : win) if (!std::isnan(v)) ++count;
    if (count != 0) gamma_scale = static_cast<double>(kh) / static_cast<double>(count);
  }
  return launch_morph2d(src, dst, w, h, ch, method, win.data(), kw, kh, ox, oy, bias, gamma_scale, d_counter, s);
}

// One primitive that counts its changed channel values in d_counter, read back (this synchronises the stream) as the
// reference's `changed` = per-channel changes / number of Update channels (image-private.h:147).
int counted_primitive(const float *src, float *dst, size_t w, size_t h, int ch, int method, const mb200_kernel_info *k,
                      double bias, unsigned long long *d_counter, long long *changed, cudaStream_t s) {
  cudaMemsetAsync(d_counter, 0, sizeof(unsigned long long), s);
  const int rc = primitive(src, dst, w, h, ch, method, k, bias, d_counter, s);
  if (rc) return rc;
  unsigned long long hostv = 0;
  cudaError_t e = cudaMemcpyAsync(&hostv, d_counter, sizeof(hostv), cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) return cuda_fail(e, "changed readback");
  *changed = static_cast<long long>(hostv / static_cast<unsigned long long>(ch));
  return MB200_OK;
}

struct Stage { int primitive; const mb200_kernel_info *kernel; };

// HitAndMiss / Thinning / Thicken (morphology.c:3722-3729): `iterations` repeats the WHOLE method (every kernel of the list
// once per round) while anything changes.  Thinning / Thicken re-iterate: each kernel works on the previous kernel's
// result.  HitAndMiss unites the kernels' results with LightenCompositeOp (:4016-4052): the first result is kept, every
// further one -- computed from the ORIGINAL image -- is composited onto it; a one-kernel list iterates on its own result.
int apply_hit_and_miss_family(const float *src, float *dst, size_t w, size_t h, int ch, int method, long iterations,
                              const mb200_kernel_info *kernel, cudaStream_t s) {
  const size_t method_limit = iterations < 0 ? (w > h ? w : h) : static_cast<size_t>(iterations);
  const bool unite = method == MB200_HitAndMissMorphology && kernel->next != nullptr;
  const size_t bytes = w * h * static_cast<size_t>(ch) * sizeof(float), npix = w * h;
  StreamAlloc a(s), b(s), united(s), counter(s);
  int rc = a.alloc(bytes);
  if (!rc) rc = b.alloc(bytes);
  if (!rc && unite) rc = united.alloc(bytes);
  if (!rc) rc = counter.alloc(sizeof(unsigned long long));
  if (rc) return rc;
  float *bufs[2] = {static_cast<float *>(a.ptr), static_cast<float *>(b.ptr)};
  unsigned long long *d_counter = static_cast<unsigned long long *>(counter.ptr);
  const float *cur = src;
  int next = 0;
  bool have_united = false;
  size_t round = 0;
  long long round_changed = 1;
  while (round < method_limit && round_changed > 0) {
    ++round;
    round_changed = 0;
    for (const mb200_kernel_info *k = kernel; k; k = k->next) {
      if (method_limit > 1) {                   // the count only decides whether another round runs
        long long changed = 0;
        rc = counted_primitive(cur, bufs[next], w, h, ch, method, k, 0.0, d_counter, &changed, s);
        round_changed += changed;
      } else {
        rc = primitive(cur, bufs[next], w, h, ch, method, k, 0.0, nullptr, s);
      }
      if (rc) return rc;
      cur = bufs[next];
      next ^= 1;
      if (unite) {
        if (!have_united) {
          const cudaError_t e = cudaMemcpyAsync(united.ptr, cur, bytes, cudaMemcpyDeviceToDevice, s);
          if (e != cudaSuccess) return cuda_fail(e, "hit-and-miss: first result");
          have_united = true;
        } else {
          rc = launch_composite_lighten(static_cast<float *>(united.ptr), cur, npix, ch, s);
          if (rc) return rc;
        }
        cur = src;
      }
    }
  }
  const cudaError_t e = cudaMemcpyAsync(dst, unite ? united.ptr : cur, bytes, cudaMemcpyDeviceToDevice, s);
  return e == cudaSuccess ? MB200_OK : cuda_fail(e, "hit-and-miss: result copy");
}

int morphology_apply(const float *src, float *dst, size_t w, size_t h, int ch, int method, long iterations,
                     const mb200_kernel_info *kernel, double bias, cudaStream_t s,
                     const UnsharpEpilogue *epilogue = nullptr, bool *epilogue_fused = nullptr) {
  // Methods that end in "difference with the original" (staging :3813-3893, CompositeImage :3995-4012):
  // the morphological part is one of the methods below, then one Difference composite.
  if (method == MB200_EdgeInMorphology || method == MB200_EdgeOutMorphology || method == MB200_EdgeMorphology ||
      method == MB200_TopHatMorphology || method == MB200_BottomHatMorphology) {
    if (kernel->next != nullptr)
      return fail(MB200_EUNSUPPORTED, "compound difference methods with a multi-kernel list stay on the CPU path");
    const size_t npix = w * h;
    if (method == MB200_EdgeMorphology) {          // dilate; erode the ORIGINAL; canvas = eroded, source = dilated
      StreamAlloc dil(s);
      int rc = dil.alloc(npix * static_cast<size_t>(ch) * sizeof(float));
      if (rc) return rc;
      rc = morphology_apply(src, static_cast<float *>(dil.ptr), w, h, ch, MB200_DilateMorphology, iterations, kernel, bias, s);
      if (!rc) rc = morphology_apply(src, dst, w, h, ch, MB200_ErodeMorphology, iterations, kernel, bias, s);
      if (!rc) rc = launch_composite_difference(dst, static_cast<const float *>(dil.ptr), npix, ch, s);
      return rc;
    }
    const int base = method == MB200_EdgeInMorphology ? MB200_ErodeMorphology
                     : method == MB200_EdgeOutMorphology ? MB200_DilateMorphology
                     : method == MB200_TopHatMorphology ? MB200_OpenMorphology : MB200_CloseMorphology;
    int rc = morphology_apply(src, dst, w, h, ch, base, iterations, kernel, bias, s);
    if (!rc) rc = launch_composite_difference(dst, src, npix, ch, s);
    return rc;
  }
  if (iterations == 0) return fail(MB200_EINVAL, "iterations == 0 is a null operation (reference returns NULL)");
  if (method == MB200_HitAndMissMorphology || method == MB200_ThinningMorphology || method == MB200_ThickenMorphology)
    return apply_hit_and_miss_family(src, dst, w, h, ch, method, iterations, kernel, s);
  size_t kernel_limit = iterations < 0 ? (w > h ? w : h) : static_cast<size_t>(iterations);
  int stage_limit = 1;
  switch (method) {
    case MB200_SmoothMorphology: stage_limit = 4; break;
    case MB200_OpenMorphology: case MB200_CloseMorphology:
    case MB200_OpenIntensityMorphology: case MB200_CloseIntensityMorphology: stage_limit = 2; break;
    case MB200_ConvolveMorphology: case MB200_CorrelateMorphology:
    case MB200_ErodeMorphology: case MB200_DilateMorphology:
    case MB200_ErodeIntensityMorphology: case MB200_DilateIntensityMorphology:
    case MB200_IterativeDistanceMorphology: break;
    default:
      return fail(MB200_EUNSUPPORTED, "morphology method %d (Distance / Voronoi: sequential two-pass primitives) is not on "
                  "the GPU path", method);
  }
  // 180-degree reflection used by Correlate/Close/Smooth (:3779-3793, RotateKernelInfo :4258)
  KernelList reflected;
  if (method == MB200_CorrelateMorphology || method == MB200_CloseMorphology || method == MB200_SmoothMorphology ||
      method == MB200_CloseIntensityMorphology) {
    reflected.reset(mb200_clone_kernel_info(kernel));
    if (!reflected) return fail(MB200_ENOMEM, "kernel clone failed");
    rotate_kernel_info(reflected.get(), 180.0);
  }
  std::vector<Stage> stages;
  const mb200_kernel_info *rk = reflected.get();
  for (const mb200_kernel_info *nk = kernel; nk; nk = nk->next, rk = rk ? rk->next : nullptr) {
    for (int stage = 1; stage <= stage_limit; ++stage) {
      Stage st{method, nk};
      switch (method) {
        case MB200_OpenMorphology: st.primitive = stage == 2 ? MB200_DilateMorphology : MB200_ErodeMorphology; break;
        case MB200_CloseMorphology: st.kernel = rk; st.primitive = stage == 2 ? MB200_ErodeMorphology : MB200_DilateMorphology; break;
        case MB200_OpenIntensityMorphology:
          st.primitive = stage == 2 ? MB200_DilateIntensityMorphology : MB200_ErodeIntensityMorphology;
          break;
        case MB200_CloseIntensityMorphology:
          st.kernel = rk;
          st.primitive = stage == 2 ? MB200_ErodeIntensityMorphology : MB200_DilateIntensityMorphology;
          break;
        case MB200_SmoothMorphology:
          if (stage == 1) st.primitive = MB200_ErodeMorphology;
          else if (stage == 2) st.primitive = MB200_DilateMorphology;
          else if (stage == 3) { st.kernel = rk; st.primitive = MB200_DilateMorphology; }
          else { st.kernel = rk; st.primitive = MB200_ErodeMorphology; }
          break;
        case MB200_CorrelateMorphology: st.kernel = rk; st.primitive = MB200_ConvolveMorphology; break;
        default: break;
      }
      stages.push_back(st);
    }
  }
  const size_t bytes = w * h * static_cast<size_t>(ch) * sizeof(float);
  int rc = MB200_OK;
  if (kernel_limit == 1) {
    // Every stage runs exactly once: ping-pong between one temporary and dst so that the last
    // primitive writes dst (no trailing copy).
    const size_t total = stages.size();
    StreamAlloc tmp(s);
    if (total > 1) { rc = tmp.alloc(bytes); }
    const float *cur = src;
    for (size_t i = 0; i < total && rc == MB200_OK; ++i) {
      float *out = ((total - 1 - i) % 2 == 0) ? dst : static_cast<float *>(tmp.ptr);
      const bool last = i + 1 == total;
      rc = primitive(cur, out, w, h, ch, stages[i].primitive, stages[i].kernel, bias, nullptr, s,
                     last ? epilogue : nullptr, last ? epilogue_fused : nullptr);
      cur = out;
    }
  } else {
    // `changed`-driven iteration (:3919-3962): needs the count after every primitive.
    StreamAlloc a(s), b(s), counter(s);
    rc = a.alloc(bytes);
    if (!rc) rc = b.alloc(bytes);
    if (!rc) rc = counter.alloc(sizeof(unsigned long long));
    const float *cur = src;
    float *bufs[2] = {static_cast<float *>(a.ptr), static_cast<float *>(b.ptr)};
    int next = 0;
    for (size_t i = 0; i < stages.size() && rc == MB200_OK; ++i) {
      size_t loop = 0;
      long long changed = 1;
      while (loop < kernel_limit && changed > 0 && rc == MB200_OK) {
        ++loop;
        rc = counted_primitive(cur, bufs[next], w, h, ch, stages[i].primitive, stages[i].kernel, bias,
                               static_cast<unsigned long long *>(counter.ptr), &changed, s);
        cur = bufs[next];
        next ^= 1;
      }
    }
    if (rc == MB200_OK) {
      cudaError_t e = cudaMemcpyAsync(dst, cur, bytes, cudaMemcpyDeviceToDevice, s);
      if (e != cudaSuccess) rc = cuda_fail(e, "result copy");
    }
  }
  return rc;
}

// Host-buffer operators: check the buffers and the geometry (`name` names the operator in the message), then run
// `op(d_src, d_dst, stream)` on the HBM copies of the host buffers (cache.cu): an attached pixel cache keeps its HBM copy
// between calls (and, in lazy mode, its result stays there until mb200_cache_sync); anything else is staged through
// stream-ordered temporaries.  Pageable memory travels through the threaded pinned bounce ring.
// The form with `och` is for operators whose output has its own channel count (the caller checks both counts).
template <typename Op>
int with_staging(const char *name, const float *src, size_t w, size_t h, int ch, float *dst, size_t ow, size_t oh, int och,
                 Op op) {
  if (!src || !dst || w == 0 || h == 0 || ch < 1 || och < 1 || ow == 0 || oh == 0)
    return fail(MB200_EINVAL, "%s: bad arguments", name);
  cudaStream_t s;
  int rc = prepare(nullptr, &s);
  if (rc) return rc;
  StageRef in, out;
  rc = stage_input(src, image_bytes(w, h, ch), s, &in);
  if (!rc) rc = stage_output(dst, image_bytes(ow, oh, och), s, &out);
  if (!rc) rc = op(static_cast<const float *>(in.dev), static_cast<float *>(out.dev), s);
  if (rc) cudaStreamSynchronize(s);
  else rc = finish_output(&out, s);
  release_stage(&in, s);
  release_stage(&out, s);
  return rc;
}
template <typename Op>
int with_staging(const char *name, const float *src, size_t w, size_t h, int ch, float *dst, size_t ow, size_t oh, Op op) {
  if (!src || !dst || !valid_image(w, h, ch) || ow == 0 || oh == 0) return fail(MB200_EINVAL, "%s: bad arguments", name);
  return with_staging(name, src, w, h, ch, dst, ow, oh, ch, op);
}

// In-place operators on a host buffer.
template <typename Op>
int in_place_host(const char *name, float *buf, size_t w, size_t h, int ch, Op op) {
  if (!buf || !valid_image(w, h, ch)) return fail(MB200_EINVAL, "%s: bad arguments", name);
  cudaStream_t s;
  int rc = prepare(nullptr, &s);
  if (rc) return rc;
  StageRef io;
  rc = stage_input(buf, image_bytes(w, h, ch), s, &io);
  if (!rc) rc = op(static_cast<float *>(io.dev), s);
  if (rc) cudaStreamSynchronize(s);
  else rc = finish_output(&io, s);
  release_stage(&io, s);
  return rc;
}

// Operators that update a host buffer (ow x oh, already holding the operator's result; resident when attached) from
// its source (w x h): `op(d_buf, d_src, stream)`.
template <typename Op>
int update_host(const char *name, float *buf, size_t ow, size_t oh, const float *src, size_t w, size_t h, int ch, Op op) {
  if (!buf || !src || !valid_image(w, h, ch) || ow == 0 || oh == 0) return fail(MB200_EINVAL, "%s: bad arguments", name);
  cudaStream_t s;
  int rc = prepare(nullptr, &s);
  if (rc) return rc;
  StageRef io, in;
  rc = stage_input(buf, image_bytes(ow, oh, ch), s, &io);
  if (!rc) rc = stage_input(src, image_bytes(w, h, ch), s, &in);
  if (!rc) rc = op(static_cast<float *>(io.dev), static_cast<const float *>(in.dev), s);
  if (rc) cudaStreamSynchronize(s);
  else rc = finish_output(&io, s);
  release_stage(&in, s);
  release_stage(&io, s);
  return rc;
}

// ResizeImage's scale factors and default filter (resize.c:3797-3816).
struct ResizeChoice {
  double x_factor, y_factor;
  int filter;
};
ResizeChoice resize_choice(size_t width, size_t height, size_t out_width, size_t out_height, int channels, int filter) {
  auto reciprocal = [](double x) { return std::fabs(x) >= 1.0e-12 ? 1.0 / x : (x < 0 ? -1.0e12 : 1.0e12); };
  ResizeChoice c;
  c.x_factor = static_cast<double>(out_width) * reciprocal(static_cast<double>(width));
  c.y_factor = static_cast<double>(out_height) * reciprocal(static_cast<double>(height));
  c.filter = MB200_LanczosFilter;
  if (filter != MB200_UndefinedFilter) c.filter = filter;
  else if (c.x_factor == 1.0 && c.y_factor == 1.0) c.filter = MB200_PointFilter;
  else if (has_alpha(channels) || (c.x_factor * c.y_factor) > 1.0) c.filter = MB200_MitchellFilter;
  return c;
}

}  // namespace

extern "C" {

int mb200_morphology_primitive_dev(const float *src, float *dst, size_t width, size_t height, int channels,
                                   int method, const mb200_kernel_info *kernel, double bias, long long *changed,
                                   void *stream) {
  cudaStream_t s;
  int rc = prepare_dev(src && dst && kernel && kernel->values && valid_image(width, height, channels),
                       "morphology_primitive", stream, &s);
  if (rc) return rc;
  if (!changed) return primitive(src, dst, width, height, channels, method, kernel, bias, nullptr, s);
  StreamAlloc counter(s);
  rc = counter.alloc(sizeof(unsigned long long));
  if (rc) return rc;
  return counted_primitive(src, dst, width, height, channels, method, kernel, bias,
                           static_cast<unsigned long long *>(counter.ptr), changed, s);
}

int mb200_morphology_image_dev(const float *src, float *dst, size_t width, size_t height, int channels,
                               int method, long iterations, const mb200_kernel_info *kernel, double bias,
                               void *stream) {
  cudaStream_t s;
  const int rc = prepare_dev(src && dst && src != dst && kernel && valid_image(width, height, channels),
                             "morphology_image", stream, &s);
  if (rc) return rc;
  return morphology_apply(src, dst, width, height, channels, method, iterations, kernel, bias, s);
}

// Distance / Voronoi: the arguments are checked before the device; forward pass into a pool temporary, reverse into dst.
static int morphology_direct_args(const float *src, const float *dst, size_t width, size_t height, int channels,
                                  int method, const mb200_kernel_info *kernel) {
  if (!src || !dst || src == dst || !valid_image(width, height, channels))
    return fail(MB200_EINVAL, "morphology direct: bad arguments");
  if (width > (1u << 30) || height > (1u << 30))
    return fail(MB200_EUNSUPPORTED, "morphology direct: images wider or taller than 2^30 are not supported");
  return morphology_direct_check(channels, method, kernel);
}

int mb200_morphology_direct_image_dev(const float *src, float *dst, size_t width, size_t height, int channels,
                                      int method, const mb200_kernel_info *kernel, void *stream) {
  int rc = morphology_direct_args(src, dst, width, height, channels, method, kernel);
  cudaStream_t s;
  if (!rc) rc = prepare(stream, &s);
  if (rc) return rc;
  StreamAlloc tmp(s);
  rc = tmp.alloc(image_bytes(width, height, channels));
  if (rc) return rc;
  return launch_morphology_direct(src, static_cast<float *>(tmp.ptr), dst, width, height, channels, method, kernel, s);
}

int mb200_distort_image_dev(const float *src, size_t width, size_t height, int channels, float *dst,
                            const mb200_distort_params *plan, const mb200_resample_options *options, void *stream) {
  if (!src || !dst || src == dst) return fail(MB200_EINVAL, "distort: bad arguments");
  int rc = distort_check(width, height, channels, plan, options);
  cudaStream_t s;
  if (!rc) rc = prepare(stream, &s);
  if (rc) return rc;
  return launch_distort(src, width, height, channels, dst, plan, options, s);
}

int mb200_geometry_image_dev(const float *src, size_t width, size_t height, int channels, float *dst,
                             const mb200_geometry_params *plan, void *stream) {
  if (!src || !dst || src == dst) return fail(MB200_EINVAL, "geometry: bad arguments");
  int rc = geometry_check(width, height, channels, plan);
  cudaStream_t s;
  if (!rc) rc = prepare(stream, &s);
  if (rc) return rc;
  return launch_geometry(src, width, height, channels, dst, plan, s);
}

// The scan writes the row summaries into a pool temporary; they come back to the host for the serial rule.
int mb200_bounding_box_dev(const float *src, size_t width, size_t height, int channels,
                           const mb200_trim_options *options, mb200_page *box, int *warning, void *stream) {
  if (!src || !box) return fail(MB200_EINVAL, "bounding box: bad arguments");
  int rc = bounding_box_check(width, height, channels, options);
  cudaStream_t s;
  if (!rc) rc = prepare(stream, &s);
  if (rc) return rc;
  std::vector<unsigned> summaries(height * 4);
  {
    StreamAlloc rows(s);
    rc = rows.alloc(summaries.size() * sizeof(unsigned));
    if (!rc) rc = launch_bounding_box(src, width, height, channels, options, static_cast<unsigned *>(rows.ptr), s);
    if (!rc) {
      const cudaError_t e = cudaMemcpyAsync(summaries.data(), rows.ptr, summaries.size() * sizeof(unsigned),
                                            cudaMemcpyDeviceToHost, s);
      if (e != cudaSuccess) rc = cuda_fail(e, "bounding box: summaries");
    }
  }
  const cudaError_t e = cudaStreamSynchronize(s);
  if (!rc && e != cudaSuccess) rc = cuda_fail(e, "bounding box");
  if (rc) return rc;
  return mb200_bounding_box_from_rows(summaries.data(), width, height, options->edges, box, warning);
}

int mb200_convolve_image_dev(const float *src, float *dst, size_t width, size_t height, int channels,
                             const mb200_kernel_info *kernel, void *stream) {
  return mb200_morphology_image_dev(src, dst, width, height, channels, MB200_ConvolveMorphology, 1, kernel, 0.0,
                                    stream);
}

int mb200_blur_image_dev(const float *src, float *dst, size_t width, size_t height, int channels, double radius,
                         double sigma, void *stream) {
  const KernelList k = blur_kernel_pair(radius, sigma);
  if (!k) return fail(MB200_ENOMEM, "blur kernel");
  return mb200_convolve_image_dev(src, dst, width, height, channels, k.get(), stream);
}

int mb200_gaussian_blur_image_dev(const float *src, float *dst, size_t width, size_t height, int channels,
                                  double radius, double sigma, void *stream) {
  const KernelList k(mb200_acquire_kernel_builtin(MB200_GaussianKernel, radius, sigma, 0.0, 0.0));
  if (!k) return fail(MB200_ENOMEM, "gaussian kernel");
  return mb200_convolve_image_dev(src, dst, width, height, channels, k.get(), stream);
}

int mb200_unsharp_mask_image_dev(const float *src, float *dst, size_t width, size_t height, int channels,
                                 double radius, double sigma, double gain, double threshold, void *stream) {
  cudaStream_t s;
  int rc = prepare_dev(src && dst && src != dst && valid_image(width, height, channels), "unsharp", stream, &s);
  if (rc) return rc;
  // BlurImage (effect.c:4295) + the point pass (:4310-4384).  With the RGBA pair kernels the point pass is the
  // epilogue of the blur's column pass: it is applied to the float-ROUNDED blur value, exactly what the reference
  // reads back from its blurred image, so the fused and the two-launch forms produce the same bits while the fused one
  // saves the 48 B/pixel of the separate pass.
  const KernelList k = blur_kernel_pair(radius, sigma);
  if (!k) return fail(MB200_ENOMEM, "blur kernel");
  const UnsharpEpilogue epi{src, gain, 65535.0 * threshold};
  bool fused = false;
  rc = morphology_apply(src, dst, width, height, channels, MB200_ConvolveMorphology, 1, k.get(), 0.0, s,
                        tuning_knobs().no_fused_unsharp ? nullptr : &epi, &fused);
  if (rc || fused) return rc;
  return launch_unsharp_combine(src, dst, width * height * static_cast<size_t>(channels), gain,
                                65535.0 * threshold, s);
}

int mb200_resize_image_dev(const float *src, size_t width, size_t height, int channels, float *dst,
                           size_t out_width, size_t out_height, int filter, void *stream) {
  return mb200_resize_image_ex_dev(src, width, height, channels, dst, out_width, out_height, filter, nullptr, stream);
}

int mb200_resize_image_ex_dev(const float *src, size_t width, size_t height, int channels, float *dst,
                              size_t out_width, size_t out_height, int filter, const mb200_filter_options *options,
                              void *stream) {
  cudaStream_t s;
  int rc = prepare_dev(src && dst && valid_image(width, height, channels), "resize", stream, &s, out_width,
                       out_height);                                                                // :3791
  if (rc) return rc;
  if (out_width == width && out_height == height && filter == MB200_UndefinedFilter)               // :3793-3795
    return clone_image(src, dst, width, height, channels, "resize: clone", s);
  const size_t px = static_cast<size_t>(channels) * sizeof(float);
  if (((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) != 0) {
    // The resize kernels move whole pixels (float2 / float4 loads and stores, 16-byte cp.async and TMA copies): a pixel
    // cache that is not 16-byte aligned (a view that starts inside a buffer) is resized through aligned copies.
    StreamAlloc in(s), out(s);
    rc = in.alloc(width * height * px);
    if (!rc) rc = out.alloc(out_width * out_height * px);
    if (rc) return rc;
    cudaError_t e = cudaMemcpyAsync(in.ptr, src, width * height * px, cudaMemcpyDeviceToDevice, s);
    if (e != cudaSuccess) return cuda_fail(e, "resize: aligned copy of the source");
    rc = mb200_resize_image_ex_dev(static_cast<const float *>(in.ptr), width, height, channels,
                                   static_cast<float *>(out.ptr), out_width, out_height, filter, options, s);
    if (rc) return rc;
    e = cudaMemcpyAsync(dst, out.ptr, out_width * out_height * px, cudaMemcpyDeviceToDevice, s);
    return e == cudaSuccess ? MB200_OK : cuda_fail(e, "resize: result copy");
  }
  const ResizeChoice c = resize_choice(width, height, out_width, out_height, channels, filter);
  std::shared_ptr<const ResizeAxis> tx, ty;
  rc = resize_axis_tables(c.filter, options, width, out_width, c.x_factor, &tx);
  if (!rc) rc = resize_axis_tables(c.filter, options, height, out_height, c.y_factor, &ty);
  if (rc) return rc;
  const TuningKnobs knobs = tuning_knobs();
  auto run_axis = [&](const float *in, size_t w, size_t h, float *out, int axis, const ResizeAxis &t) -> int {
    if (channels == 4 && !knobs.no_resize_stream) {         // streaming kernels (+ border gather CTAs)
      const int rs = launch_resize_stream(in, w, h, out, axis, t, s);
      if (rs != MB200_EUNSUPPORTED) return rs;
    }
    // the tiled regular kernel along x is opt-in (slower than the gather kernel when last measured)
    return launch_resize_axis(in, w, h, channels, out, axis, t, axis == 1 || knobs.resize_regular_h, s);
  };
  // Equal integer reduction on both axes (the reference filters vertically first when x_factor <= y_factor, :3854-3861):
  // one fused launch keeps the vertically filtered intermediate of every output tile in shared memory, with the same
  // bits as the two passes.  It moves 20 B per source pixel through HBM instead of 36, which pays once the two-pass
  // intermediate no longer stays in L2; below that the two passes' extra traffic never leaves the chip and they are
  // faster (DESIGN §5.4).
  const bool big = width * out_height * px > l2_bytes();
  if (channels == 4 && c.x_factor == c.y_factor && !knobs.no_resize_stream && !knobs.no_resize_fused &&
      (knobs.resize_fused || big)) {
    rc = launch_resize_fused(src, width, height, dst, *tx, *ty, s);
    if (rc != MB200_EUNSUPPORTED) return rc;
  }
  StreamAlloc tmp(s);
  if (c.x_factor > c.y_factor) {                                                                   // :3846-3853
    rc = tmp.alloc(out_width * height * px);
    if (rc) return rc;
    rc = run_axis(src, width, height, static_cast<float *>(tmp.ptr), 0, *tx);
    if (rc) return rc;
    rc = run_axis(static_cast<float *>(tmp.ptr), out_width, height, dst, 1, *ty);
  } else {                                                                                         // :3854-3861
    rc = tmp.alloc(width * out_height * px);
    if (rc) return rc;
    rc = run_axis(src, width, height, static_cast<float *>(tmp.ptr), 1, *ty);
    if (rc) return rc;
    rc = run_axis(static_cast<float *>(tmp.ptr), width, out_height, dst, 0, *tx);
  }
  return rc;
}

int mb200_transform_colorspace_ex_dev(float *buf, size_t width, size_t height, int channels, int from, int to,
                                      const mb200_colorspace_options *options, void *stream) {
  cudaStream_t s;
  const int rc = prepare_dev(buf && valid_image(width, height, channels), "colorspace", stream, &s);
  if (rc) return rc;
  return launch_colorspace(buf, width * height, channels, from, to, options, s);
}

int mb200_transform_colorspace_dev(float *buf, size_t width, size_t height, int channels, int from, int to,
                                   void *stream) {
  return mb200_transform_colorspace_ex_dev(buf, width, height, channels, from, to, nullptr, stream);
}

int mb200_colorspace_channels(int colorspace, int has_alpha) {
  const int base = colorspace == MB200_CMYKColorspace ? 4
                 : (colorspace == MB200_GRAYColorspace || colorspace == MB200_LinearGRAYColorspace) ? 1 : 3;
  return base + (has_alpha != 0 ? 1 : 0);
}

int mb200_transform_colorspace_layout_dev(const float *src, int src_channels, float *dst, int dst_channels, size_t width,
                                          size_t height, int from, int to, const mb200_colorspace_options *options,
                                          void *stream) {
  int rc = colorspace_layout_check(src, src_channels, dst, dst_channels, width, height, from, to, options);
  cudaStream_t s;
  if (!rc) rc = prepare(stream, &s);
  if (rc) return rc;
  return launch_colorspace_layout(src, src_channels, dst, dst_channels, width * height, from, to, options, s);
}

// ------------------------------------------------------------ host buffers

int mb200_blur_image(const float *src, float *dst, size_t w, size_t h, int ch, double radius, double sigma) {
  return with_staging("blur", src, w, h, ch, dst, w, h, [&](const float *s, float *d, cudaStream_t st) {
    return mb200_blur_image_dev(s, d, w, h, ch, radius, sigma, st);
  });
}

int mb200_gaussian_blur_image(const float *src, float *dst, size_t w, size_t h, int ch, double radius,
                              double sigma) {
  return with_staging("gaussian blur", src, w, h, ch, dst, w, h, [&](const float *s, float *d, cudaStream_t st) {
    return mb200_gaussian_blur_image_dev(s, d, w, h, ch, radius, sigma, st);
  });
}

int mb200_convolve_image(const float *src, float *dst, size_t w, size_t h, int ch, const mb200_kernel_info *kernel) {
  if (!kernel) return fail(MB200_EINVAL, "convolve: bad arguments");
  return with_staging("convolve", src, w, h, ch, dst, w, h, [&](const float *s, float *d, cudaStream_t st) {
    return mb200_convolve_image_dev(s, d, w, h, ch, kernel, st);
  });
}

int mb200_morphology_image(const float *src, float *dst, size_t w, size_t h, int ch, int method, long iterations,
                           const mb200_kernel_info *kernel, double bias) {
  if (!kernel) return fail(MB200_EINVAL, "morphology: bad arguments");
  return with_staging("morphology", src, w, h, ch, dst, w, h, [&](const float *s, float *d, cudaStream_t st) {
    return mb200_morphology_image_dev(s, d, w, h, ch, method, iterations, kernel, bias, st);
  });
}

int mb200_morphology_direct_image(const float *src, float *dst, size_t w, size_t h, int ch, int method,
                                  const mb200_kernel_info *kernel) {
  const int rc = morphology_direct_args(src, dst, w, h, ch, method, kernel);
  if (rc) return rc;
  return with_staging("morphology direct", src, w, h, ch, dst, w, h, [&](const float *s, float *d, cudaStream_t st) {
    return mb200_morphology_direct_image_dev(s, d, w, h, ch, method, kernel, st);
  });
}

int mb200_distort_image(const float *src, size_t w, size_t h, int ch, float *dst, const mb200_distort_params *plan,
                        const mb200_resample_options *options) {
  if (!src || !dst) return fail(MB200_EINVAL, "distort: bad arguments");
  const int rc = distort_check(w, h, ch, plan, options);
  if (rc) return rc;
  return with_staging("distort", src, w, h, ch, dst, plan->columns, plan->rows, [&](const float *s, float *d, cudaStream_t st) {
    return mb200_distort_image_dev(s, w, h, ch, d, plan, options, st);
  });
}

int mb200_geometry_image(const float *src, size_t w, size_t h, int ch, float *dst, const mb200_geometry_params *plan) {
  if (!src || !dst) return fail(MB200_EINVAL, "geometry: bad arguments");
  const int rc = geometry_check(w, h, ch, plan);
  if (rc) return rc;
  return with_staging("geometry", src, w, h, ch, dst, plan->columns, plan->rows, ch,
                      [&](const float *s, float *d, cudaStream_t st) {
    return mb200_geometry_image_dev(s, w, h, ch, d, plan, st);
  });
}

int mb200_bounding_box(const float *src, size_t w, size_t h, int ch, const mb200_trim_options *options,
                       mb200_page *box, int *warning) {
  if (!src || !box) return fail(MB200_EINVAL, "bounding box: bad arguments");
  int rc = bounding_box_check(w, h, ch, options);
  cudaStream_t s;
  if (!rc) rc = prepare(nullptr, &s);
  if (rc) return rc;
  StageRef in;                                                   // read only: nothing is copied back
  rc = stage_input(src, image_bytes(w, h, ch), s, &in);
  if (!rc) rc = mb200_bounding_box_dev(static_cast<const float *>(in.dev), w, h, ch, options, box, warning, s);
  if (rc) cudaStreamSynchronize(s);
  release_stage(&in, s);
  return rc;
}

int mb200_unsharp_mask_image(const float *src, float *dst, size_t w, size_t h, int ch, double radius, double sigma,
                             double gain, double threshold) {
  return with_staging("unsharp", src, w, h, ch, dst, w, h, [&](const float *s, float *d, cudaStream_t st) {
    return mb200_unsharp_mask_image_dev(s, d, w, h, ch, radius, sigma, gain, threshold, st);
  });
}

int mb200_resize_image_ex(const float *src, size_t w, size_t h, int ch, float *dst, size_t ow, size_t oh, int filter,
                          const mb200_filter_options *options) {
  return with_staging("resize", src, w, h, ch, dst, ow, oh, [&](const float *s, float *d, cudaStream_t st) {
    return mb200_resize_image_ex_dev(s, w, h, ch, d, ow, oh, filter, options, st);
  });
}
int mb200_resize_image(const float *src, size_t w, size_t h, int ch, float *dst, size_t ow, size_t oh, int filter) {
  return mb200_resize_image_ex(src, w, h, ch, dst, ow, oh, filter, nullptr);
}

int mb200_transform_colorspace_ex(float *buf, size_t w, size_t h, int ch, int from, int to,
                                  const mb200_colorspace_options *options) {
  return in_place_host("colorspace", buf, w, h, ch,
                       [&](float *d, cudaStream_t st) { return launch_colorspace(d, w * h, ch, from, to, options, st); });
}

int mb200_transform_colorspace(float *buf, size_t w, size_t h, int ch, int from, int to) {
  return mb200_transform_colorspace_ex(buf, w, h, ch, from, to, nullptr);
}

// The checks run before the buffers are staged, so a refused call moves no data.
int mb200_transform_colorspace_layout(const float *src, int src_channels, float *dst, int dst_channels, size_t w, size_t h,
                                      int from, int to, const mb200_colorspace_options *options) {
  const int rc = colorspace_layout_check(src, src_channels, dst, dst_channels, w, h, from, to, options);
  if (rc) return rc;
  return with_staging("colorspace layout", src, w, h, src_channels, dst, w, h, dst_channels,
                      [&](const float *s, float *d, cudaStream_t st) {
                        return launch_colorspace_layout(s, src_channels, d, dst_channels, w * h, from, to, options, st);
                      });
}

}  // extern "C"

// ---- threshold.c point operators ---------------------------------------------------------
namespace {
// The ParseGeometry step of Black/WhiteThresholdImage (threshold.c:955-985) for "v[,v[,v[,v]]][%]".
int parse_thresholds(const char *spec, double (&t)[4]) {
  if (spec == nullptr) return fail(MB200_EINVAL, "thresholds == NULL (the reference returns MagickTrue untouched)");
  double v[4] = {0, 0, 0, 0};
  int n = 0;
  bool percent = false;
  const char *p = spec;
  while (*p) {
    while (*p == ' ') ++p;
    if (*p == '\0') break;
    if (n == 4) return fail(MB200_EUNSUPPORTED, "threshold geometry '%s' has more than four values", spec);
    char *end = nullptr;
    v[n] = std::strtod(p, &end);
    if (end == p) return fail(MB200_EUNSUPPORTED, "threshold geometry '%s' is not of the form v[,v[,v[,v]]][%%]", spec);
    ++n;
    p = end;
    while (*p == ' ') ++p;
    if (*p == '%') { percent = true; ++p; }
    while (*p == ' ') ++p;
    if (*p == ',') ++p;
    else if (*p != '\0') return fail(MB200_EUNSUPPORTED, "threshold geometry '%s' is not of the form v[,v[,v[,v]]][%%]", spec);
  }
  if (n == 0) return fail(MB200_EUNSUPPORTED, "empty threshold geometry");
  t[0] = v[0];
  t[1] = n > 1 ? v[1] : v[0];
  t[2] = n > 2 ? v[2] : v[0];
  t[3] = n > 3 ? v[3] : 100.0;
  if (percent)
    for (double &x : t) x *= (65535.0 / 100.0);
  return MB200_OK;
}

int threshold_dev(float *buf, size_t width, size_t height, int channels, int op, const double *t, void *stream) {
  cudaStream_t s;
  const int rc = prepare_dev(buf && valid_image(width, height, channels), "threshold", stream, &s);
  if (rc) return rc;
  return launch_threshold(buf, width * height, channels, op, t, s);
}

// What Black/WhiteThresholdImage decline on the GPU path, then the thresholds.
int black_white_thresholds(int channels, int colorspace, const char *thresholds, double (&t)[4]) {
  if (channels < 3)
    return fail(MB200_EUNSUPPORTED, "Black/WhiteThresholdImage promote gray images to sRGB (threshold.c:949)");
  if (colorspace == MB200_RGBColorspace)
    return fail(MB200_EUNSUPPORTED, "linear RGB: the intensity needs EncodePixelGamma (pixel.c:2421)");
  return parse_thresholds(thresholds, t);
}

int black_white_dev(float *buf, size_t width, size_t height, int channels, int colorspace, const char *thresholds, int op,
                    void *stream) {
  if (!buf || !valid_image(width, height, channels)) return fail(MB200_EINVAL, "threshold: bad arguments");
  double t[4];
  const int rc = black_white_thresholds(channels, colorspace, thresholds, t);
  if (rc) return rc;
  return threshold_dev(buf, width, height, channels, op, t, stream);
}

int black_white_host(const char *name, float *buf, size_t w, size_t h, int ch, int colorspace, const char *thresholds,
                     int op) {
  double t[4];
  if (buf && valid_image(w, h, ch)) {          // reports the decline before staging
    const int rc = black_white_thresholds(ch, colorspace, thresholds, t);
    if (rc) return rc;
  }
  return in_place_host(name, buf, w, h, ch, [&](float *d, cudaStream_t st) {
    return black_white_dev(d, w, h, ch, colorspace, thresholds, op, st);
  });
}

}  // namespace

extern "C" {

int mb200_bilevel_image_dev(float *buf, size_t width, size_t height, int channels, double threshold, void *stream) {
  const double t[4] = {threshold, 0, 0, 0};
  return threshold_dev(buf, width, height, channels, 0, t, stream);
}
int mb200_black_threshold_image_dev(float *buf, size_t width, size_t height, int channels, int colorspace,
                                    const char *thresholds, void *stream) {
  return black_white_dev(buf, width, height, channels, colorspace, thresholds, 1, stream);
}
int mb200_white_threshold_image_dev(float *buf, size_t width, size_t height, int channels, int colorspace,
                                    const char *thresholds, void *stream) {
  return black_white_dev(buf, width, height, channels, colorspace, thresholds, 2, stream);
}
int mb200_clamp_image_dev(float *buf, size_t width, size_t height, int channels, void *stream) {
  return threshold_dev(buf, width, height, channels, 3, nullptr, stream);
}

int mb200_bilevel_image(float *buf, size_t w, size_t h, int ch, double threshold) {
  return in_place_host("bilevel", buf, w, h, ch,
                       [&](float *d, cudaStream_t st) { return mb200_bilevel_image_dev(d, w, h, ch, threshold, st); });
}
int mb200_black_threshold_image(float *buf, size_t w, size_t h, int ch, int colorspace, const char *thresholds) {
  return black_white_host("black threshold", buf, w, h, ch, colorspace, thresholds, 1);
}
int mb200_white_threshold_image(float *buf, size_t w, size_t h, int ch, int colorspace, const char *thresholds) {
  return black_white_host("white threshold", buf, w, h, ch, colorspace, thresholds, 2);
}
int mb200_clamp_image(float *buf, size_t w, size_t h, int ch) {
  return in_place_host("clamp", buf, w, h, ch,
                       [&](float *d, cudaStream_t st) { return mb200_clamp_image_dev(d, w, h, ch, st); });
}

}  // extern "C"

// ---- AdaptiveThresholdImage (threshold.cu), AutoThresholdImage, RangeThresholdImage, PerceptibleImage -----------------
namespace {

unsigned update_bits(int channels, unsigned update_mask) { return update_mask & ((1u << channels) - 1u); }

int check_adaptive_window(size_t window_width, size_t window_height) {
  if (window_width > MB200_ADAPTIVE_THRESHOLD_MAX_WINDOW || window_height > MB200_ADAPTIVE_THRESHOLD_MAX_WINDOW)
    return fail(MB200_EUNSUPPORTED, "adaptive threshold: window %zux%zu is larger than %d", window_width, window_height,
                MB200_ADAPTIVE_THRESHOLD_MAX_WINDOW);
  return MB200_OK;
}

// AutoThresholdImage counts 32-bit histogram bins (checked before anything is staged)
int check_auto_threshold(size_t w, size_t h, int method, const double *threshold_percent) {
  if (!threshold_percent || method < MB200_UndefinedThresholdMethod || method > MB200_TriangleThresholdMethod)
    return fail(MB200_EINVAL, "auto threshold: bad arguments");
  if (w != 0 && h > (((static_cast<size_t>(1) << 32) - 1) / w))
    return fail(MB200_EUNSUPPORTED, "auto threshold: images of 2^32 pixels or more are not supported");
  return MB200_OK;
}

// PerceptibleReciprocal (gem-private.h)
double perceptible_reciprocal(double x) {
  const double sign = x < 0.0 ? -1.0 : 1.0;
  return (sign * x) >= 1.0e-12 ? 1.0 / x : sign / 1.0e-12;
}

int check_range_threshold(int channels) {
  if (channels < 3) return fail(MB200_EUNSUPPORTED, "range threshold: gray images are transformed to sRGB first (threshold.c:2407)");
  return MB200_OK;
}

}  // namespace

extern "C" {

int mb200_adaptive_threshold_image_dev(const float *src, float *dst, size_t width, size_t height, int channels,
                                       size_t window_width, size_t window_height, double bias, unsigned update_mask,
                                       void *stream) {
  cudaStream_t s;
  int rc = prepare_dev(src && dst && valid_image(width, height, channels), "adaptive threshold", stream, &s);
  if (!rc) rc = check_adaptive_window(window_width, window_height);
  if (rc) return rc;
  if (window_width == 0 || window_height == 0) return clone_image(src, dst, width, height, channels, "adaptive threshold copy", s);
  return launch_adaptive_threshold(src, dst, width, height, channels, window_width, window_height, bias,
                                   update_bits(channels, update_mask), s);
}

int mb200_auto_threshold_image_dev(float *buf, size_t width, size_t height, int channels, int method,
                                   double *threshold_percent, void *stream) {
  cudaStream_t s;
  int rc = prepare_dev(buf && valid_image(width, height, channels), "auto threshold", stream, &s);
  if (!rc) rc = check_auto_threshold(width, height, method, threshold_percent);
  if (rc) return rc;
  unsigned counts[256];
  rc = auto_threshold_histogram(buf, width * height, channels, counts, s);
  if (rc) return rc;
  const double threshold = auto_threshold_percent(counts, method);
  const double t[4] = {65535.0 * threshold / 100.0, 0, 0, 0};         // BilevelImage(QuantumRange*threshold/100)
  rc = launch_threshold(buf, width * height, channels, 0, t, s);
  if (!rc) *threshold_percent = threshold;
  return rc;
}

int mb200_range_threshold_image_dev(float *buf, size_t width, size_t height, int channels, double low_black,
                                    double low_white, double high_white, double high_black, int per_channel,
                                    unsigned update_mask, void *stream) {
  cudaStream_t s;
  int rc = prepare_dev(buf && valid_image(width, height, channels), "range threshold", stream, &s);
  if (!rc) rc = check_range_threshold(channels);
  if (rc) return rc;
  const double t[6] = {low_black, low_white, high_white, high_black,
                       65535.0 * perceptible_reciprocal(low_white - low_black),
                       65535.0 * perceptible_reciprocal(high_black - high_white)};
  return launch_threshold(buf, width * height, channels, 4, t, s, update_bits(channels, update_mask), per_channel != 0);
}

int mb200_perceptible_image_dev(float *buf, size_t width, size_t height, int channels, double epsilon,
                                unsigned update_mask, void *stream) {
  cudaStream_t s;
  const int rc = prepare_dev(buf && valid_image(width, height, channels), "perceptible", stream, &s);
  if (rc) return rc;
  const double t[4] = {epsilon, 0, 0, 0};
  return launch_threshold(buf, width * height, channels, 5, t, s, update_bits(channels, update_mask));
}

int mb200_adaptive_threshold_image(const float *src, float *dst, size_t w, size_t h, int ch, size_t window_width,
                                   size_t window_height, double bias, unsigned update_mask) {
  const int rc = check_adaptive_window(window_width, window_height);
  if (rc) return rc;
  return with_staging("adaptive threshold", src, w, h, ch, dst, w, h, [&](const float *s, float *d, cudaStream_t st) {
    return mb200_adaptive_threshold_image_dev(s, d, w, h, ch, window_width, window_height, bias, update_mask, st);
  });
}

int mb200_auto_threshold_image(float *buf, size_t w, size_t h, int ch, int method, double *threshold_percent) {
  const int rc = check_auto_threshold(w, h, method, threshold_percent);
  if (rc) return rc;
  return in_place_host("auto threshold", buf, w, h, ch, [&](float *d, cudaStream_t st) {
    return mb200_auto_threshold_image_dev(d, w, h, ch, method, threshold_percent, st);
  });
}

int mb200_range_threshold_image(float *buf, size_t w, size_t h, int ch, double low_black, double low_white,
                                double high_white, double high_black, int per_channel, unsigned update_mask) {
  const int rc = check_range_threshold(ch);
  if (rc) return rc;
  return in_place_host("range threshold", buf, w, h, ch, [&](float *d, cudaStream_t st) {
    return mb200_range_threshold_image_dev(d, w, h, ch, low_black, low_white, high_white, high_black, per_channel,
                                           update_mask, st);
  });
}

int mb200_perceptible_image(float *buf, size_t w, size_t h, int ch, double epsilon, unsigned update_mask) {
  return in_place_host("perceptible", buf, w, h, ch, [&](float *d, cudaStream_t st) {
    return mb200_perceptible_image_dev(d, w, h, ch, epsilon, update_mask, st);
  });
}

}  // extern "C"

// ---- SharpenImage / EdgeImage: effect.c builds a kernel inline and calls ConvolveImage ------------------------
extern "C" {

int mb200_sharpen_image_dev(const float *src, float *dst, size_t width, size_t height, int channels, double radius,
                            double sigma, void *stream) {
  const KernelList k(mb200_sharpen_kernel(radius, sigma));
  if (!k) return fail(MB200_ENOMEM, "sharpen kernel");
  return mb200_convolve_image_dev(src, dst, width, height, channels, k.get(), stream);
}

int mb200_edge_image_dev(const float *src, float *dst, size_t width, size_t height, int channels, double radius,
                         void *stream) {
  const KernelList k(mb200_edge_kernel(radius));
  if (!k) return fail(MB200_ENOMEM, "edge kernel");
  return mb200_convolve_image_dev(src, dst, width, height, channels, k.get(), stream);
}

int mb200_sharpen_image(const float *src, float *dst, size_t w, size_t h, int ch, double radius, double sigma) {
  return with_staging("sharpen", src, w, h, ch, dst, w, h, [&](const float *s, float *d, cudaStream_t st) {
    return mb200_sharpen_image_dev(s, d, w, h, ch, radius, sigma, st);
  });
}

int mb200_edge_image(const float *src, float *dst, size_t w, size_t h, int ch, double radius) {
  return with_staging("edge", src, w, h, ch, dst, w, h, [&](const float *s, float *d, cudaStream_t st) {
    return mb200_edge_image_dev(s, d, w, h, ch, radius, st);
  });
}

}  // extern "C"

// ---- Copy-trait channels of a `-channel` selection ------------------------------------------------------------------------
extern "C" {

int mb200_restore_channels_dev(float *dst, const float *src, size_t width, size_t height, int channels, unsigned update_mask,
                               void *stream) {
  cudaStream_t s;
  const int rc = prepare_dev(dst && src && valid_image(width, height, channels), "restore channels", stream, &s);
  if (rc) return rc;
  if ((update_mask & ((1u << channels) - 1u)) == ((1u << channels) - 1u)) return MB200_OK;      // nothing to restore
  return launch_restore_channels(dst, src, width * height, channels, update_mask, s);
}

int mb200_resize_copy_channels_dev(const float *src, size_t width, size_t height, int channels, float *dst, size_t out_width,
                                   size_t out_height, int filter, unsigned update_mask, void *stream) {
  cudaStream_t s;
  int rc = prepare_dev(dst && src && valid_image(width, height, channels) && out_width != 0 && out_height != 0,
                       "resize copy channels", stream, &s);
  if (rc) return rc;
  if ((update_mask & ((1u << channels) - 1u)) == ((1u << channels) - 1u)) return MB200_OK;
  const ResizeChoice c = resize_choice(width, height, out_width, out_height, channels, filter);
  std::vector<long> nx(out_width), ny(out_height);
  rc = mb200_resize_nearest(c.filter, width, out_width, c.x_factor, nx.data());
  if (!rc) rc = mb200_resize_nearest(c.filter, height, out_height, c.y_factor, ny.data());
  if (rc) return rc;
  std::vector<int> table(out_width + out_height);
  for (size_t i = 0; i < out_width; ++i) table[i] = static_cast<int>(nx[i]);
  for (size_t i = 0; i < out_height; ++i) table[out_width + i] = static_cast<int>(ny[i]);
  StreamAlloc d_table(s);
  rc = d_table.alloc(table.size() * sizeof(int));
  if (rc) return rc;
  cudaError_t e = cudaMemcpyAsync(d_table.ptr, table.data(), table.size() * sizeof(int), cudaMemcpyHostToDevice, s);
  if (e != cudaSuccess) return cuda_fail(e, "resize copy channels: table upload");
  const int *d = static_cast<const int *>(d_table.ptr);
  return launch_resize_copy_channels(dst, src, width, out_width, out_height, channels, d, d + out_width, update_mask, s);
}

// host buffers: dst already holds the operator's result (resident when attached), src is the operator's source
int mb200_restore_channels(float *dst, const float *src, size_t w, size_t h, int ch, unsigned update_mask) {
  return update_host("restore channels", dst, w, h, src, w, h, ch, [&](float *d, const float *s, cudaStream_t st) {
    return mb200_restore_channels_dev(d, s, w, h, ch, update_mask, st);
  });
}

int mb200_resize_copy_channels(const float *src, size_t w, size_t h, int ch, float *dst, size_t ow, size_t oh, int filter,
                               unsigned update_mask) {
  return update_host("resize copy channels", dst, ow, oh, src, w, h, ch, [&](float *d, const float *s, cudaStream_t st) {
    return mb200_resize_copy_channels_dev(s, w, h, ch, d, ow, oh, filter, update_mask, st);
  });
}

}  // extern "C"

// ---- EqualizeImage (enhance.c:2040) and EmbossImage (effect.c:1600: inline kernel + ConvolveImage + EqualizeImage) -----------
extern "C" {

int mb200_equalize_image_dev(float *buf, size_t width, size_t height, int channels, int sync_channels, void *stream) {
  cudaStream_t s;
  const int rc = prepare_dev(buf && valid_image(width, height, channels), "equalize", stream, &s);
  if (rc) return rc;
  return launch_equalize(buf, width * height, channels, sync_channels, s);
}

int mb200_emboss_image_dev(const float *src, float *dst, size_t width, size_t height, int channels, double radius,
                           double sigma, void *stream) {
  const KernelList k(mb200_emboss_kernel(radius, sigma));
  if (!k) return fail(MB200_ENOMEM, "emboss kernel");
  const int rc = mb200_convolve_image_dev(src, dst, width, height, channels, k.get(), stream);
  if (rc) return rc;
  return mb200_equalize_image_dev(dst, width, height, channels, 1, stream);      // effect.c:1679, default channel mask
}

int mb200_equalize_image(float *buf, size_t w, size_t h, int ch, int sync_channels) {
  return in_place_host("equalize", buf, w, h, ch,
                       [&](float *d, cudaStream_t st) { return mb200_equalize_image_dev(d, w, h, ch, sync_channels, st); });
}

int mb200_emboss_image(const float *src, float *dst, size_t w, size_t h, int ch, double radius, double sigma) {
  return with_staging("emboss", src, w, h, ch, dst, w, h, [&](const float *s, float *d, cudaStream_t st) {
    return mb200_emboss_image_dev(s, d, w, h, ch, radius, sigma, st);
  });
}

}  // extern "C"

// ---- StatisticImage (statistic.c:2918), RotationalBlurImage (effect.c:3129), BilateralBlurImage (effect.c:821) ----------
extern "C" {

int mb200_statistic_image_dev(const float *src, float *dst, size_t width, size_t height, int channels, int type,
                              size_t window_width, size_t window_height, void *stream) {
  cudaStream_t s;
  const int rc = prepare_dev(src && dst && src != dst && valid_image(width, height, channels), "statistic", stream, &s);
  if (rc) return rc;
  return launch_statistic(src, dst, width, height, channels, type, window_width, window_height, s);
}

int mb200_rotational_blur_image_dev(const float *src, float *dst, size_t width, size_t height, int channels, double angle,
                                    void *stream) {
  cudaStream_t s;
  const int rc = prepare_dev(src && dst && src != dst && valid_image(width, height, channels), "rotational blur", stream,
                             &s);
  if (rc) return rc;
  return launch_rotational_blur(src, dst, width, height, channels, angle, s);
}

int mb200_bilateral_blur_image_dev(const float *src, float *dst, size_t width, size_t height, int channels,
                                   size_t window_width, size_t window_height, double intensity_sigma, double spatial_sigma,
                                   void *stream) {
  cudaStream_t s;
  const int rc = prepare_dev(src && dst && src != dst && valid_image(width, height, channels), "bilateral blur", stream,
                             &s);
  if (rc) return rc;
  return launch_bilateral_blur(src, dst, width, height, channels, window_width, window_height, intensity_sigma, spatial_sigma, s);
}

int mb200_adaptive_blur_image_dev(const float *src, float *dst, size_t width, size_t height, int channels, double radius,
                                  double sigma, void *stream) {
  cudaStream_t s;
  const int rc = prepare_dev(src && dst && src != dst && valid_image(width, height, channels), "adaptive blur", stream,
                             &s);
  if (rc) return rc;
  return launch_adaptive(src, dst, width, height, channels, radius, sigma, 0, s);
}

int mb200_adaptive_sharpen_image_dev(const float *src, float *dst, size_t width, size_t height, int channels, double radius,
                                     double sigma, void *stream) {
  cudaStream_t s;
  const int rc = prepare_dev(src && dst && src != dst && valid_image(width, height, channels), "adaptive sharpen", stream,
                             &s);
  if (rc) return rc;
  return launch_adaptive(src, dst, width, height, channels, radius, sigma, 1, s);
}

int mb200_adaptive_blur_image(const float *src, float *dst, size_t w, size_t h, int ch, double radius, double sigma) {
  return with_staging("adaptive blur", src, w, h, ch, dst, w, h, [&](const float *s, float *d, cudaStream_t st) {
    return mb200_adaptive_blur_image_dev(s, d, w, h, ch, radius, sigma, st);
  });
}

int mb200_adaptive_sharpen_image(const float *src, float *dst, size_t w, size_t h, int ch, double radius, double sigma) {
  return with_staging("adaptive sharpen", src, w, h, ch, dst, w, h, [&](const float *s, float *d, cudaStream_t st) {
    return mb200_adaptive_sharpen_image_dev(s, d, w, h, ch, radius, sigma, st);
  });
}

int mb200_selective_blur_image_dev(const float *src, float *dst, size_t width, size_t height, int channels, double radius,
                                   double sigma, double threshold, void *stream) {
  cudaStream_t s;
  const int rc = prepare_dev(src && dst && src != dst && valid_image(width, height, channels), "selective blur", stream,
                             &s);
  if (rc) return rc;
  return launch_selective_blur(src, dst, width, height, channels, radius, sigma, threshold, s);
}

int mb200_selective_blur_image(const float *src, float *dst, size_t w, size_t h, int ch, double radius, double sigma,
                               double threshold) {
  return with_staging("selective blur", src, w, h, ch, dst, w, h, [&](const float *s, float *d, cudaStream_t st) {
    return mb200_selective_blur_image_dev(s, d, w, h, ch, radius, sigma, threshold, st);
  });
}

int mb200_statistic_image(const float *src, float *dst, size_t w, size_t h, int ch, int type, size_t ww, size_t wh) {
  return with_staging("statistic", src, w, h, ch, dst, w, h, [&](const float *s, float *d, cudaStream_t st) {
    return mb200_statistic_image_dev(s, d, w, h, ch, type, ww, wh, st);
  });
}

int mb200_rotational_blur_image(const float *src, float *dst, size_t w, size_t h, int ch, double angle) {
  return with_staging("rotational blur", src, w, h, ch, dst, w, h, [&](const float *s, float *d, cudaStream_t st) {
    return mb200_rotational_blur_image_dev(s, d, w, h, ch, angle, st);
  });
}

int mb200_bilateral_blur_image(const float *src, float *dst, size_t w, size_t h, int ch, size_t ww, size_t wh,
                               double intensity_sigma, double spatial_sigma) {
  return with_staging("bilateral blur", src, w, h, ch, dst, w, h, [&](const float *s, float *d, cudaStream_t st) {
    return mb200_bilateral_blur_image_dev(s, d, w, h, ch, ww, wh, intensity_sigma, spatial_sigma, st);
  });
}

}  // extern "C"

// ---- DespeckleImage (effect.c:1308), LocalContrastImage (effect.c:2013), WaveletDenoiseImage (visual-effects.c:3515) -------
extern "C" {

int mb200_despeckle_image_dev(const float *src, float *dst, size_t width, size_t height, int channels, void *stream) {
  cudaStream_t s;
  int rc = prepare_dev(src && dst && src != dst && valid_image(width, height, channels), "despeckle", stream, &s);
  if (rc) return rc;
  StreamAlloc tmp(s);
  rc = tmp.alloc(image_bytes(width, height, channels));
  if (rc) return rc;
  return launch_despeckle(src, dst, static_cast<float *>(tmp.ptr), width, height, channels, s);
}

int mb200_local_contrast_image_dev(const float *src, float *dst, size_t width, size_t height, int channels, double radius,
                                   double strength, void *stream) {
  cudaStream_t s;
  int rc = prepare_dev(src && dst && src != dst && valid_image(width, height, channels), "local contrast", stream, &s);
  if (!rc) rc = local_contrast_supported(width, height, radius);
  if (rc) return rc;
  StreamAlloc planes(s);
  rc = planes.alloc(2 * image_bytes(width, height, 1));
  if (rc) return rc;
  float *luma = static_cast<float *>(planes.ptr);
  return launch_local_contrast(src, dst, luma, luma + width * height, width, height, channels, radius, strength, s);
}

int mb200_wavelet_denoise_image_dev(const float *src, float *dst, size_t width, size_t height, int channels,
                                    double threshold, double softness, void *stream) {
  cudaStream_t s;
  int rc = prepare_dev(src && dst && src != dst && valid_image(width, height, channels), "wavelet denoise", stream, &s);
  if (!rc) rc = wavelet_denoise_supported(width, height);
  if (rc) return rc;
  StreamAlloc planes(s);
  rc = planes.alloc(3 * image_bytes(width, height, channels >= 3 ? 3 : 1));
  if (rc) return rc;
  return launch_wavelet_denoise(src, dst, static_cast<float *>(planes.ptr), width, height, channels, threshold, softness, s);
}

int mb200_despeckle_image(const float *src, float *dst, size_t w, size_t h, int ch) {
  return with_staging("despeckle", src, w, h, ch, dst, w, h, [&](const float *s, float *d, cudaStream_t st) {
    return mb200_despeckle_image_dev(s, d, w, h, ch, st);
  });
}

int mb200_local_contrast_image(const float *src, float *dst, size_t w, size_t h, int ch, double radius, double strength) {
  if (valid_image(w, h, ch) && local_contrast_supported(w, h, radius) != MB200_OK) return MB200_EUNSUPPORTED;  // no staging
  return with_staging("local contrast", src, w, h, ch, dst, w, h, [&](const float *s, float *d, cudaStream_t st) {
    return mb200_local_contrast_image_dev(s, d, w, h, ch, radius, strength, st);
  });
}

int mb200_wavelet_denoise_image(const float *src, float *dst, size_t w, size_t h, int ch, double threshold,
                                double softness) {
  if (valid_image(w, h, ch) && wavelet_denoise_supported(w, h) != MB200_OK) return MB200_EUNSUPPORTED;           // no staging
  return with_staging("wavelet denoise", src, w, h, ch, dst, w, h, [&](const float *s, float *d, cudaStream_t st) {
    return mb200_wavelet_denoise_image_dev(s, d, w, h, ch, threshold, softness, st);
  });
}

}  // extern "C"

// ---- ScaleImage (resize.c:4106) ---------------------------------------------------------------------------------------------
extern "C" {

int mb200_scale_image_dev(const float *src, size_t width, size_t height, int channels, float *dst, size_t out_width,
                          size_t out_height, void *stream) {
  cudaStream_t s;
  int rc = prepare_dev(src && dst && valid_image(width, height, channels), "scale", stream, &s, out_width,
                       out_height);                                                                // :4153
  if (rc) return rc;
  if (out_width == width && out_height == height)                                                 // :4155
    return clone_image(src, dst, width, height, channels, "scale: clone", s);
  // contribution lists of both axes (host, the reference's state machines), packed into one upload:
  // [xoff (ow+1) | yoff (oh+1) | xidx | yidx] ints, then [xwt | ywt] doubles
  std::vector<long> xoff(out_width + 1), yoff(out_height + 1);
  const long nx = mb200_scale_contributions(0, width, out_width, xoff.data(), nullptr, nullptr, 0);
  const long ny = mb200_scale_contributions(1, height, out_height, yoff.data(), nullptr, nullptr, 0);
  if (nx < 0 || ny < 0) return static_cast<int>(nx < 0 ? nx : ny);
  std::vector<int> ints(out_width + 1 + out_height + 1 + static_cast<size_t>(nx + ny));
  std::vector<double> wts(static_cast<size_t>(nx + ny));
  int *xo = ints.data(), *yo = xo + out_width + 1, *xi = yo + out_height + 1, *yi = xi + nx;
  if (mb200_scale_contributions(0, width, out_width, xoff.data(), xi, wts.data(), static_cast<size_t>(nx)) < 0 ||
      mb200_scale_contributions(1, height, out_height, yoff.data(), yi, wts.data() + nx, static_cast<size_t>(ny)) < 0)
    return MB200_EINVAL;
  for (size_t i = 0; i <= out_width; ++i) xo[i] = static_cast<int>(xoff[i]);
  for (size_t i = 0; i <= out_height; ++i) yo[i] = static_cast<int>(yoff[i]);
  StreamAlloc d_ints(s), d_wts(s);
  rc = d_ints.alloc(ints.size() * sizeof(int));
  if (!rc) rc = d_wts.alloc(wts.size() * sizeof(double));
  if (rc) return rc;
  cudaError_t e = cudaMemcpyAsync(d_ints.ptr, ints.data(), ints.size() * sizeof(int), cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(d_wts.ptr, wts.data(), wts.size() * sizeof(double), cudaMemcpyHostToDevice, s);
  if (e != cudaSuccess) return cuda_fail(e, "scale: table upload");
  const int *di = static_cast<const int *>(d_ints.ptr);
  const double *dw = static_cast<const double *>(d_wts.ptr);
  return launch_scale(src, width, height, channels, dst, out_width, out_height, di, di + out_width + 1 + out_height + 1, dw,
                      di + out_width + 1, di + out_width + 1 + out_height + 1 + nx, dw + nx, s);
}


int mb200_scale_image(const float *src, size_t w, size_t h, int ch, float *dst, size_t ow, size_t oh) {
  return with_staging("scale", src, w, h, ch, dst, ow, oh,
                      [&](const float *s, float *d, cudaStream_t st) { return mb200_scale_image_dev(s, w, h, ch, d, ow, oh, st); });
}

}  // extern "C"

// ---- SampleImage (resize.c:3907) --------------------------------------------------------------------------------
extern "C" {

int mb200_sample_image_dev(const float *src, size_t width, size_t height, int channels, float *dst, size_t out_width,
                           size_t out_height, void *stream) {
  cudaStream_t s;
  const int rc = prepare_dev(src && dst && valid_image(width, height, channels), "sample", stream, &s, out_width,
                             out_height);                                                          // :3946
  if (rc) return rc;
  if (out_width == width && out_height == height)                                                 // :3948
    return clone_image(src, dst, width, height, channels, "sample: clone", s);
  return launch_sample(src, width, height, channels, dst, out_width, out_height, s);
}

int mb200_sample_image(const float *src, size_t w, size_t h, int ch, float *dst, size_t ow, size_t oh) {
  return with_staging("sample", src, w, h, ch, dst, ow, oh, [&](const float *s, float *d, cudaStream_t st) {
    return mb200_sample_image_dev(s, w, h, ch, d, ow, oh, st);
  });
}

}  // extern "C"

// ---- ThumbnailImage (resize.c:4591-4650), pixel path: SampleImage to 4x the target when both integer reduction
// factors exceed 4, ResizeImage(Box) to 2x when they exceed 2, then ResizeImage(filter; the reference passes
// image->filter, LanczosSharp when undefined).  The metadata the reference attaches afterwards (profile stripping,
// Thumb::* properties) is control plane and stays with the caller.
extern "C" {

int mb200_thumbnail_image_dev(const float *src, size_t width, size_t height, int channels, float *dst, size_t columns,
                              size_t rows, int filter, void *stream) {
  cudaStream_t s;
  int rc = prepare_dev(src && dst && valid_image(width, height, channels), "thumbnail", stream, &s, columns, rows);
  if (rc) return rc;
  if (columns == width && rows == height) return clone_image(src, dst, width, height, channels, "thumbnail: clone", s);
  const size_t px = static_cast<size_t>(channels) * sizeof(float);
  const long x_factor = static_cast<long>(width) / static_cast<long>(columns);
  const long y_factor = static_cast<long>(height) / static_cast<long>(rows);
  const float *cur = src;
  size_t cw = width, chh = height;
  StreamAlloc a(s), b(s);
  if (x_factor > 4 && y_factor > 4) {
    rc = a.alloc(4 * columns * 4 * rows * px);
    if (rc) return rc;
    rc = mb200_sample_image_dev(cur, cw, chh, channels, static_cast<float *>(a.ptr), 4 * columns, 4 * rows, s);
    if (rc) return rc;
    cur = static_cast<const float *>(a.ptr); cw = 4 * columns; chh = 4 * rows;
  }
  if (x_factor > 2 && y_factor > 2) {
    rc = b.alloc(2 * columns * 2 * rows * px);
    if (rc) return rc;
    rc = mb200_resize_image_dev(cur, cw, chh, channels, static_cast<float *>(b.ptr), 2 * columns, 2 * rows, MB200_BoxFilter, s);
    if (rc) return rc;
    cur = static_cast<const float *>(b.ptr); cw = 2 * columns; chh = 2 * rows;
  }
  return mb200_resize_image_dev(cur, cw, chh, channels, dst, columns, rows,
                                filter == MB200_UndefinedFilter ? MB200_LanczosSharpFilter : filter, s);
}

int mb200_thumbnail_image(const float *src, size_t w, size_t h, int ch, float *dst, size_t columns, size_t rows, int filter) {
  return with_staging("thumbnail", src, w, h, ch, dst, columns, rows, [&](const float *s, float *d, cudaStream_t st) {
    return mb200_thumbnail_image_dev(s, w, h, ch, d, columns, rows, filter, st);
  });
}

}  // extern "C"

// ---- MotionBlurImage (effect.c:2347) ------------------------------------------------------------------------------
extern "C" {

int mb200_motion_blur_image_dev(const float *src, float *dst, size_t width, size_t height, int channels, double radius,
                                double sigma, double angle, void *stream) {
  cudaStream_t s;
  const int rc = prepare_dev(src && dst && src != dst && valid_image(width, height, channels), "motion blur", stream, &s);
  if (rc) return rc;
  double taps[129];
  long ox[129], oy[129];
  const long n = mb200_motion_blur_kernel(radius, sigma, angle, taps, ox, oy, 129);
  if (n < 0) return fail(MB200_EUNSUPPORTED, "motion blur: more than 129 taps");
  return launch_motion_blur(src, dst, width, height, channels, taps, ox, oy, static_cast<int>(n), s);
}

int mb200_motion_blur_image(const float *src, float *dst, size_t w, size_t h, int ch, double radius, double sigma,
                            double angle) {
  return with_staging("motion blur", src, w, h, ch, dst, w, h, [&](const float *s, float *d, cudaStream_t st) {
    return mb200_motion_blur_image_dev(s, d, w, h, ch, radius, sigma, angle, st);
  });
}

}  // extern "C"

// ---- ContrastImage / ModulateImage / GrayscaleImage / FunctionImage (enhance.c, statistic.c), in place ----------------
namespace {
int check_modulate(int illuminant) {
  if (illuminant < MB200_AIlluminant || illuminant > MB200_F11Illuminant)
    return fail(MB200_EINVAL, "modulate: illuminant %d is not an IlluminantType", illuminant);
  return MB200_OK;
}
int check_grayscale(int method) {
  if (method < MB200_UndefinedPixelIntensityMethod || method > MB200_RMSPixelIntensityMethod)
    return fail(MB200_EINVAL, "grayscale: method %d is not a PixelIntensityMethod", method);
  return MB200_OK;
}
int check_function(int function, size_t n, const double *params) {
  if (function < MB200_UndefinedFunction || function > MB200_SinusoidFunction)
    return fail(MB200_EINVAL, "function: %d is not a MagickFunction", function);
  if (n > 0 && params == nullptr) return fail(MB200_EINVAL, "function: parameters == NULL");
  if (n > MB200_MAX_FUNCTION_PARAMETERS)
    return fail(MB200_EUNSUPPORTED, "function: %zu parameters (at most %d)", n, MB200_MAX_FUNCTION_PARAMETERS);
  return MB200_OK;
}
}  // namespace

extern "C" {

int mb200_contrast_image_dev(float *buf, size_t width, size_t height, int channels, int sharpen, void *stream) {
  cudaStream_t s;
  const int rc = prepare_dev(buf && valid_image(width, height, channels), "contrast", stream, &s);
  if (rc) return rc;
  return launch_contrast(buf, width * height, channels, sharpen != 0, s);
}

int mb200_modulate_image_dev(float *buf, size_t width, size_t height, int channels, double percent_brightness,
                             double percent_saturation, double percent_hue, int colorspace, int illuminant, void *stream) {
  cudaStream_t s;
  int rc = prepare_dev(buf && valid_image(width, height, channels), "modulate", stream, &s);
  if (!rc) rc = check_modulate(illuminant);
  if (rc) return rc;
  return launch_modulate(buf, width * height, channels, percent_brightness, percent_saturation, percent_hue, colorspace,
                         illuminant, s);
}

int mb200_grayscale_image_dev(float *buf, size_t width, size_t height, int channels, int method, int image_colorspace,
                              void *stream) {
  cudaStream_t s;
  int rc = prepare_dev(buf && valid_image(width, height, channels), "grayscale", stream, &s);
  if (!rc) rc = check_grayscale(method);
  if (rc) return rc;
  return launch_grayscale(buf, width * height, channels, method, image_colorspace, s);
}

int mb200_function_image_dev(float *buf, size_t width, size_t height, int channels, int function, size_t number_parameters,
                             const double *parameters, unsigned update_mask, void *stream) {
  cudaStream_t s;
  int rc = prepare_dev(buf && valid_image(width, height, channels), "function", stream, &s);
  if (!rc) rc = check_function(function, number_parameters, parameters);
  if (rc) return rc;
  return launch_function(buf, width * height, channels, function, number_parameters, parameters, update_mask, s);
}

// Host forms: the argument checks run before the buffer is staged, so a refused call moves no data.
int mb200_contrast_image(float *buf, size_t w, size_t h, int ch, int sharpen) {
  return in_place_host("contrast", buf, w, h, ch,
                       [&](float *d, cudaStream_t st) { return mb200_contrast_image_dev(d, w, h, ch, sharpen, st); });
}

int mb200_modulate_image(float *buf, size_t w, size_t h, int ch, double percent_brightness, double percent_saturation,
                         double percent_hue, int colorspace, int illuminant) {
  const int rc = check_modulate(illuminant);
  if (rc) return rc;
  return in_place_host("modulate", buf, w, h, ch, [&](float *d, cudaStream_t st) {
    return mb200_modulate_image_dev(d, w, h, ch, percent_brightness, percent_saturation, percent_hue, colorspace, illuminant,
                                    st);
  });
}

int mb200_grayscale_image(float *buf, size_t w, size_t h, int ch, int method, int image_colorspace) {
  const int rc = check_grayscale(method);
  if (rc) return rc;
  return in_place_host("grayscale", buf, w, h, ch, [&](float *d, cudaStream_t st) {
    return mb200_grayscale_image_dev(d, w, h, ch, method, image_colorspace, st);
  });
}

int mb200_function_image(float *buf, size_t w, size_t h, int ch, int function, size_t number_parameters,
                         const double *parameters, unsigned update_mask) {
  const int rc = check_function(function, number_parameters, parameters);
  if (rc) return rc;
  return in_place_host("function", buf, w, h, ch, [&](float *d, cudaStream_t st) {
    return mb200_function_image_dev(d, w, h, ch, function, number_parameters, parameters, update_mask, st);
  });
}

}  // extern "C"

// ---- level and stretch operators (level.cu) -----------------------------------------------------------------------
namespace {

unsigned channel_bits(int channels, unsigned update_mask) { return update_mask & ((1u << channels) - 1u); }

// The histograms count in 32 bits (checked before anything is staged, so a refused call moves no data).
int check_histogram_pixels(size_t w, size_t h, const char *op) {
  if (w != 0 && h > (((static_cast<size_t>(1) << 32) - 1) / w))
    return fail(MB200_EUNSUPPORTED, "%s: images of 2^32 pixels or more are not supported", op);
  return MB200_OK;
}

}  // namespace

extern "C" {

int mb200_contrast_stretch_image_dev(float *buf, size_t width, size_t height, int channels, double black_point,
                                     double white_point, int per_channel, unsigned update_mask, float *black, float *white,
                                     void *stream) {
  cudaStream_t s;
  int rc = prepare_dev(buf && black && white && valid_image(width, height, channels), "contrast stretch", stream, &s);
  if (!rc) rc = check_histogram_pixels(width, height, "contrast stretch");
  if (rc) return rc;
  return launch_contrast_stretch(buf, width, height, channels, black_point, white_point, per_channel != 0,
                                 channel_bits(channels, update_mask), black, white, s);
}

int mb200_linear_stretch_image_dev(float *buf, size_t width, size_t height, int channels, double black_point,
                                   double white_point, unsigned update_mask, double *black_bin, double *white_bin,
                                   void *stream) {
  cudaStream_t s;
  int rc = prepare_dev(buf && black_bin && white_bin && valid_image(width, height, channels), "linear stretch", stream, &s);
  if (!rc) rc = check_histogram_pixels(width, height, "linear stretch");
  if (rc) return rc;
  return launch_linear_stretch(buf, width, height, channels, black_point, white_point, channel_bits(channels, update_mask),
                               black_bin, white_bin, s);
}

int mb200_level_image_dev(float *buf, size_t width, size_t height, int channels, double black_point, double white_point,
                          double gamma, unsigned update_mask, void *stream) {
  cudaStream_t s;
  const int rc = prepare_dev(buf && valid_image(width, height, channels), "level", stream, &s);
  if (rc) return rc;
  return launch_level(buf, width * height, channels, black_point, white_point, gamma, channel_bits(channels, update_mask),
                      false, s);
}

int mb200_levelize_image_dev(float *buf, size_t width, size_t height, int channels, double black_point, double white_point,
                             double gamma, unsigned update_mask, void *stream) {
  cudaStream_t s;
  const int rc = prepare_dev(buf && valid_image(width, height, channels), "levelize", stream, &s);
  if (rc) return rc;
  return launch_level(buf, width * height, channels, black_point, white_point, gamma, channel_bits(channels, update_mask),
                      true, s);
}

int mb200_minmax_stretch_image_dev(float *buf, size_t width, size_t height, int channels, double black, double white,
                                   double gamma, int per_channel, unsigned update_mask, void *stream) {
  cudaStream_t s;
  const int rc = prepare_dev(buf && valid_image(width, height, channels), "minmax stretch", stream, &s);
  if (rc) return rc;
  return launch_minmax_stretch(buf, width, height, channels, black, white, gamma, per_channel != 0,
                               channel_bits(channels, update_mask), s);
}

int mb200_gamma_image_dev(float *buf, size_t width, size_t height, int channels, double gamma, unsigned update_mask,
                          void *stream) {
  cudaStream_t s;
  const int rc = prepare_dev(buf && valid_image(width, height, channels), "gamma", stream, &s);
  if (rc) return rc;
  return launch_gamma(buf, width * height, channels, gamma, channel_bits(channels, update_mask), s);
}

int mb200_identify_gray_dev(const float *buf, size_t width, size_t height, int channels, int *type, void *stream) {
  cudaStream_t s;
  const int rc = prepare_dev(buf && type && valid_image(width, height, channels), "identify gray", stream, &s);
  if (rc) return rc;
  return launch_identify_gray(buf, width * height, channels, type, s);
}

int mb200_contrast_stretch_image(float *buf, size_t w, size_t h, int ch, double black_point, double white_point,
                                 int per_channel, unsigned update_mask, float *black, float *white) {
  int rc = black && white ? check_histogram_pixels(w, h, "contrast stretch") : fail(MB200_EINVAL, "contrast stretch: bad arguments");
  if (rc) return rc;
  return in_place_host("contrast stretch", buf, w, h, ch, [&](float *d, cudaStream_t st) {
    return mb200_contrast_stretch_image_dev(d, w, h, ch, black_point, white_point, per_channel, update_mask, black, white,
                                            st);
  });
}

int mb200_linear_stretch_image(float *buf, size_t w, size_t h, int ch, double black_point, double white_point,
                               unsigned update_mask, double *black_bin, double *white_bin) {
  int rc = black_bin && white_bin ? check_histogram_pixels(w, h, "linear stretch")
                                  : fail(MB200_EINVAL, "linear stretch: bad arguments");
  if (rc) return rc;
  return in_place_host("linear stretch", buf, w, h, ch, [&](float *d, cudaStream_t st) {
    return mb200_linear_stretch_image_dev(d, w, h, ch, black_point, white_point, update_mask, black_bin, white_bin, st);
  });
}

int mb200_level_image(float *buf, size_t w, size_t h, int ch, double black_point, double white_point, double gamma,
                      unsigned update_mask) {
  return in_place_host("level", buf, w, h, ch, [&](float *d, cudaStream_t st) {
    return mb200_level_image_dev(d, w, h, ch, black_point, white_point, gamma, update_mask, st);
  });
}

int mb200_levelize_image(float *buf, size_t w, size_t h, int ch, double black_point, double white_point, double gamma,
                         unsigned update_mask) {
  return in_place_host("levelize", buf, w, h, ch, [&](float *d, cudaStream_t st) {
    return mb200_levelize_image_dev(d, w, h, ch, black_point, white_point, gamma, update_mask, st);
  });
}

int mb200_minmax_stretch_image(float *buf, size_t w, size_t h, int ch, double black, double white, double gamma,
                               int per_channel, unsigned update_mask) {
  return in_place_host("minmax stretch", buf, w, h, ch, [&](float *d, cudaStream_t st) {
    return mb200_minmax_stretch_image_dev(d, w, h, ch, black, white, gamma, per_channel, update_mask, st);
  });
}

int mb200_gamma_image(float *buf, size_t w, size_t h, int ch, double gamma, unsigned update_mask) {
  return in_place_host("gamma", buf, w, h, ch, [&](float *d, cudaStream_t st) {
    return mb200_gamma_image_dev(d, w, h, ch, gamma, update_mask, st);
  });
}

int mb200_identify_gray(const float *buf, size_t w, size_t h, int ch, int *type) {
  if (!buf || !type || !valid_image(w, h, ch)) return fail(MB200_EINVAL, "identify gray: bad arguments");
  cudaStream_t s;
  int rc = prepare(nullptr, &s);
  if (rc) return rc;
  StageRef in;                                                   // read only: nothing is copied back
  rc = stage_input(buf, image_bytes(w, h, ch), s, &in);
  if (!rc) rc = mb200_identify_gray_dev(static_cast<const float *>(in.dev), w, h, ch, type, s);
  if (rc) cudaStreamSynchronize(s);
  release_stage(&in, s);
  return rc;
}

}  // extern "C"
