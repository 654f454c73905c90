// resize_tables.cpp -- the per-axis tables of ResizeImage (resize.c:3761): planned on the host from the reference's
// contribution lists (resize_filter.cpp), uploaded once and cached per (device, filter, options, in_n, out_n), so that
// batches of equally sized images (BASELINE configs[4]) rebuild neither the weights on the host nor upload them.
#include "mb200_internal.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <memory>
#include <mutex>
#include <vector>

namespace mb200 {

ResizeAxis::~ResizeAxis() {
  int cur = 0;
  cudaGetDevice(&cur);
  if (device >= 0 && cur != device) cudaSetDevice(device);
  cudaFree(d_start); cudaFree(d_count); cudaFree(d_weights); cudaFree(d_wreg); cudaFree(d_wsets); cudaFree(d_border);
  cudaFree(d_tiles_x); cudaFree(d_tiles_y); cudaFree(d_is_border);
  if (device >= 0 && cur != device) cudaSetDevice(cur);
}

namespace {

// Host side of the device buffers of one ResizeAxis (an empty vector leaves its buffer null).
struct AxisPlan {
  std::vector<int> start, count;
  std::vector<double> weights;        // tap-major [taps][out_n], for coalesced weight loads
  std::vector<double> wreg, wsets;
  std::vector<int> border, tiles_x, tiles_y;
  std::vector<unsigned char> is_border;
};

// Turns the contribution lists of one axis (start / count / weights[out_n][taps]) into the tables of every resize
// kernel: the scalars go to *t, the arrays to *p.
void plan_axis(const std::vector<long> &start, const std::vector<int> &count, const std::vector<double> &w, ResizeAxis *t,
               AxisPlan *p) {
  const size_t out_n = t->out_n;
  const long taps = t->taps;
  // widest source span of any aligned block of 32 outputs
  for (size_t o = 0; o < out_n; o += 32) {
    const size_t last = std::min(o + 32, out_n) - 1;
    long hi = 0;
    for (size_t k = o; k <= last; ++k) hi = std::max(hi, start[k] + count[k]);
    t->max_span = std::max(t->max_span, static_cast<int>(hi - start[o]));
  }
  // regular pattern (integer-ratio reduction): constant tap count and window stride in the interior
  if (out_n >= 64) {
    const size_t mid = out_n / 2;
    const int n = count[mid];
    const long st = start[mid + 1] - start[mid];
    size_t regular = 0;
    for (size_t o = 0; o + 1 < out_n; ++o)
      if (count[o] == n && count[o + 1] == n && start[o + 1] - start[o] == st) ++regular;
    if (st >= 2 && n > 0 && regular * 10 >= out_n * 9) {
      t->reg_stride = static_cast<int>(st);
      t->reg_taps = n;
      p->wreg.assign(out_n * static_cast<size_t>(n), 0.0);
      for (size_t o = 0; o < out_n; ++o)
        for (int j = 0; j < n && j < count[o]; ++j) p->wreg[o * n + j] = w[o * taps + j];
      // runs of outputs whose weights are bit-identical (same binade of bisect, resize.c:3398-3443)
      struct Run { size_t lo, len; };
      std::vector<Run> runs;
      size_t lo = 0;
      for (size_t o = 1; o <= out_n; ++o) {
        const bool same = o < out_n && count[o] == n && count[lo] == n && start[o] - start[o - 1] == st &&
                          std::memcmp(&w[o * taps], &w[lo * taps], static_cast<size_t>(n) * sizeof(double)) == 0;
        if (!same) {
          if (count[lo] == n && o - lo >= 8) runs.push_back({lo, o - lo});
          lo = o;
        }
      }
      std::sort(runs.begin(), runs.end(), [](const Run &a, const Run &b) { return a.len > b.len; });
      if (runs.size() > MB200_RESIZE_MAX_SEGMENTS) runs.resize(MB200_RESIZE_MAX_SEGMENTS);
      std::sort(runs.begin(), runs.end(), [](const Run &a, const Run &b) { return a.lo < b.lo; });
      size_t covered = 0;
      for (const Run &r : runs) covered += r.len;
      if (!runs.empty() && covered * 10 >= out_n * 6) {
        long next = 0;
        for (const Run &r : runs) {
          t->seg_o[t->nseg] = static_cast<int>(r.lo);
          t->seg_n[t->nseg] = static_cast<int>(r.len);
          t->seg_src[t->nseg] = static_cast<int>(start[r.lo]);
          ++t->nseg;
          p->wsets.insert(p->wsets.end(), &w[r.lo * taps], &w[r.lo * taps] + n);
          for (long o = next; o < static_cast<long>(r.lo); ++o) p->border.push_back(static_cast<int>(o));
          next = static_cast<long>(r.lo + r.len);
        }
        for (long o = next; o < static_cast<long>(out_n); ++o) p->border.push_back(static_cast<int>(o));
        t->nborder = static_cast<int>(p->border.size());
        if (p->border.empty()) p->border.push_back(0);      // keep the buffer non-null
      }
    }
  }
  if (t->nseg > 0) {
    int tw = 0, th = 0;
    resize_fused_tile(t->reg_stride, t->reg_taps, &tw, &th);
    if (tw > 0) {
      auto cut = [&](int tile, std::vector<int> &out) {
        for (int k = 0; k < t->nseg; ++k)
          for (int rel = 0; rel < t->seg_n[k]; rel += tile) {
            out.push_back(t->seg_o[k] + rel);
            out.push_back(std::min(tile, t->seg_n[k] - rel));
            out.push_back(t->seg_src[k] + t->reg_stride * rel);
            out.push_back(k);
          }
      };
      cut(tw, p->tiles_x);
      cut(th, p->tiles_y);
      t->ntiles_x = static_cast<int>(p->tiles_x.size() / 4);
      t->ntiles_y = static_cast<int>(p->tiles_y.size() / 4);
      p->is_border.assign(out_n, 0);
      for (int k = 0; k < t->nborder; ++k) p->is_border[static_cast<size_t>(p->border[k])] = 1;
    }
  }
  p->start.assign(start.begin(), start.end());
  p->count = count;
  p->weights.resize(w.size());
  for (size_t o = 0; o < out_n; ++o)
    for (long j = 0; j < taps; ++j) p->weights[static_cast<size_t>(j) * out_n + o] = w[o * taps + j];
}

template <typename T>
cudaError_t upload(const std::vector<T> &host, T **dev) {
  if (host.empty()) return cudaSuccess;
  const size_t bytes = host.size() * sizeof(T);
  cudaError_t e = cudaMalloc(dev, bytes);
  if (e == cudaSuccess) e = cudaMemcpy(*dev, host.data(), bytes, cudaMemcpyHostToDevice);
  return e;
}

cudaError_t upload_axis(const AxisPlan &p, ResizeAxis *t) {
  cudaError_t e = upload(p.start, &t->d_start);
  if (e == cudaSuccess) e = upload(p.count, &t->d_count);
  if (e == cudaSuccess) e = upload(p.weights, &t->d_weights);
  if (e == cudaSuccess) e = upload(p.wreg, &t->d_wreg);
  if (e == cudaSuccess) e = upload(p.wsets, &t->d_wsets);
  if (e == cudaSuccess) e = upload(p.border, &t->d_border);
  if (e == cudaSuccess) e = upload(p.tiles_x, &t->d_tiles_x);
  if (e == cudaSuccess) e = upload(p.tiles_y, &t->d_tiles_y);
  if (e == cudaSuccess) e = upload(p.is_border, &t->d_is_border);
  return e;
}

// Bounded LRU of shared entries, most recently used last: a call holds a reference while its launches are being
// queued, eviction drops the cache's reference and the last owner frees the device buffers.
std::mutex g_tables_mutex;
std::vector<std::shared_ptr<const ResizeAxis>> g_tables;
constexpr size_t kMaxCachedTables = 64;

// Call with g_tables_mutex held.
std::shared_ptr<const ResizeAxis> find(int device, int filter, const mb200_filter_options &opt, size_t in_n,
                                       size_t out_n) {
  for (size_t i = 0; i < g_tables.size(); ++i) {
    const std::shared_ptr<const ResizeAxis> t = g_tables[i];
    if (t->device == device && t->filter == filter && t->in_n == in_n && t->out_n == out_n &&
        std::memcmp(&t->options, &opt, sizeof(opt)) == 0) {
      if (i + 1 != g_tables.size()) { g_tables.erase(g_tables.begin() + i); g_tables.push_back(t); }
      return t;
    }
  }
  return nullptr;
}

}  // namespace

int resize_axis_tables(int filter, const mb200_filter_options *options, size_t in_n, size_t out_n, double factor,
                       std::shared_ptr<const ResizeAxis> *out) {
  mb200_filter_options opt{};           // normalised copy: the cache compares the bytes
  if (options) {
    opt.set = options->set;
    if (opt.set & MB200_FO_WINDOW) { opt.window = options->window; opt.keep_filter = options->keep_filter ? 1 : 0; }
    if (opt.set & MB200_FO_LOBES) opt.lobes = options->lobes;
    if (opt.set & MB200_FO_SIGMA) opt.sigma = options->sigma;
    if (opt.set & MB200_FO_KAISER_BETA) opt.kaiser_beta = options->kaiser_beta;
    if (opt.set & MB200_FO_BLUR) opt.blur = options->blur;
    if (opt.set & MB200_FO_SUPPORT) opt.support = options->support;
    if (opt.set & MB200_FO_WIN_SUPPORT) opt.win_support = options->win_support;
    if (opt.set & MB200_FO_B) opt.b = options->b;
    if (opt.set & MB200_FO_C) opt.c = options->c;
  }
  int dev = 0;
  cudaGetDevice(&dev);
  {
    std::lock_guard<std::mutex> lock(g_tables_mutex);
    if ((*out = find(dev, filter, opt, in_n, out_n))) return MB200_OK;
  }
  // built outside the lock
  const long taps = mb200_resize_contributions_ex(filter, &opt, in_n, out_n, factor, nullptr, nullptr, nullptr, 0);
  if (taps < 0) return static_cast<int>(taps);
  std::vector<long> start(out_n);
  std::vector<int> count(out_n);
  std::vector<double> w(out_n * static_cast<size_t>(taps));
  const long r = mb200_resize_contributions_ex(filter, &opt, in_n, out_n, factor, start.data(), count.data(), w.data(),
                                               static_cast<size_t>(taps));
  if (r < 0) return static_cast<int>(r);
  std::shared_ptr<ResizeAxis> t = std::make_shared<ResizeAxis>();
  t->device = dev; t->filter = filter; t->options = opt; t->in_n = in_n; t->out_n = out_n; t->taps = taps;
  AxisPlan plan;
  plan_axis(start, count, w, t.get(), &plan);
  const cudaError_t e = upload_axis(plan, t.get());
  if (e != cudaSuccess) return cuda_fail(e, "resize: table upload");     // ~ResizeAxis frees what was allocated
  std::lock_guard<std::mutex> lock(g_tables_mutex);
  if ((*out = find(dev, filter, opt, in_n, out_n))) return MB200_OK;     // another thread built the same table meanwhile
  if (g_tables.size() >= kMaxCachedTables) g_tables.erase(g_tables.begin());     // least recently used
  g_tables.push_back(t);
  *out = t;
  return MB200_OK;
}

}  // namespace mb200
