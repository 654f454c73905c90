// What rate does FP64 mma.sync reach on sm_90a per shape, and is it a separate pipe from DFMA?
//   shapes: m8n8k4 (DMMA.8x8x4), m16n8k4, m16n8k8, m16n8k16 (DMMA.16x8x4 / 16x8x8 / 16x8x16)
//   mode 0: all warps DFMA;  mode 1: all warps DMMA;  mode 2: even warps DFMA, odd warps DMMA
// One CTA of W warps per SM, W = 8, 12, 16.  Before timing, every shape's fragment layout is checked against a host
// product (the layouts conv_mma.cu relies on).
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o dmma dmma.cu
#include <cmath>
#include <cstdio>
#include <cuda_runtime.h>

// SHAPE 0..3 = m8n8k4, m16n8k4, m16n8k8, m16n8k16.  Per lane: NA A doubles, NB B doubles, NC accumulator doubles.
template <int SHAPE> struct Shape;
template <> struct Shape<0> { static constexpr int NA = 1, NB = 1, NC = 2, M = 8, K = 4; };
template <> struct Shape<1> { static constexpr int NA = 2, NB = 1, NC = 4, M = 16, K = 4; };
template <> struct Shape<2> { static constexpr int NA = 4, NB = 2, NC = 4, M = 16, K = 8; };
template <> struct Shape<3> { static constexpr int NA = 8, NB = 4, NC = 4, M = 16, K = 16; };

template <int SHAPE>
__device__ __forceinline__ void mma(double *d, const double *a, const double *b) {
  if constexpr (SHAPE == 0) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                 : "+d"(d[0]), "+d"(d[1]) : "d"(a[0]), "d"(b[0]));
  } else if constexpr (SHAPE == 1) {
    asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                 : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3]) : "d"(a[0]), "d"(a[1]), "d"(b[0]));
  } else if constexpr (SHAPE == 2) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                 "{%0,%1,%2,%3};"
                 : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
                 : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
  } else {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
                 "{%12,%13,%14,%15}, {%0,%1,%2,%3};"
                 : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
                 : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]),
                   "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
  }
}

// Fragment coordinates (g = lane / 4, t = lane % 4):
//   m8n8k4:  A[g][t], B[t][g], D[g][2t + e]
//   m16n8kK: A element i: row g + 8 (i & 1), column t + 4 (i >> 1); B element i: row t + 4 i, column g;
//            D element i: row g + 8 (i >> 1), column 2t + (i & 1)
template <int SHAPE>
__global__ void layout_check(const double *A, const double *B, double *D) {   // A: M x K row major, B: K x 8
  using S = Shape<SHAPE>;
  const int lane = threadIdx.x, g = lane >> 2, t = lane & 3;
  double a[S::NA], b[S::NB], d[S::NC];
  for (int i = 0; i < S::NA; ++i)
    a[i] = SHAPE == 0 ? A[g * S::K + t] : A[(g + 8 * (i & 1)) * S::K + t + 4 * (i >> 1)];
  for (int i = 0; i < S::NB; ++i) b[i] = B[(t + 4 * i) * 8 + g];
  for (int i = 0; i < S::NC; ++i) d[i] = 0.0;
  mma<SHAPE>(d, a, b);
  for (int i = 0; i < S::NC; ++i) {
    const int row = SHAPE == 0 ? g : g + 8 * (i >> 1), col = 2 * t + (i & 1);
    D[row * 8 + col] = d[i];
  }
}

template <int SHAPE>
bool check_layout() {
  using S = Shape<SHAPE>;
  double hA[256], hB[128], hD[128], want[128];
  for (int i = 0; i < S::M * S::K; ++i) hA[i] = (i * 37 % 101) / 16.0 - 3.0;
  for (int i = 0; i < S::K * 8; ++i) hB[i] = (i * 53 % 89) / 8.0 - 5.0;
  for (int m = 0; m < S::M; ++m)
    for (int n = 0; n < 8; ++n) {
      double s = 0;
      for (int k = 0; k < S::K; ++k) s += hA[m * S::K + k] * hB[k * 8 + n];
      want[m * 8 + n] = s;
    }
  double *dA, *dB, *dD;
  cudaMalloc(&dA, sizeof hA); cudaMalloc(&dB, sizeof hB); cudaMalloc(&dD, sizeof hD);
  cudaMemcpy(dA, hA, sizeof hA, cudaMemcpyHostToDevice);
  cudaMemcpy(dB, hB, sizeof hB, cudaMemcpyHostToDevice);
  layout_check<SHAPE><<<1, 32>>>(dA, dB, dD);
  cudaMemcpy(hD, dD, sizeof hD, cudaMemcpyDeviceToHost);
  cudaFree(dA); cudaFree(dB); cudaFree(dD);
  double err = 0;
  for (int i = 0; i < S::M * 8; ++i) err = fmax(err, fabs(hD[i] - want[i]));
  printf("layout m%dn8k%d: max |err| %.3g %s\n", S::M, S::K, err, err < 1e-9 ? "ok" : "MISMATCH");
  return err < 1e-9;
}

template <int SHAPE, int NACC>
__global__ void __launch_bounds__(512) k(double *out, double a0, double b0, int iters, int mode) {
  using S = Shape<SHAPE>;
  const int warp = threadIdx.x >> 5;
  const bool use_mma = mode == 1 || (mode == 2 && (warp & 1));
  constexpr int NREG = NACC * S::NC;                // the DFMA warps keep as many accumulators
  double acc[NREG];
#pragma unroll
  for (int i = 0; i < NREG; ++i) acc[i] = threadIdx.x + i;
  if (use_mma) {
    double a[S::NA], b[S::NB];
#pragma unroll
    for (int i = 0; i < S::NA; ++i) a[i] = a0 + i;
#pragma unroll
    for (int i = 0; i < S::NB; ++i) b[i] = b0 + i;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
      for (int i = 0; i < NACC; ++i) mma<SHAPE>(acc + i * S::NC, a, b);
    }
  } else {
    for (int it = 0; it < iters; ++it) {
#pragma unroll
      for (int i = 0; i < NREG; ++i) acc[i] = fma(acc[i], a0, b0);
    }
  }
  double s = 0;
  for (int i = 0; i < NREG; ++i) s += acc[i];
  if (s == 123.456) out[0] = s;
}

template <typename F> float timeit(F f) {
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  f(); cudaDeviceSynchronize();
  cudaEventRecord(a); f(); cudaEventRecord(b); cudaEventSynchronize(b);
  float ms; cudaEventElapsedTime(&ms, a, b); return ms;
}

template <int SHAPE>
void run_shape(double *buf, int sms, int clock_khz) {
  using S = Shape<SHAPE>;
  constexpr int NACC = 8;
  const int iters = 8192 * 64 / (S::M * S::K);      // the same FMAs per shape
  for (int warps : {8, 12, 16}) {
    for (int mode = 0; mode < 3; ++mode) {
      float ms = timeit([&] { k<SHAPE, NACC><<<sms, warps * 32>>>(buf, 1.0000001, 1e-9, iters, mode); });
      const cudaError_t e = cudaGetLastError();
      if (e != cudaSuccess) { printf("launch failed: %s\n", cudaGetErrorString(e)); return; }
      const double wtot = (double) sms * warps * iters;
      const double dfma_w = 32.0 * NACC * S::NC, dmma_w = NACC * S::M * 8.0 * S::K;     // FMAs per warp-iteration
      double fma_dfma = 0, fma_dmma = 0;
      if (mode == 0) fma_dfma = wtot * dfma_w;
      if (mode == 1) fma_dmma = wtot * dmma_w;
      if (mode == 2) { fma_dfma = wtot / 2 * dfma_w; fma_dmma = wtot / 2 * dmma_w; }
      // cycles per DMMA per scheduler (4 per SM) at the maximum SM clock
      const double n_dmma = mode == 0 ? 0 : wtot * NACC * (mode == 2 ? 0.5 : 1.0);
      const double cyc = n_dmma > 0 ? ms * 1e-3 * clock_khz * 1e3 / (n_dmma / (sms * 4.0)) : 0.0;
      printf("m%dn8k%-2d warps/SM=%2d mode=%d: %8.3f ms  DFMA %6.2f T/s  DMMA %6.2f T FMA/s  total %6.2f T FMA/s"
             "  %5.1f cyc/DMMA/scheduler\n",
             S::M, S::K, warps, mode, ms, fma_dfma / ms * 1e-9, fma_dmma / ms * 1e-9, (fma_dfma + fma_dmma) / ms * 1e-9,
             cyc);
    }
  }
}

int main() {
  cudaDeviceProp p;
  cudaGetDeviceProperties(&p, 0);
  int clock_khz = 0;
  cudaDeviceGetAttribute(&clock_khz, cudaDevAttrClockRate, 0);
  printf("%s, %d SMs, max SM clock %d MHz\n", p.name, p.multiProcessorCount, clock_khz / 1000);
  bool ok = check_layout<0>() & check_layout<1>() & check_layout<2>() & check_layout<3>();
  void *buf; cudaMalloc(&buf, 1024);
  const int sms = p.multiProcessorCount;
  run_shape<0>((double *) buf, sms, clock_khz);
  run_shape<1>((double *) buf, sms, clock_khz);
  run_shape<2>((double *) buf, sms, clock_khz);
  run_shape<3>((double *) buf, sms, clock_khz);
  return ok ? 0 : 1;
}
