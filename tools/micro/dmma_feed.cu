// How fast does FP64 mma.sync run when its operands are fed the way conv_mma.cu feeds them?
//   mode 0: m8n8k4, A and B constant registers (the roof: tools/micro/dmma.cu)
//   mode 1: m8n8k4, B from shared memory (one conflict-free LDS.64 per DMMA), A rotating over 10 registers
//   mode 2: mode 1 + one dependent DFMA chain step per 2 DMMAs (the premultiply / reciprocal work)
//   mode 3: mode 1 + one F2F pair per 4 DMMAs
//   mode 4: m16n8k16, B from shared memory (four conflict-free LDS.64 per DMMA), A held in 3 x 8 registers: the
//           wide-tile pass's 3 k-steps x 4 tiles per 16 outputs (64-row ring per warp, 18 KB)
// Modes 1 and 4 also run at 8 and 12 warps per SM (extra dynamic shared memory limits the CTAs per SM).
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o dmma_feed dmma_feed.cu
#include <cstdio>
#include <cuda_runtime.h>
__device__ __forceinline__ void dmma(double &d0, double &d1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}
__device__ __forceinline__ void dmma16(double (&d)[4], const double *a, const double (&b)[4]) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
               "{%12,%13,%14,%15}, {%0,%1,%2,%3};"
               : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
               : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]),
                 "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
}
template <int MODE>
__global__ void __launch_bounds__(128, 4) k(double *out, const double *in, int iters) {
  __shared__ double ring[4][40 * 36];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double *r = ring[warp];
  for (int i = lane; i < 40 * 36; i += 32) r[i] = in[i & 255];
  __syncwarp();
  double a[10];
  for (int s = 0; s < 10; ++s) a[s] = in[s + lane];
  double acc[4][2] = {};
  double f = in[lane], g = 1.0;
  float h = static_cast<float>(in[lane + 1]);
  const int off = (lane & 3) * 36 + (lane >> 2);
  for (int it = 0; it < iters; ++it) {
    const double *p0 = r + off + (it % 6) * 8 * 36 % (40 * 36);
#pragma unroll
    for (int s = 0; s < 10; ++s) {
      const double *p = p0 + (s * 4 * 36) % (8 * 36);
      double b0, b1, b2, b3;
      if (MODE == 0) { b0 = b1 = b2 = b3 = f; }
      else { b0 = p[0]; b1 = p[16]; b2 = p[8]; b3 = p[24]; }
      const double av = MODE == 0 ? a[0] : a[s];
      dmma(acc[0][0], acc[0][1], av, b0);
      dmma(acc[1][0], acc[1][1], av, b1);
      if (MODE == 2) g = fma(g, 1.0000001, 1e-9);
      dmma(acc[2][0], acc[2][1], av, b2);
      dmma(acc[3][0], acc[3][1], av, b3);
      if (MODE == 2) g = fma(g, 0.9999999, 1e-9);
      if (MODE == 3) { h = static_cast<float>(static_cast<double>(h) ); asm volatile("" : "+f"(h)); }
    }
  }
  double s = g + h;
  for (int t = 0; t < 4; ++t) s += acc[t][0] + acc[t][1];
  if (s == 123.456) out[0] = s;
}
// mode 4: per iteration 16 new ring rows, 3 k-steps x 4 tiles of m16n8k16
__global__ void __launch_bounds__(128, 3) k16(double *out, const double *in, int iters) {
  extern __shared__ double ring16[];
  constexpr int PW = 36, RR = 64;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double *r = ring16 + warp * RR * PW;
  for (int i = lane; i < RR * PW; i += 32) r[i] = in[i & 255];
  __syncwarp();
  double a[3][8];
  for (int s = 0; s < 3; ++s)
    for (int i = 0; i < 8; ++i) a[s][i] = in[8 * s + i + lane];
  double acc[4][4] = {};
  const int off = (lane & 3) * PW + (lane >> 2);
  for (int it = 0; it < iters; ++it) {
    const int rb = (it & 3) * 16;
#pragma unroll
    for (int s = 0; s < 3; ++s) {
      double b[4][4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const double *p = r + off + ((rb + 16 * s + 4 * i) & (RR - 1)) * PW;
        b[0][i] = p[0]; b[1][i] = p[16]; b[2][i] = p[8]; b[3][i] = p[24];
      }
#pragma unroll
      for (int t = 0; t < 4; ++t) dmma16(acc[t], a[s], b[t]);
    }
  }
  double s = 0;
  for (int t = 0; t < 4; ++t) s += acc[t][0] + acc[t][1] + acc[t][2] + acc[t][3];
  if (s == 123.456) out[0] = s;
}
template <typename F> float timeit(F f) {
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  f(); cudaDeviceSynchronize();
  cudaEventRecord(a); f(); cudaEventRecord(b); cudaEventSynchronize(b);
  float ms; cudaEventElapsedTime(&ms, a, b); return ms;
}
int main() {
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, 0);
  int clock_khz = 0;
  cudaDeviceGetAttribute(&clock_khz, cudaDevAttrClockRate, 0);
  const int sms = prop.multiProcessorCount;
  const double ghz = clock_khz * 1e-6;
  printf("%s, %d SMs, max SM clock %d MHz\n", prop.name, sms, clock_khz / 1000);
  double *buf, *in; cudaMalloc(&buf, 1024); cudaMalloc(&in, 4096); cudaMemset(in, 0, 4096);
  const int iters = 4096;
  const size_t pad3 = 70 * 1024 - sizeof(double) * 4 * 40 * 36;    // k<1> at 3 CTAs per SM
  const size_t pad2 = 100 * 1024 - sizeof(double) * 4 * 40 * 36;   // k<1> at 2 CTAs per SM
  cudaFuncSetAttribute(k<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(pad2));
  const int smem16 = 4 * 64 * 36 * 8;                                // 73.7 KB: 3 CTAs per SM
  cudaFuncSetAttribute(k16, cudaFuncAttributeMaxDynamicSharedMemorySize, 110 * 1024);
  for (int mode = 0; mode < 4; ++mode) {
    const int ctas = sms * 4;
    float ms = 0;
    if (mode == 0) ms = timeit([&] { k<0><<<ctas, 128>>>(buf, in, iters); });
    if (mode == 1) ms = timeit([&] { k<1><<<ctas, 128>>>(buf, in, iters); });
    if (mode == 2) ms = timeit([&] { k<2><<<ctas, 128>>>(buf, in, iters); });
    if (mode == 3) ms = timeit([&] { k<3><<<ctas, 128>>>(buf, in, iters); });
    const double dm = (double) ctas * 4 * iters * 40;
    printf("mode %d m8n8k4   16 warps/SM: %.3f ms  %.2f T FMA/s in DMMA  (%.2f cycles per DMMA per scheduler)\n", mode,
           ms, dm * 256 / ms * 1e-9, ms * 1e-3 * ghz * 1e9 / (dm / (sms * 4)));
  }
  for (int per_sm : {2, 3}) {
    const int ctas = sms * per_sm;
    const size_t pad = per_sm == 3 ? pad3 : pad2;
    float ms = timeit([&] { k<1><<<ctas, 128, pad>>>(buf, in, iters); });
    double dm = (double) ctas * 4 * iters * 40;
    printf("mode 1 m8n8k4   %2d warps/SM: %.3f ms  %.2f T FMA/s in DMMA  (%.2f cycles per DMMA per scheduler)\n",
           4 * per_sm, ms, dm * 256 / ms * 1e-9, ms * 1e-3 * ghz * 1e9 / (dm / (sms * 4)));
    const int smem = per_sm == 3 ? smem16 : 100 * 1024;
    const int it16 = iters * 40 / 12 / 8;                 // the same FMAs as mode 1
    ms = timeit([&] { k16<<<ctas, 128, smem>>>(buf, in, it16); });
    dm = (double) ctas * 4 * it16 * 12;
    printf("mode 4 m16n8k16 %2d warps/SM: %.3f ms  %.2f T FMA/s in DMMA  (%.2f cycles per DMMA per scheduler)\n",
           4 * per_sm, ms, dm * 2048 / ms * 1e-9, ms * 1e-3 * ghz * 1e9 / (dm / (sms * 4)));
  }
  const cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) { printf("error: %s\n", cudaGetErrorString(e)); return 1; }
  return 0;
}
