// Microbenchmark: issue rate of FFMA vs FFMA2 (fma.rn.f32x2) per SM sub-partition.
#include <cstdio>
#include <cuda_runtime.h>
template <int MODE>
__global__ void k(float* out, long long* cyc, int iters) {
  float2 a[8];
  for (int i = 0; i < 8; ++i) a[i] = make_float2(threadIdx.x * 0.001f + i, 1.0f + i);
  float2 m = make_float2(1.0001f, 0.9999f), c = make_float2(0.5f, 0.25f);
  __syncthreads();
  long long t0 = clock64();
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (MODE == 0) { a[i].x = fmaf(a[i].x, m.x, c.x); }
      else if (MODE == 1) { a[i].x = fmaf(a[i].x, m.x, c.x); a[i].y = fmaf(a[i].y, m.y, c.y); }
      else if (MODE == 2) { a[i] = __ffma2_rn(a[i], m, c); }
      else { a[i] = __fmul2_rn(a[i], m); }
    }
  }
  long long t1 = clock64();
  float s = 0.f;
  for (int i = 0; i < 8; ++i) s += a[i].x + a[i].y;
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}
template <int MODE> void run(const char* name, int threads) {
  float* out; long long* cyc;
  cudaMalloc(&out, 4 * 1024 * 132); cudaMalloc(&cyc, 8 * 132);
  const int iters = 1000;
  k<MODE><<<1, threads>>>(out, cyc, iters);
  k<MODE><<<1, threads>>>(out, cyc, iters);
  cudaDeviceSynchronize();
  long long h; cudaMemcpy(&h, cyc, 8, cudaMemcpyDeviceToHost);
  const int warps_per_sched = threads / 128 > 0 ? threads / 128 : 1;
  printf("%-28s threads=%4d  cycles/iter(8 instr-groups)=%.2f  -> %.2f cyc per warp-instr-group per scheduler\n",
         name, threads, (double)h / iters, (double)h / iters / 8 / warps_per_sched);
}
int main() {
  for (int t : {32, 128, 256, 512}) {
    run<0>("FFMA (1 fma)", t); run<1>("2x FFMA (2 fma)", t); run<2>("FFMA2 (2 fma)", t); run<3>("FMUL2", t);
  }
  return 0;
}
