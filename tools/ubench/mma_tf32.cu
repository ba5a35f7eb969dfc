// Microbenchmark: issue rate of the legacy register-fragment tensor path (mma.sync m16n8k8 tf32).
#include <cstdio>
#include <cuda_runtime.h>
__global__ void k(float* out, long long* cyc, int iters) {
  float d[8][4];
  for (int i = 0; i < 8; ++i) for (int j = 0; j < 4; ++j) d[i][j] = 0.f;
  unsigned a[4] = {0x3f800000u + threadIdx.x, 0x3f900000u, 0x3fa00000u, 0x3fb00000u};
  unsigned b[2] = {0x3f800000u, 0x3f000000u + threadIdx.x};
  __syncthreads();
  long long t0 = clock64();
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 8; ++i)
      asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                   : "+f"(d[i][0]), "+f"(d[i][1]), "+f"(d[i][2]), "+f"(d[i][3])
                   : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
  }
  long long t1 = clock64();
  float s = 0.f;
  for (int i = 0; i < 8; ++i) for (int j = 0; j < 4; ++j) s += d[i][j];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}
int main() {
  float* out; long long* cyc;
  cudaMalloc(&out, 4 * 1024 * 132); cudaMalloc(&cyc, 8 * 132);
  const int iters = 1000;
  for (int t : {32, 128, 256, 512}) {
    k<<<1, t>>>(out, cyc, iters); k<<<1, t>>>(out, cyc, iters);
    cudaDeviceSynchronize();
    long long h; cudaMemcpy(&h, cyc, 8, cudaMemcpyDeviceToHost);
    const int wps = t / 128 > 0 ? t / 128 : 1;
    printf("mma.sync m16n8k8 tf32: threads=%4d  cycles per 8 independent mma = %.1f -> %.2f cyc per mma per scheduler (1024 MAC each)\n",
           t, (double)h / iters, (double)h / iters / 8 / wps);
  }
  return 0;
}
