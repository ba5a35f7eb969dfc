// fp32 CUDA-core implementation of the conv_image contraction + fused consumers.
// Verification path (N2NMN_FLAG_PROJ_FP32_SIMT): exact fp32 FMAs, no TF32 rounding, so GPU tests
// can tell a tensor-core descriptor bug from a rounding difference. Not tuned.
#pragma once
#include "proj_common.cuh"

namespace n2nmn {

constexpr int kSimtRows = 8;      // rows per inner step (one per warp in the epilogue)
constexpr int kSimtKChunk = 256;  // K staged per step
constexpr int kSimtMaxColIters = 4;  // Mp <= 1024

__global__ void __launch_bounds__(256)
proj_simt_kernel(ProjParams p) {
  extern __shared__ float smem[];
  pdl_trigger();
  pdl_wait();
  float* xs = smem;                                  // [kSimtRows][kSimtKChunk]
  float* ms = smem + kSimtRows * kSimtKChunk;        // [kSimtRows][Mp]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int col_iters = p.Mp / 256;

  for (int ti = blockIdx.x; ti < p.num_tiles; ti += gridDim.x) {   // one CTA per tile
    const ProjWork wk = p.work[ti];
    const int wk_pass = wk.pass, wk_row0 = wk.row0;
    const int g0 = wk.seg * p.seg_images;
    const float* __restrict__ feat = p.feat_seg[wk.seg];
    const float* __restrict__ W = p.w_orig[wk.set];
    for (int r0 = 0; r0 < 128; r0 += kSimtRows) {
      const int row_base = wk_row0 + r0;
      if (row_base >= p.total_rows) break;
      float acc[kSimtMaxColIters][kSimtRows];
#pragma unroll
      for (int j = 0; j < kSimtMaxColIters; ++j)
#pragma unroll
        for (int r = 0; r < kSimtRows; ++r) acc[j][r] = 0.f;
      for (int k0 = 0; k0 < p.Dk; k0 += kSimtKChunk) {
        __syncthreads();
        for (int i = tid; i < kSimtRows * kSimtKChunk; i += blockDim.x) {
          const int r = i / kSimtKChunk, k = i - r * kSimtKChunk;
          const int row = row_base + r;
          xs[i] = (row < p.total_rows && k0 + k < p.Dk)
                      ? feat[(size_t)row * p.feat_pitch + k0 + k] : 0.f;
        }
        __syncthreads();
        const int kmax = min(kSimtKChunk, p.Dk - k0);
        for (int k = 0; k < kmax; ++k) {
#pragma unroll
          for (int j = 0; j < kSimtMaxColIters; ++j) {
            const int c = tid + 256 * j;
            if (j < col_iters && c < p.M) {
              const float w = __ldg(W + (size_t)(k0 + k) * p.M + c);
#pragma unroll
              for (int r = 0; r < kSimtRows; ++r)
                acc[j][r] = fmaf(xs[r * kSimtKChunk + k], w, acc[j][r]);
            }
          }
        }
      }
      __syncthreads();
#pragma unroll
      for (int j = 0; j < kSimtMaxColIters; ++j) {
        const int c = tid + 256 * j;
        if (j < col_iters) {
          const float b = p.bias[wk.set][c];
#pragma unroll
          for (int r = 0; r < kSimtRows; ++r) ms[r * p.Mp + c] = (c < p.M) ? acc[j][r] + b : 0.f;
        }
      }
      __syncthreads();
      // epilogue: warp `warp` owns row row_base + warp
      const int row = row_base + warp;
      if (row < p.total_rows) {
        const int bl = row / p.HW, pix = row - bl * p.HW;
        const int b = g0 + bl;   // image index across the segments
        const float* mrow = ms + warp * p.Mp;
        if (wk.set == PS_FIND) {
          const int beg = p.img_ptr[b] + wk_pass * kMaxProjNodesPerPass;
          const int end = min(p.img_ptr[b + 1], beg + kMaxProjNodesPerPass);
          for (int e = beg; e < end; ++e) {
            const float* tw = p.tauw + (size_t)p.node_text[e] * p.Mp;
            const float* t2 = p.tau2 + (size_t)p.node_text[e] * p.Mp;
            float num = 0.f, den = 0.f;
            for (int c = lane; c < p.Mp; c += 32) {
              const float m = mrow[c];
              num = fmaf(m, tw[c], num);
              den = fmaf(m * m, t2[c], den);
            }
            num = warp_sum(num);
            den = warp_sum(den);
            if (lane == 0)
              p.arena[(size_t)p.node_out[e] * p.HW + pix] =
                  num * rsqrtf(fmaxf(den, kEps)) + p.elt_b[0];
          }
        }
        {
          const int slot = p.mslot[wk.set * p.num_images + b];
          if (slot >= 0 && wk_pass == 0) {
            float* dst = p.mbuf + ((size_t)slot * p.HW + pix) * p.Mp;
            for (int c = lane; c < p.Mp; c += 32) dst[c] = mrow[c];
          }
        }
      }
    }
  }
}

}  // namespace n2nmn
