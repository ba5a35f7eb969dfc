// One-off data-layout kernels: weight repacking at n2nmn_set_weight time and the VQA
// coordinate-channel augmentation at bind time.
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"
#include "optim.cuh"

namespace n2nmn {

// W [K][M] (TF layout, models_clevr/nmn3_modules.py:101 'conv_image/weights') ->
// Wt [Mp][Kp] K-major with zero padding: the B operand layout of the wgmma contraction.
__global__ void transpose_pad_kernel(const float* __restrict__ W, int K, int M,
                                     float* __restrict__ Wt, int Kp, int Mp) {
  __shared__ float tile[32][33];
  const int k0 = blockIdx.x * 32, m0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int k = k0 + i, m = m0 + threadIdx.x;
    tile[i][threadIdx.x] = (k < K && m < M) ? W[(size_t)k * M + m] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int m = m0 + i, k = k0 + threadIdx.x;
    if (m < Mp && k < Kp) Wt[(size_t)m * Kp + k] = tile[threadIdx.x][i];
  }
}

__global__ void pad_copy_kernel(const float* __restrict__ src, int n, float* __restrict__ dst,
                                int np) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < np) dst[i] = (i < n) ? src[i] : 0.f;
}

// [rows][M] -> [rows][Mp] with zero padding, so rows are 16-byte aligned for float4 loads.
__global__ void pitch_rows_kernel(const float* __restrict__ src, int rows, int M,
                                  float* __restrict__ dst, int Mp) {
  const int r = blockIdx.x;
  if (r >= rows) return;
  for (int c = threadIdx.x; c < Mp; c += blockDim.x)
    dst[(size_t)r * Mp + c] = (c < M) ? src[(size_t)r * M + c] : 0.f;
}

// Feature grids that travel over PCIe as IEEE fp16 (n2nmn_forward_group_host_f16_async): widen to
// the fp32 layout every kernel reads. 8 values per thread: one 16-byte load, two 16-byte stores.
// n8 = count / 8 (the staging buffers are padded to a multiple of 8).
__global__ void widen_f16_kernel(const uint4* __restrict__ src, float4* __restrict__ dst,
                                 size_t n8) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n8;
       i += (size_t)gridDim.x * blockDim.x) {
    const uint4 v = src[i];
    const __half2* h = reinterpret_cast<const __half2*>(&v);
    const float2 a = __half22float2(h[0]), b = __half22float2(h[1]);
    const float2 c = __half22float2(h[2]), d = __half22float2(h[3]);
    dst[2 * i] = make_float4(a.x, a.y, b.x, b.y);
    dst[2 * i + 1] = make_float4(c.x, c.y, d.x, d.y);
  }
}

// ---- all variables from one flat buffer in two launches (after every optimiser step) ------------
// RepackSeg (optim.cuh) kind 0: plain copy of `count` floats; kind 1: [rows][cols] -> [rows][pitch]
// zero padded.
// grid = (16, variables)
__global__ void repack_all_kernel(const float* __restrict__ wflat, const RepackSeg* __restrict__ segs,
                                  float* __restrict__ wbuf, int pitch) {
  const RepackSeg s = segs[blockIdx.y];
  const float* src = wflat + s.src_off;
  float* dst = wbuf + s.dst_off;
  if (s.kind == 0) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < s.count; i += gridDim.x * blockDim.x)
      dst[i] = src[i];
  } else {
    const int rows = s.count / s.cols, n = rows * pitch;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
      const int r = i / pitch, cidx = i - r * pitch;
      dst[i] = cidx < s.cols ? src[(size_t)r * s.cols + cidx] : 0.f;
    }
  }
}
// The K-major padded copies of the conv_image / fc_att weights (wgmma B operand) and their padded
// biases, every projection set in one launch: grid = (Kp/32, Mp/32, sets), block (32, 8).
struct ProjRepack {
  int w_off[NUM_PROJ_SETS], b_off[NUM_PROJ_SETS];   // offsets in the flat buffer (-1: set not owned)
  float* wt[NUM_PROJ_SETS];
  float* bias[NUM_PROJ_SETS];
  int set_of_z[NUM_PROJ_SETS];
};
__global__ void proj_repack_kernel(const float* __restrict__ wflat, ProjRepack pr, int K, int M,
                                   int Kp, int Mp) {
  __shared__ float tile[32][33];
  const int set = pr.set_of_z[blockIdx.z];
  const float* W = wflat + pr.w_off[set];
  float* Wt = pr.wt[set];
  const int k0 = blockIdx.x * 32, m0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int k = k0 + i, m = m0 + threadIdx.x;
    tile[i][threadIdx.x] = (k < K && m < M) ? W[(size_t)k * M + m] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int m = m0 + i, k = k0 + threadIdx.x;
    if (m < Mp && k < Kp) Wt[(size_t)m * Kp + k] = tile[threadIdx.x][i];
  }
  if (blockIdx.x == 0 && blockIdx.y == 0 && pr.b_off[set] >= 0) {
    const float* b = wflat + pr.b_off[set];
    for (int i = threadIdx.y * 32 + threadIdx.x; i < Mp; i += 32 * blockDim.y)
      pr.bias[set][i] = i < M ? b[i] : 0.f;
  }
}

// conv_quad^T [Mp][quad_pitch] (common.cuh: Transform as a quadratic form), the B operand of
// quad_kernel (text_proj.cuh): column o < n: K̃_o ∘ w2; columns [n, quad_u_pitch): zero; then one
// column per pair i <= j: (2-δ_ij) K̃_i ∘ K̃_j, with K̃ = [conv_maps taps (row pitch Mp) ;
// conv_maps bias]. One CTA per output column. Re-run whenever one of the three variables changes.
__global__ void conv_quad_kernel(const float* __restrict__ conv_k, const float* __restrict__ conv_b,
                                 const float* __restrict__ w2, int ks, int M, int Mp,
                                 float* __restrict__ out) {
  const int n = quad_n(ks), nu = quad_u_pitch(ks), qp = quad_pitch(ks), o = blockIdx.x;
  int i = o, j = -1;
  bool zero = false;
  if (o >= n && o < nu) zero = true;
  if (o >= nu) {                        // pair index -> (i, j), i <= j
    int idx = o - nu;
    i = 0;
    while (i < n && idx >= n - i) { idx -= n - i; ++i; }
    j = i + idx;
    if (i >= n) zero = true;           // padding columns beyond the last pair
  }
  for (int c = threadIdx.x; c < Mp; c += blockDim.x) {
    float v = 0.f;
    if (c < M && !zero) {
      const float ki = (i < n - 1) ? conv_k[(size_t)i * Mp + c] : conv_b[c];
      if (j < 0) v = ki * w2[c];
      else {
        const float kj = (j < n - 1) ? conv_k[(size_t)j * Mp + c] : conv_b[c];
        v = ki * kj * (i == j ? 1.f : 2.f);
      }
    }
    out[(size_t)c * qp + o] = v;
  }
}

// add_spatial_coordinate_map (models_vqa/nmn3_modules.py:11-31): dst[r, :] =
// [src[r, 0:D], x, y, 0...] with x = linspace(-1,1,W)[col], y = linspace(-1,1,H)[row]; also used
// (with_coords = 0) to re-pitch feature grids whose channel count is not a multiple of 4.
__global__ void augment_features_kernel(const float* __restrict__ src, int rows, int D, int H,
                                        int W, int with_coords, float* __restrict__ dst,
                                        int pitch) {
  const int r = blockIdx.x;
  if (r >= rows) return;
  const int pix = r % (H * W);
  const int y = pix / W, x = pix - y * W;
  // tf.linspace(-1., 1., n)[i] = -1 + i * (2 / (n - 1)); n == 1 gives -1
  const float xv = (W > 1) ? -1.f + (float)x * (2.f / (float)(W - 1)) : -1.f;
  const float yv = (H > 1) ? -1.f + (float)y * (2.f / (float)(H - 1)) : -1.f;
  for (int c = threadIdx.x; c < pitch; c += blockDim.x) {
    float v = 0.f;
    if (c < D) v = src[(size_t)r * D + c];
    else if (with_coords && c == D) v = xv;
    else if (with_coords && c == D + 1) v = yv;
    dst[(size_t)r * pitch + c] = v;
  }
}

}  // namespace n2nmn
