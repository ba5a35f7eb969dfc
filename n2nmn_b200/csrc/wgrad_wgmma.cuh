// Weight gradient of the feature-side layers on the Hopper tensor cores:
//   dW_set[k, c] += Σ_entries Σ_p X_b[p, k] · B_entry[p, c]        (backward.cuh, FeatGradSrc)
// as wgmma TF32 products with the pixels p as the contraction index. p is the slow index of the
// feature grid X [p][k] and of the B maps [p][c], exactly as the forward pass and the reverse walk
// leave them; TF32 wgmma reads shared-memory operands K-major only, so every 32-pixel stage is
// staged TRANSPOSED: the CTA's threads load X (32 pixels x 128 features) and B (32 pixels x 256
// channels) with coalesced 16-byte loads and store them as K-major 128B-swizzled tiles
// Xᵀ [128 rows k][32 p] and Bᵀ [256 rows c][32 p] (the layout TMA's SWIZZLE_128B would write).
// The global loads of stage s+1 are issued before waiting on the wgmma of stage s.
//   CTA = one 128-feature slab of k x one 256-channel tile (blockIdx.z; Mp is a multiple of 256)
//   x a chunk of the entries (sorted by weight set by the host), 256 threads = 2 warpgroups of 64
//   features each: wgmma.m64n256k8, 4 per stage; the accumulator is flushed with float2
//   reductions when the weight set changes and at the end. Pixels >= H·W are zero, and so are the
//   features k >= Dk of a ragged last slab (VQA: Dk = 2050, the two coordinate channels last);
//   their gradient rows are not written. The feature rows are read at their pitch (the
//   coordinate-augmented / re-pitched copy of the forward pass, or the caller's grid).
// Operands are the fp32 bits read as TF32 (as in the forward contraction); fp32 accumulate.
#pragma once
#include "backward.cuh"
#include "ptx_sm90.cuh"

namespace n2nmn {

constexpr int kWgM = 128, kWgN = 256, kWgP = 32, kWgThreads = 256;
constexpr int kWgABytes = kWgM * kWgP * 4;   // 16 KB
constexpr int kWgBBytes = kWgN * kWgP * 4;   // 32 KB
constexpr size_t kWgSmemBytes = (size_t)kWgABytes + kWgBBytes + 1024;

struct WgradParams {
  const float* feat;           // [images][HW][pitch]
  const float* dmap;           // B maps [entries][HW][Mp]
  const BwdEntry* entries;     // [num_entries] {set, image}
  const int32_t* order;        // entry indices sorted by weight set
  int num_entries, per_cta, HW, Dk, M, Mp, pitch;
  float* gflat;
  GradOffsets go;
};

// element (row r, pixel p) of a K-major SWIZZLE_128B tile with 32 fp32 per row
__device__ __forceinline__ int sw128_index(int r, int p) {
  return r * kWgP + ((((p >> 2) ^ (r & 7))) << 2) + (p & 3);
}

__global__ void __launch_bounds__(kWgThreads, 1)
wgrad_wgmma_kernel(const WgradParams p) {
  extern __shared__ __align__(1024) uint8_t wg_smem_raw[];
  uint8_t* smem = wg_smem_raw + ((1024u - (ptx::smem_u32(wg_smem_raw) & 1023u)) & 1023u);
  float* sa = reinterpret_cast<float*>(smem);                 // Xᵀ [128][32]
  float* sb = reinterpret_cast<float*>(smem + kWgABytes);     // Bᵀ [256][32]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2, t = tid & 127;
  const int k0 = blockIdx.x * kWgM, n0 = blockIdx.z * kWgN;
  const int e0 = blockIdx.y * p.per_cta, e1 = min(p.num_entries, e0 + p.per_cta);
  const int stages_per_entry = (p.HW + kWgP - 1) / kWgP;
  const int n_stages = (e1 > e0 ? e1 - e0 : 0) * stages_per_entry;
  // thread -> (pixel, column quad) of its loads: a warp covers 8 pixels x 4 quads (64 B per row)
  const int p_lo = lane >> 2, q_lo = lane & 3;

  float4 xa[4], xb[8];
  auto load = [&](int s) {
    const int e = p.order[e0 + s / stages_per_entry];
    const int p0 = (s % stages_per_entry) * kWgP;
    const float* X = p.feat + (size_t)p.entries[e].b * p.HW * p.pitch + k0;
    const float* B = p.dmap + (size_t)e * p.HW * p.Mp + n0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {   // 32 pixels x 32 quads of 128 features
      const int px = p0 + i * 8 + p_lo, q = warp * 4 + q_lo;
      xa[i] = (px < p.HW && k0 + 4 * q < p.Dk)
                  ? __ldg(reinterpret_cast<const float4*>(X + (size_t)px * p.pitch) + q)
                  : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {   // 32 pixels x 64 quads of 256 channels
      const int px = p0 + (i >> 1) * 8 + p_lo, q = (i & 1) * 32 + warp * 4 + q_lo;
      xb[i] = px < p.HW ? __ldg(reinterpret_cast<const float4*>(B + (size_t)px * p.Mp) + q)
                        : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  auto store = [&]() {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int px = i * 8 + p_lo, r = 4 * (warp * 4 + q_lo);
      sa[sw128_index(r + 0, px)] = xa[i].x; sa[sw128_index(r + 1, px)] = xa[i].y;
      sa[sw128_index(r + 2, px)] = xa[i].z; sa[sw128_index(r + 3, px)] = xa[i].w;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int px = (i >> 1) * 8 + p_lo, r = 4 * ((i & 1) * 32 + warp * 4 + q_lo);
      sb[sw128_index(r + 0, px)] = xb[i].x; sb[sw128_index(r + 1, px)] = xb[i].y;
      sb[sw128_index(r + 2, px)] = xb[i].z; sb[sw128_index(r + 3, px)] = xb[i].w;
    }
  };

  float acc[kWgN / 2];
  const int q = t & 3;
  auto flush = [&](int set) {
    ptx::wgmma_wait<0>();
    ptx::fence_regs(acc);
    float* W = p.gflat + p.go.proj_w[set];
    const bool pair_ok = (p.M & 1) == 0 && (reinterpret_cast<uintptr_t>(W) & 7) == 0;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int k = k0 + 64 * wg + ptx::acc_row(t, 2 * h);
      if (k >= p.Dk) continue;
#pragma unroll
      for (int j = 0; j < kWgN / 8; ++j) {
        const int col = n0 + 8 * j + 2 * q;
        const float a = acc[4 * j + 2 * h], b = acc[4 * j + 2 * h + 1];
        float* dst = W + (size_t)k * p.M + col;
        if (pair_ok && col + 1 < p.M) {
          if (a != 0.f || b != 0.f) atomicAdd(reinterpret_cast<float2*>(dst), make_float2(a, b));
        } else {
          if (col < p.M && a != 0.f) atomicAdd(dst, a);
          if (col + 1 < p.M && b != 0.f) atomicAdd(dst + 1, b);
        }
      }
    }
  };

  const uint32_t a_desc_base = ptx::smem_u32(sa) + wg * 64 * 128;
  const uint32_t b_desc_base = ptx::smem_u32(sb);
  int cur_set = -1;
  bool fresh = true;
  if (n_stages > 0) load(0);
  for (int s = 0; s < n_stages; ++s) {
    const int set = p.entries[p.order[e0 + s / stages_per_entry]].set;
    if (set != cur_set) {
      if (cur_set >= 0) flush(cur_set);
      cur_set = set;
      fresh = true;
    }
    ptx::wgmma_wait<0>();   // the previous stage's wgmma no longer read the tiles
    __syncthreads();
    store();
    ptx::fence_proxy_async();   // generic-proxy stores -> visible to wgmma (async proxy)
    __syncthreads();
    if (s + 1 < n_stages) load(s + 1);   // in flight under this stage's wgmma
    ptx::fence_regs(acc);
    ptx::wgmma_fence();
    const uint64_t da = ptx::make_smem_desc_sw128(a_desc_base);
    const uint64_t db = ptx::make_smem_desc_sw128(b_desc_base);
#pragma unroll
    for (int k = 0; k < kWgP / 8; ++k)   // 32 bytes (2 x 16-byte units) along the pixels
      ptx::wgmma_m64n256k8_tf32(acc, da + 2 * k, db + 2 * k, !(fresh && k == 0));
    ptx::wgmma_commit();
    fresh = false;
  }
  if (cur_set >= 0) flush(cur_set);
}

// Bias gradient of the same layers: db_set[c] += Σ_p B_entry[p, c]. One CTA per B map; 4 row
// groups x 256 columns so that every thread has many independent loads (one thread per column over
// all rows is a long latency chain).
__global__ void __launch_bounds__(1024)
bmap_colsum_kernel(const float* __restrict__ dmap, const BwdEntry* __restrict__ entries, int HW,
                   int M, int Mp, float* __restrict__ gflat, GradOffsets go) {
  __shared__ float part[4][256];
  const int e = blockIdx.x, c = threadIdx.x & 255, rg = threadIdx.x >> 8;
  const float* B = dmap + (size_t)e * HW * Mp;
  float* dst = gflat + go.proj_b[entries[e].set];
  for (int c0 = 0; c0 < M; c0 += 256) {
    const int col = c0 + c;
    float s = 0.f;
    if (col < M) {
#pragma unroll 8
      for (int p = rg; p < HW; p += 4) s += B[(size_t)p * Mp + col];
    }
    part[rg][c] = s;
    __syncthreads();
    if (rg == 0 && col < M) {
      const float t = (part[0][c] + part[1][c]) + (part[2][c] + part[3][c]);
      if (t != 0.f) atomicAdd(dst + col, t);
    }
    __syncthreads();
  }
}

}  // namespace n2nmn
