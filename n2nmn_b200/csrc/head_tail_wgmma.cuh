// fc_eltwise of the answer heads with many classes (VQA: 3001) on the Hopper tensor cores with
// fp32 parity: scores[root, :] = ê[root, :]·W_out + b as THREE wgmma TF32 products
//   ê_hi·W_hi + ê_lo·W_hi + ê_hi·W_lo      (x_hi = the fp32 value as the tensor core reads it, i.e.
//                                            truncated to TF32; x_lo = x - x_hi, exact in fp32)
// accumulated in one register tile — the same error-compensated scheme as mma_tile.cuh, at the
// wgmma issue rate instead of mma.sync's.
// Operands, all K-major (channel contiguous), TMA SWIZZLE_128B boxes of 32 channels:
//   A_hi = ê [roots][Mp] exactly as head_kernel writes it, A_lo = its truncation remainder (second
//   buffer written by head_kernel), B_hi / B_lo = W_outᵀ [classes padded to 128][Mp] and its
//   remainder, prepared when the weights are set (out_wt_split_kernel).
// CTA = 128 roots x 128 classes, K streamed 32 channels per stage through a 3-stage ring of 64 KB;
// warpgroup 0 = TMA producer (one elected lane), warpgroups 1 and 2 = 64 roots each: 12 wgmma
// m64n128k8 per stage, then accumulator + bias -> the roots' score rows.
#pragma once
#include "node_eval.cuh"
#include "ptx_sm90.cuh"

namespace n2nmn {

constexpr int kHtM = 128, kHtN = 128, kHtK = 32, kHtStages = 3, kHtThreads = 384;
constexpr int kHtTileBytes = 128 * kHtK * 4;            // 16 KB: 128 rows x 32 channels
constexpr int kHtStageBytes = 4 * kHtTileBytes;         // A_hi, A_lo, B_hi, B_lo
constexpr size_t kHtSmemBytes = (size_t)kHtStages * kHtStageBytes + 256 + 1024;

struct HeadTailMaps { CUtensorMap a_hi, a_lo, b_hi, b_lo; };   // box (32 channels, 128 rows)

// W_out [M][C] -> W_outᵀ [Cpad][Mp] as (hi = the value, lo = value - trunc_tf32(value)), zero padded.
__global__ void out_wt_split_kernel(const float* __restrict__ W, int M, int C, float* __restrict__ hi,
                                    float* __restrict__ lo, int Mp, int Cpad) {
  __shared__ float tile[32][33];
  const int c0 = blockIdx.x * 32, k0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int k = k0 + i, cc = c0 + threadIdx.x;
    tile[i][threadIdx.x] = (k < M && cc < C) ? W[(size_t)k * C + cc] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int cc = c0 + i, k = k0 + threadIdx.x;
    if (cc < Cpad && k < Mp) {
      const float v = tile[threadIdx.x][i];
      const float t = __uint_as_float(__float_as_uint(v) & 0xffffe000u);
      hi[(size_t)cc * Mp + k] = v;
      lo[(size_t)cc * Mp + k] = v - t;
    }
  }
}

__global__ void __launch_bounds__(kHtThreads, 1)
head_tail_wgmma_kernel(const __grid_constant__ HeadTailMaps tm, const float* __restrict__ bias,
                       float* const* __restrict__ dst, int row0, int R, int C, int K) {
  extern __shared__ __align__(1024) uint8_t ht_smem_raw[];
  // SWIZZLE_128B tiles need 1024-byte alignment
  uint8_t* ht_smem = ht_smem_raw + ((1024u - (ptx::smem_u32(ht_smem_raw) & 1023u)) & 1023u);
  uint64_t* full = reinterpret_cast<uint64_t*>(ht_smem + kHtStages * kHtStageBytes);
  uint64_t* empty = full + kHtStages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
  const int c0 = blockIdx.x * kHtN, r0 = blockIdx.y * kHtM;
  const int ksteps = (K + kHtK - 1) / kHtK;
  pdl_trigger();
  if (threadIdx.x == 0) {
    ptx::prefetch_tensormap(&tm.a_hi); ptx::prefetch_tensormap(&tm.a_lo);
    ptx::prefetch_tensormap(&tm.b_hi); ptx::prefetch_tensormap(&tm.b_lo);
    for (int s = 0; s < kHtStages; ++s) { ptx::mbar_init(&full[s], 1); ptx::mbar_init(&empty[s], 8); }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    if (warp == 0 && ptx::elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      // the weight planes do not depend on the head kernel: their first stages go out before the
      // dependency wait, the ê planes after it
      int ahead = 0;
      for (; ahead < kHtStages && ahead < ksteps; ++ahead) {
        uint8_t* st = ht_smem + ahead * kHtStageBytes;
        ptx::mbar_arrive_expect_tx(&full[ahead], kHtStageBytes);
        ptx::tma_load_2d(st + 2 * kHtTileBytes, &tm.b_hi, ahead * kHtK, c0, &full[ahead]);
        ptx::tma_load_2d(st + 3 * kHtTileBytes, &tm.b_lo, ahead * kHtK, c0, &full[ahead]);
      }
      pdl_wait();
      for (int ks = 0; ks < ksteps; ++ks) {
        uint8_t* st = ht_smem + stage * kHtStageBytes;
        if (ks >= ahead) {
          ptx::mbar_wait(&empty[stage], phase ^ 1);
          ptx::mbar_arrive_expect_tx(&full[stage], kHtStageBytes);
          ptx::tma_load_2d(st + 2 * kHtTileBytes, &tm.b_hi, ks * kHtK, c0, &full[stage]);
          ptx::tma_load_2d(st + 3 * kHtTileBytes, &tm.b_lo, ks * kHtK, c0, &full[stage]);
        }
        ptx::tma_load_2d(st, &tm.a_hi, ks * kHtK, row0 + r0, &full[stage]);
        ptx::tma_load_2d(st + kHtTileBytes, &tm.a_lo, ks * kHtK, row0 + r0, &full[stage]);
        if (++stage == kHtStages) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  const int t = threadIdx.x - 128 * wg;
  float acc[kHtN / 2];
  int stage = 0;
  uint32_t phase = 0;
  for (int ks = 0; ks < ksteps; ++ks) {
    ptx::mbar_wait(&full[stage], phase);
    const uint32_t base = ptx::smem_u32(ht_smem + stage * kHtStageBytes);
    const uint32_t a_off = (wg - 1) * 64 * 128;   // this warpgroup's 64 roots
    const uint64_t a_hi = ptx::make_smem_desc_sw128(base + a_off);
    const uint64_t a_lo = ptx::make_smem_desc_sw128(base + kHtTileBytes + a_off);
    const uint64_t b_hi = ptx::make_smem_desc_sw128(base + 2 * kHtTileBytes);
    const uint64_t b_lo = ptx::make_smem_desc_sw128(base + 3 * kHtTileBytes);
    ptx::fence_regs(acc);
    ptx::wgmma_fence();
#pragma unroll
    for (int k = 0; k < kHtK / 8; ++k) {   // 32 bytes (2 x 16-byte units) along K per step
      ptx::wgmma_m64n128k8_tf32(acc, a_lo + 2 * k, b_hi + 2 * k, (ks | k) != 0);
      ptx::wgmma_m64n128k8_tf32(acc, a_hi + 2 * k, b_lo + 2 * k, 1);
      ptx::wgmma_m64n128k8_tf32(acc, a_hi + 2 * k, b_hi + 2 * k, 1);
    }
    ptx::wgmma_commit();
    ptx::wgmma_wait<1>();
    ptx::fence_regs(acc);
    if (ks > 0 && lane == 0) ptx::mbar_arrive(&empty[stage == 0 ? kHtStages - 1 : stage - 1]);
    if (++stage == kHtStages) { stage = 0; phase ^= 1; }
  }
  ptx::wgmma_wait<0>();
  ptx::fence_regs(acc);
  // the destination rows are written by the head kernel (PDL predecessor)
  pdl_wait();
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = r0 + 64 * (wg - 1) + ptx::acc_row(t, 2 * h);
    float* out = r < R ? dst[row0 + r] : nullptr;
    if (out == nullptr) continue;
#pragma unroll
    for (int j = 0; j < kHtN / 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int cc = c0 + ptx::acc_col(t, 4 * j + e);
        if (cc < C) out[cc] = acc[4 * j + 2 * h + e] + bias[cc];
      }
    }
  }
}

}  // namespace n2nmn
