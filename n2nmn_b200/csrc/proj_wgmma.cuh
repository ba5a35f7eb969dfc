// K2: conv_image contraction on the Hopper tensor cores (wgmma, TF32 operands, fp32 accumulate)
// with the module epilogue fused on the register accumulator. See proj_common.cuh for the math and
// what is fused.
//
// Tiling. One tile = 128 rows of the flattened (image, pixel) axis x all Mp output columns, walked
// as Mp/256 N-tiles. The persistent grid walks the schedule's tile list (common.cuh): CTA i takes
// the tiles i, i + gridDim.x, ... K is streamed in 32-float (128-byte, one swizzle atom) slices
// through a 4-stage TMA ring (SWIZZLE_128B, K-major): per stage the 128 feature rows (16 KB) and
// the 256 weight columns of the N-tile (32 KB). fp32 operands are read as TF32 straight from the
// caller's fp32 feature grid: no conversion pass.
//
// Warp roles (384 threads): warpgroup 0 = TMA producer (one elected lane; its registers are handed
// to the consumers with setmaxnreg), warpgroups 1 and 2 = consumers. Consumer warpgroup w owns rows
// [64w, 64w + 64) of the tile: it issues wgmma.m64n256k8 (4 per stage), then runs the epilogue on
// its accumulator fragment. A thread holds 2 rows x 64 columns of the N-tile (ptx::acc_row/acc_col):
// the per-row reductions of the fused Find consumers are summed over the four threads of a quad
// with shuffles, and the running (num, den) of every (row, consumer node) lives in shared memory so
// that the node loop is a rolled loop. While a warpgroup runs its epilogue the producer keeps
// filling the ring for the next N-tile.
//
// Precision: TF32 operands (10-bit mantissa), fp32 accumulate. tests/test_gpu_parity.py holds every
// attention map to 1e-3 abs against the fp32/fp64 oracle.
#pragma once
#include "proj_common.cuh"
#include "ptx_sm90.cuh"

namespace n2nmn {

constexpr int kBM = 128;           // rows per tile
constexpr int kBN = 256;           // columns per N-tile (wgmma N)
constexpr int kBNHalf = kBN / 2;   // rows of one weight TMA box (the box limit is 256; 128 keeps
                                   // the B map shared with the CUDA-core checks of the layout)
constexpr int kBK = 32;            // fp32 elements per K slice = 128 bytes
constexpr int kWgmmaK = 8;         // K per wgmma for tf32 (32 bytes)
constexpr int kABytes = kBM * kBK * 4;        // 16384
constexpr int kBBytes = kBN * kBK * 4;        // 32768
constexpr int kStageBytes = kABytes + kBBytes;
constexpr int kProjStages = 4;
constexpr int kProjThreads = 384;
constexpr int kProducerRegs = 40, kConsumerRegs = 232;   // 128*40 + 256*232 <= 64 K registers
// running (num, den) of every (consumer node, row): [8 nodes][2][128 rows]
constexpr int kPartFloats = kMaxProjNodesPerPass * 2 * kBM;
// dynamic smem: ring + partial sums + barriers (+ 1 KB for the 1024-byte alignment of the ring)
__host__ __device__ constexpr int proj_smem_bytes() {
  return kProjStages * kStageBytes + kPartFloats * 4 + 256 + 1024;
}

struct ProjTensorMaps {
  CUtensorMap a[kMaxSeg];            // features of each segment [rows, Dk] fp32, box 32 x 128
  CUtensorMap b[NUM_PROJ_SETS];      // W^T [Mp, Kp] fp32 (K-major), box 32 x 128 (half an N-tile)
};

__global__ void __launch_bounds__(kProjThreads, 1)
proj_wgmma_kernel(const __grid_constant__ ProjTensorMaps tm, const ProjParams p) {
  extern __shared__ __align__(1024) uint8_t proj_smem_raw[];
  // SWIZZLE_128B tiles need 1024-byte alignment
  uint8_t* smem = proj_smem_raw + ((1024u - (ptx::smem_u32(proj_smem_raw) & 1023u)) & 1023u);
  float* s_part = reinterpret_cast<float*>(smem + kProjStages * kStageBytes);
  uint64_t* full = reinterpret_cast<uint64_t*>(s_part + kPartFloats);
  uint64_t* empty = full + kProjStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2;   // 0 = producer, 1..2 = consumers
  pdl_trigger();   // let the node kernel's CTAs start prefetching their parameters

  if (threadIdx.x == 0) {
    for (int i = 0; i < kMaxSeg; ++i)
      if (i < p.num_seg) ptx::prefetch_tensormap(&tm.a[i]);
    for (int i = 0; i < NUM_PROJ_SETS; ++i) ptx::prefetch_tensormap(&tm.b[i]);
    for (int s = 0; s < kProjStages; ++s) {
      ptx::mbar_init(&full[s], 1);   // the producer's arrive.expect_tx
      ptx::mbar_init(&empty[s], 8);  // one arrive per consumer warp
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ===================================================================== TMA producer
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kProducerRegs));
    if (warp == 0 && ptx::elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int ti = blockIdx.x; ti < p.num_tiles; ti += gridDim.x) {
        const ProjWork* wk = p.work + ti;
        const int row0 = wk->row0, seg = wk->seg, set = wk->set;
        for (int nt = 0; nt < p.n_tiles; ++nt) {
          for (int kb = 0; kb < p.k_blocks; ++kb) {
            ptx::mbar_wait(&empty[stage], phase ^ 1);
            ptx::mbar_arrive_expect_tx(&full[stage], kStageBytes);
            uint8_t* dst = smem + stage * kStageBytes;
            ptx::tma_load_2d(dst, &tm.a[seg], kb * kBK, row0, &full[stage]);
            ptx::tma_load_2d(dst + kABytes, &tm.b[set], kb * kBK, nt * kBN, &full[stage]);
            ptx::tma_load_2d(dst + kABytes + kBNHalf * kBK * 4, &tm.b[set], kb * kBK,
                             nt * kBN + kBNHalf, &full[stage]);
            if (++stage == kProjStages) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
    return;
  }

  // ======================================================================= consumers
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kConsumerRegs));
  const int t = threadIdx.x - 128 * wg;           // thread inside the consumer warpgroup
  const int q = t & 3;                            // column pair of the quad
  const int rbase = 64 * (wg - 1) + ptx::acc_row(t, 0);   // tile row of register half 0 (+8: 1)
  // tauw / tau2 come from the text-projection kernel, which may still be running (PDL); the
  // producer never touches its output and starts immediately.
  pdl_wait();
  auto release = [&](int s) {   // one arrive per consumer warp
    if (lane == 0) ptx::mbar_arrive(&empty[s]);
  };
  int stage = 0;
  uint32_t phase = 0;
  float acc[kBN / 2];
  for (int ti = blockIdx.x; ti < p.num_tiles; ti += gridDim.x) {
    const ProjWork* wkp = p.work + ti;
    const int pass = wkp->pass;
    const int row0 = wkp->row0, set = wkp->set;
    const int g0 = wkp->seg * p.seg_images;   // first image of this tile's segment
    // the two rows of this thread and their consumers
    int e_beg[2], n_nodes[2], pix[2];
    float* mdst[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = row0 + rbase + 8 * h;
      const bool row_ok = row < p.total_rows;
      const int b = row_ok ? row / p.HW : 0;
      pix[h] = row - b * p.HW;
      e_beg[h] = 0;
      n_nodes[h] = 0;
      mdst[h] = nullptr;
      if (row_ok) {
        if (set == PS_FIND) {
          e_beg[h] = p.img_ptr[g0 + b] + pass * kMaxProjNodesPerPass;
          n_nodes[h] = max(min(p.img_ptr[g0 + b + 1] - e_beg[h], kMaxProjNodesPerPass), 0);
        }
        // stored map (always for the non-Find sets; for PS_FIND only in training schedules)
        const int slot = p.mslot[set * p.num_images + g0 + b];
        if (slot >= 0 && pass == 0) mdst[h] = p.mbuf + ((size_t)slot * p.HW + pix[h]) * p.Mp;
      }
    }
    const float* __restrict__ bias = p.bias[set];

    for (int nt = 0; nt < p.n_tiles; ++nt) {
      // ---- mainloop: 4 wgmma per stage; a stage is released once the next one's are issued
      for (int kb = 0; kb < p.k_blocks; ++kb) {
        ptx::mbar_wait(&full[stage], phase);
        const uint32_t sa = ptx::smem_u32(smem + stage * kStageBytes);
        const uint64_t da = ptx::make_smem_desc_sw128(sa + (wg - 1) * 64 * 128);
        const uint64_t db = ptx::make_smem_desc_sw128(sa + kABytes);
        ptx::fence_regs(acc);
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBK / kWgmmaK; ++k)   // 32 bytes (2 x 16-byte units) along K
          ptx::wgmma_m64n256k8_tf32(acc, da + 2 * k, db + 2 * k, (kb | k) != 0);
        ptx::wgmma_commit();
        if (kb == 0 && set == PS_FIND) {
          // While the first slice's MMAs run: pull the text rows the epilogue reads (this N-tile's
          // columns of tauw / tau2 for every consumer node of the thread's two rows, 8 lines per
          // row, 2 per thread of the quad) into L1, so that the rolled node loop below finds
          // them there instead of waiting on L2 for each node in turn.
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            if (n_nodes[h] > 0) ptx::prefetch_l1(p.node_out + e_beg[h]);
#pragma unroll
            for (int jn = 0; jn < kMaxProjNodesPerPass; ++jn) {
              if (jn < n_nodes[h]) {
                const size_t off = (size_t)p.node_text[e_beg[h] + jn] * p.Mp + nt * kBN + 32 * q;
                ptx::prefetch_l1(p.tauw + off);
                ptx::prefetch_l1(p.tauw + off + 128);
                ptx::prefetch_l1(p.tau2 + off);
                ptx::prefetch_l1(p.tau2 + off + 128);
              }
            }
          }
        }
        ptx::wgmma_wait<1>();
        ptx::fence_regs(acc);
        if (kb > 0) release(stage == 0 ? kProjStages - 1 : stage - 1);
        if (++stage == kProjStages) { stage = 0; phase ^= 1; }
      }
      ptx::wgmma_wait<0>();
      ptx::fence_regs(acc);
      release(stage == 0 ? kProjStages - 1 : stage - 1);

      // ---- epilogue on the accumulator: + bias, stored map, fused Find consumers
      const int colq = nt * kBN + 2 * q;   // + 8 j: columns of registers 4j .. 4j+3
#pragma unroll
      for (int j = 0; j < kBN / 8; ++j) {
        const float2 bb = __ldg(reinterpret_cast<const float2*>(bias + colq + 8 * j));
        acc[4 * j + 0] += bb.x; acc[4 * j + 1] += bb.y;
        acc[4 * j + 2] += bb.x; acc[4 * j + 3] += bb.y;
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (mdst[h] != nullptr) {
#pragma unroll
          for (int j = 0; j < kBN / 8; ++j)
            *reinterpret_cast<float2*>(mdst[h] + colq + 8 * j) =
                make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        }
      }
      if (set != PS_FIND) continue;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        // warp-uniform bound of the per-row node counts: unused node slots are a uniform branch
        int n_max = n_nodes[h];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) n_max = max(n_max, __shfl_xor_sync(0xffffffffu, n_max, o));
        float* pa = s_part + rbase + 8 * h;   // + jn * 2 * kBM (+ kBM)
#pragma unroll 1
        for (int jn = 0; jn < n_max; ++jn) {
          float n0 = 0.f, n1 = 0.f, d0 = 0.f, d1 = 0.f;
          if (jn < n_nodes[h]) {
            const size_t off = (size_t)p.node_text[e_beg[h] + jn] * p.Mp + colq;
            const float* tw = p.tauw + off;
            const float* t2 = p.tau2 + off;
            // One text row at a time, all 32 of its loads in flight before the first FMA (the
            // accumulator leaves room for one row, not two). The squares m² are formed here,
            // inside the node loop: hoisted out of it they would hold 64 registers and leave
            // room for only 2-3 loads in flight, i.e. ~25 serial load round-trips per node.
            float2 w[kBN / 8];
#pragma unroll
            for (int j = 0; j < kBN / 8; ++j) w[j] = __ldg(reinterpret_cast<const float2*>(tw + 8 * j));
#pragma unroll
            for (int j = 0; j < kBN / 8; ++j) {
              n0 = fmaf(acc[4 * j + 2 * h], w[j].x, n0);
              n1 = fmaf(acc[4 * j + 2 * h + 1], w[j].y, n1);
            }
#pragma unroll
            for (int j = 0; j < kBN / 8; ++j) w[j] = __ldg(reinterpret_cast<const float2*>(t2 + 8 * j));
#pragma unroll
            for (int j = 0; j < kBN / 8; ++j) {
              float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
              asm volatile("" : "+f"(v0), "+f"(v1));   // keeps v² in the loop
              d0 = fmaf(v0 * v0, w[j].x, d0);
              d1 = fmaf(v1 * v1, w[j].y, d1);
            }
          }
          float n = n0 + n1, d = d0 + d1;
          n += __shfl_xor_sync(0xffffffffu, n, 1);
          d += __shfl_xor_sync(0xffffffffu, d, 1);
          n += __shfl_xor_sync(0xffffffffu, n, 2);
          d += __shfl_xor_sync(0xffffffffu, d, 2);
          if (q == 0 && jn < n_nodes[h]) {
            float* pj = pa + jn * (2 * kBM);
            if (nt == 0) { pj[0] = n; pj[kBM] = d; }
            else { pj[0] += n; pj[kBM] += d; }
          }
        }
      }
    }
    // the N-tiles of a row meet here (the same thread wrote every partial sum it reads)
    if (set == PS_FIND && q == 0) {
      const float b2 = __ldg(p.elt_b);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float* pa = s_part + rbase + 8 * h;
        for (int j = 0; j < n_nodes[h]; ++j) {
          const float nn = pa[j * 2 * kBM], dd = pa[j * 2 * kBM + kBM];
          p.arena[(size_t)p.node_out[e_beg[h] + j] * p.HW + pix[h]] = nn * rsqrtf(fmaxf(dd, kEps)) + b2;
        }
      }
    }
  }
}

}  // namespace n2nmn
