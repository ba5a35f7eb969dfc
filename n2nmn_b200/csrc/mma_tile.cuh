// 64 x 32 (or 32 x 32) fp32-parity GEMM tile on mma.sync m16n8k8 with error-compensated TF32,
// operands streamed through a cp.async ring. Shared by the seq2seq kernels (seq2seq.cu) and the
// text projections (text_proj.cuh).
#pragma once
#include "common.cuh"
#include "tile_gemm.cuh"

namespace n2nmn {

// ---- 64 x 32 output tile on mma.sync m16n8k8 with error-compensated TF32 (3 products per
// fragment pair: hi*hi + hi*lo + lo*hi, fp32 accumulate: ~2^-21 relative, i.e. fp32 parity —
// the decoded TOKENS must match the reference's fp32 graph, so plain TF32 is not an option).
// Operands are split by truncation (hi = the top 19 bits, lo = x - hi exactly; the tensor core
// ignores the low 13 bits of lo): 2 ALU instructions per element where cvt.rna is a sequence.
//   C[r, c] = Σ_k A[r, k] B[k, c],  A = [A0 | A1] (two row-major sources side by side: the layer
//   input and the recurrent state), B row-major with pitch ldb.
// 8 warps = 4 row tiles of 16 x 2 halves of every 128-deep K chunk; chunks stream through a
// 3-stage cp.async ring (A 64x128, B 128x32 per stage). B (weights) of the first stages is
// requested BEFORE griddepcontrol.wait: under programmatic dependent launch the weight fetch of
// step t+1 overlaps the tail of step t.
constexpr int kMmaCols = 32, kMmaKC = 128, kMmaThreads = 256;
constexpr int kMmaAPitch = kMmaKC + 4;     // rows g / g+8 and k / k+4 of a fragment: distinct banks
constexpr int kMmaBPitch = kMmaCols + 8;
// a stage = A [16 WM][kMmaAPitch] then B [kMmaKC][kMmaBPitch]: 3 stages (162 KB) for 64-row tiles,
// 5 stages (187 KB) for 32-row tiles: at N <= 64 a step is bound by the latency of its operand
// stream, i.e. by the bytes in flight per SM (measured 2.59 -> 1.97 ms per batch from 3 to 5)
__host__ __device__ constexpr int mma_stage_floats(int wm) {
  return 16 * wm * kMmaAPitch + kMmaKC * kMmaBPitch;
}
constexpr int kMmaStagesNarrow = 5;
__host__ __device__ constexpr int mma_stages(int wm) { return wm == 2 ? kMmaStagesNarrow : 3; }
__host__ __device__ constexpr size_t mma_smem_bytes(int wm, int stages = 0) {
  return (size_t)(stages > 0 ? stages : mma_stages(wm)) * mma_stage_floats(wm) * sizeof(float);
}

struct GemmOperands {
  const float* a0; int k0, lda0;   // A columns [0, k0)
  const float* a1; int k1, lda1;   // A columns [k0, k0 + k1)  (k1 may be 0)
  int R;                           // valid rows
  const float* B; int ldb, C;      // B [k0 + k1][ldb], C valid columns
  // gathered A (text projection): pointer to the K-contiguous data of each of the tile's rows
  // (nullptr = a row of zeros), indexed by the row inside the tile; a0 / a1 / R are then unused
  const float* const* a_rows = nullptr;
};

__device__ __forceinline__ void split_trunc(float x, uint32_t& hi, uint32_t& lo) {
  hi = __float_as_uint(x) & 0xffffe000u;
  lo = __float_as_uint(x - __uint_as_float(hi));
}
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0,
                                         uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
      "{%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// WM = row tiles of 16 per CTA (4: 64 rows, 2: 32 rows); the 8 warps split every K chunk
// KH = 8 / WM ways. acc[nt][0..3]: rows (wm*16 + g, +8), columns nt*8 + 2*tig (+1) of the tile;
// valid in the warps with kh == 0 (returns true there) after the call.
// after_wait(): called once griddepcontrol.wait has returned and the first A chunks are in
// flight — the place to start the loads the epilogue will need.
// kExact = true: three products per fragment pair (fp32 parity); false: one TF32 product with the
// operands rounded to nearest (add half an ulp; the tensor core drops the low 13 bits).
// ST = ring depth (default: mma_stages(WM)); short-K callers (text projection: 3 chunks) take 2
// stages so that two CTAs share an SM. K-steps entirely beyond K are skipped.
template <int WM, bool kExact = true, int ST = 0, class AfterWait>
__device__ __forceinline__ bool mma_tile(float* smem, const GemmOperands& p, int row0, int c0,
                                         float (&acc)[4][4], AfterWait after_wait) {
  constexpr int KH = 8 / WM, ROWS = 16 * WM, KW = kMmaKC / KH;   // k extent per warp per chunk
  constexpr int kMmaStageFloats = mma_stage_floats(WM), kMmaStages = ST > 0 ? ST : mma_stages(WM);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wm = warp % WM, kh = warp / WM, g = lane >> 2, tig = lane & 3;
  const int K = p.k0 + p.k1, nchunks = (K + kMmaKC - 1) / kMmaKC;
  auto load_b = [&](int chunk, int stage) {
    float* Bs = smem + stage * kMmaStageFloats + ROWS * kMmaAPitch;
    const int kc0 = chunk * kMmaKC;
    for (int i = tid; i < kMmaKC * (kMmaCols / 4); i += kMmaThreads) {
      const int kk = i >> 3, q = i & 7, k = kc0 + kk, col = c0 + 4 * q;
      float* dst = Bs + kk * kMmaBPitch + 4 * q;
      if (k < K && col < p.C) tp_cp16(dst, p.B + (size_t)k * p.ldb + col);
      else *reinterpret_cast<float4*>(dst) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  auto load_a = [&](int chunk, int stage) {
    float* As = smem + stage * kMmaStageFloats;
    const int kc0 = chunk * kMmaKC;
    for (int i = tid; i < ROWS * (kMmaKC / 4); i += kMmaThreads) {
      const int r = i >> 5, q = i & 31, k = kc0 + 4 * q, row = row0 + r;
      float* dst = As + r * kMmaAPitch + 4 * q;
      if (p.a_rows != nullptr) {
        const float* base = p.a_rows[r];
        if (base != nullptr && k < K) tp_cp16(dst, base + k);
        else *reinterpret_cast<float4*>(dst) = make_float4(0.f, 0.f, 0.f, 0.f);
      } else if (row < p.R && k < K) {
        const float* src = k < p.k0 ? p.a0 + (size_t)row * p.lda0 + k
                                    : p.a1 + (size_t)row * p.lda1 + (k - p.k0);
        tp_cp16(dst, src);
      } else {
        *reinterpret_cast<float4*>(dst) = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
  };
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int s = 0; s < kMmaStages - 1; ++s)
    if (s < nchunks) load_b(s, s);
  pdl_wait();   // everything below may read what the previous kernel in the stream wrote
  for (int s = 0; s < kMmaStages - 1; ++s) {
    if (s < nchunks) load_a(s, s);
    tp_commit();
  }
  after_wait();
  for (int c = 0; c < nchunks; ++c) {
    tp_wait<kMmaStages - 2>();
    __syncthreads();
    const int nx = c + kMmaStages - 1;
    if (nx < nchunks) { load_b(nx, nx % kMmaStages); load_a(nx, nx % kMmaStages); }
    tp_commit();
    const float* As = smem + (c % kMmaStages) * kMmaStageFloats + (wm * 16 + g) * kMmaAPitch;
    const float* Bs = smem + (c % kMmaStages) * kMmaStageFloats + ROWS * kMmaAPitch + g;
#pragma unroll 2
    for (int ks = 0; ks < KW / 8; ++ks) {
      const int kb = kh * KW + ks * 8;
      if (c * kMmaKC + kb >= K) break;   // (zero-filled beyond K: nothing to add)
      if constexpr (kExact) {
        uint32_t ah[4], al[4];
        split_trunc(As[kb + tig], ah[0], al[0]);
        split_trunc(As[8 * kMmaAPitch + kb + tig], ah[1], al[1]);
        split_trunc(As[kb + tig + 4], ah[2], al[2]);
        split_trunc(As[8 * kMmaAPitch + kb + tig + 4], ah[3], al[3]);
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
          uint32_t bh0, bl0, bh1, bl1;
          split_trunc(Bs[(kb + tig) * kMmaBPitch + nt * 8], bh0, bl0);
          split_trunc(Bs[(kb + tig + 4) * kMmaBPitch + nt * 8], bh1, bl1);
          mma_tf32(acc[nt], al, bh0, bh1);
          mma_tf32(acc[nt], ah, bl0, bl1);
          mma_tf32(acc[nt], ah, bh0, bh1);
        }
      } else {
        const uint32_t a[4] = {__float_as_uint(As[kb + tig]) + 0x1000u,
                               __float_as_uint(As[8 * kMmaAPitch + kb + tig]) + 0x1000u,
                               __float_as_uint(As[kb + tig + 4]) + 0x1000u,
                               __float_as_uint(As[8 * kMmaAPitch + kb + tig + 4]) + 0x1000u};
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
          mma_tf32(acc[nt], a, __float_as_uint(Bs[(kb + tig) * kMmaBPitch + nt * 8]) + 0x1000u,
                   __float_as_uint(Bs[(kb + tig + 4) * kMmaBPitch + nt * 8]) + 0x1000u);
      }
    }
  }
  tp_wait<0>();
  __syncthreads();
  // the K parts meet in shared memory (the stages are free now)
  if (kh > 0) {
    float* red = smem + (((kh - 1) * WM + wm) * 32 + lane) * 17;
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) red[i * 4 + j] = acc[i][j];
  }
  __syncthreads();
  if (kh == 0) {
#pragma unroll
    for (int part = 0; part < KH - 1; ++part) {
      const float* red = smem + ((part * WM + wm) * 32 + lane) * 17;
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] += red[i * 4 + j];
    }
  }
  return kh == 0;
}

}  // namespace n2nmn
