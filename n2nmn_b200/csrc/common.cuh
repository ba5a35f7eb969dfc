// Shared device-side types and helpers for the N2NMN module-network kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace n2nmn {

constexpr float kEps = 1e-12f;   // tf.nn.l2_normalize epsilon (models_clevr/nmn3_modules.py:107)
constexpr int kNodeThreads = 256;
constexpr int kMaxProjNodesPerPass = 8;
// One launch may cover several independent batches ("segments": separate feature / word-vector /
// score buffers of identical shape) so that the kernels see enough work per launch. Images and
// questions are numbered across the segments: g = seg * N + b.
constexpr int kMaxSeg = 16;

// Opcodes mirror enum n2nmn_op in include/n2nmn_b200.h.
enum Op : int {
  OP_SCENE = 0, OP_FIND, OP_FILTER, OP_FIND_SAME_PROPERTY, OP_TRANSFORM, OP_AND, OP_OR,
  OP_EXIST, OP_COUNT, OP_EQUAL_NUM, OP_MORE_NUM, OP_LESS_NUM, OP_SAME_PROPERTY, OP_DESCRIBE,
  NUM_OPS
};

// Weight-set indices.
// Feature-grid contractions done on the tensor cores, one weight matrix [Dk][M] each:
//   PS_FIND     FindModule/conv_image      -> consumed in the fused epilogue (never stored)
//   PS_FSP_IMG  FindSameProperty/conv_image -> stored map m[p,:]
//   PS_*_ATT*   the fc_att layers. fc_att(Σ_p s_p·X[p,:]) = Σ_p s_p·(X[p,:]·W_att + b) because the
//               softmax weights s sum to one, so the per-image map G = X·W_att + b is computed once
//               on the tensor cores and the node kernel only does the 150-row weighted sum.
enum ProjSetId { PS_FIND = 0, PS_FSP_IMG, PS_FSP_ATT, PS_DESC_ATT, PS_SP_ATT0, PS_SP_ATT1,
                 NUM_PROJ_SETS };
enum TextSetId { TS_FIND = 0, TS_FSP, TS_TRANSFORM, TS_SAMEPROP, TS_DESCRIBE, NUM_TEXT_SETS };
enum OutSetId { OS_SAMEPROP = 0, OS_DESCRIBE, NUM_OUT_SETS };
enum ScoreSetId { SS_EXIST = 0, SS_COUNT, SS_EQUAL, SS_MORE, SS_LESS, NUM_SCORE_SETS };
enum EltSetId { ES_FIND = 0, ES_FSP, ES_TRANSFORM, NUM_ELT_SETS };

// One expression-tree node as the kernels see it (48 bytes).
struct NodeRec {
  int32_t op;
  int32_t t, b;      // time index (token position) and question / image index
  int32_t in0, in1;  // arena slots of the attention inputs (-1 if none)
  int32_t out;       // arena slot of the attention output, or score row for answer modules
  int32_t text;      // row in the text-projection buffers (-1 if the module takes no text)
  int32_t aux;       // mbuf slot: FSP conv_image map / Describe fc_att map / SameProperty fc_att_0
                     // (Scene: the bits of pos_val). Schedules with pooled_direct: for Describe /
                     // SameProperty the row of the pooled-feature buffer instead (head_kernel.cuh)
  int32_t aux2;      // mbuf slot: FSP fc_att map / SameProperty fc_att_1 (pooled_direct: 2nd row)
  // Slots of the per-question attention stack the tree kernel keeps in shared memory (live maps
  // of one question; an output may reuse the slot of an input it consumes). -1 = none.
  int32_t s0, s1, so;
};

// Everything the kernels need to know about the model; pointers are device pointers into the
// context-owned packed weight buffer.
struct DevModel {
  int H, W, HW, Dk, feat_pitch, Dt, M, Mp, C, ksize, family;
  const float* feat;        // segment 0: [N*HW, feat_pitch] (Dk valid channels)
  const float* word_vecs;   // segment 0: [T, N, Dt]
  int N, T;                 // images (= questions) per segment, decoder steps
  int num_seg;
  const float* feat_seg[kMaxSeg];
  const float* wv_seg[kMaxSeg];
  // conv_image contraction: original [Dk][M] (fp32 CUDA-core path), bias padded to Mp
  const float* proj_w[NUM_PROJ_SETS];
  const float* proj_b[NUM_PROJ_SETS];
  const float* txt_w[NUM_TEXT_SETS];   // [Dt][Mp] (row pitch Mp, zero padded)
  const float* txt_b[NUM_TEXT_SETS];   // [M]
  const float* elt_w[NUM_ELT_SETS];    // conv_eltwise weights [M]
  const float* elt_b[NUM_ELT_SETS];    // [1]
  const float* conv_k;                 // conv_maps [k*k][Mp] (row pitch Mp, zero padded)
  const float* conv_b;                 // [M]
  // Transform as a quadratic form: [Mp][quad_pitch(ksize)] (conv_quad_kernel in prep.cuh)
  const float* conv_quad;
  const float* out_w[NUM_OUT_SETS];    // fc_eltwise [M][C]
  const float* out_b[NUM_OUT_SETS];
  const float* sc_w[NUM_SCORE_SETS];   // fc_scores [L][C]
  const float* sc_b[NUM_SCORE_SETS];
};

// Text-projection outputs, all [rows][Mp] with zero padding in columns >= M.
struct TextBufs {
  float* tau;    // t·W + b
  float* tauw;   // tau ∘ conv_eltwise weights of the consuming module (or tau)
  float* tau2;   // tau²
  float* tq;     // Transform rows only: [rows][quad_pitch] coefficients (u, Q) of the node
};

// TransformModule (models_clevr/nmn3_modules.py:185-216) as a quadratic form. With the extended
// window w̃ = [the k·k taps of the zero-padded input around the pixel, 1] and the extended filter
// bank K̃ = [conv_maps taps ; conv_maps bias] (n = k·k + 1 rows of M channels):
//     conv output  A_c = Σ_i w̃_i K̃_ic
//     numerator    Σ_c A_c τ_c w2_c     = Σ_i w̃_i u_i,          u_i  = Σ_c K̃_ic w2_c · τ_c
//     denominator  Σ_c (A_c τ_c)²       = Σ_{i<=j} w̃_i w̃_j Q_ij, Q_ij = Σ_c (2-δ_ij) K̃_ic K̃_jc · τ_c²
// so a node costs n + n(n+1)/2 dot products over the channels (done once, batched over the nodes,
// in the text kernel against the precomputed matrix `conv_quad`) plus n + n(n+1)/2 FMAs per
// pixel, instead of k·k·M FMAs per pixel: 7x less arithmetic at k = 5, M = 250, no filter bank
// in shared memory, and exact fp32 (the round-1 stencil ran on TF32 mma fragments).
// Coefficient row of a node: u[0..n), zero padding up to quad_u_pitch (a multiple of 4: a column
// quad of the coefficient product is then either all-u or all-Q), then the upper triangle of Q row
// by row; quad_pitch floats in all.
__host__ __device__ inline int quad_n(int ksize) { return ksize * ksize + 1; }
__host__ __device__ inline int quad_u_pitch(int ksize) { return (quad_n(ksize) + 3) & ~3; }
__host__ __device__ inline int quad_rows(int ksize) {
  return quad_u_pitch(ksize) + quad_n(ksize) * (quad_n(ksize) + 1) / 2;
}
__host__ __device__ inline int quad_pitch(int ksize) { return (quad_rows(ksize) + 3) & ~3; }

// Host-compiled launch tables (built by schedule.cpp, consumed by the kernels).
struct TextGroup { int32_t set, start, count, pad; };   // <= kTextRowsPerCta rows of one text set
constexpr int kTextRowsPerCta = 64;
// One tile of the contraction kernel: 128 rows of one segment against one weight set. row0 = first
// row inside the segment's [N*HW] row axis; pass = which block of <= 8 Find consumers the fused
// epilogue serves.
struct ProjWork { int32_t row0, seg, pass, set; };
// One CTA of the answer-head kernel (head_kernel.cuh): `count` <= kHeadNodesMax root nodes of
// the same type (Describe or SameProperty), listed in head_list[first .. first+count).
struct HeadWork { int32_t first, count, op, pad; };
constexpr int kHeadNodesMax = 16;
// Root nodes per head-kernel CTA: their pooled feature rows (Kp floats each, kept as a TF32 hi and
// a lo plane), the two fc_att outputs [nn][Mp] and 16 KB of scratch share <= 160 KB of shared
// memory (head_smem_layout). 16 for CLEVR, 8 for the stress grid, 4 for VQA.
__host__ __device__ inline int head_smem_floats(int nn, int pitch, int Mp) {
  return 2 * nn * (pitch + 4) + 2 * nn * Mp + 8 * kHeadNodesMax * 32;
}
__host__ __device__ inline int head_nodes_per_cta(int Dk, int Mp) {
  const int kp = (Dk + 31) / 32 * 32;
  return (head_smem_floats(16, kp, Mp) * 4 <= 160 * 1024) ? 16
         : (head_smem_floats(8, kp, Mp) * 4 <= 160 * 1024) ? 8 : 4;
}

// Programmatic dependent launch (PDL): a kernel launched with the programmatic-serialization
// attribute may start while its predecessor in the stream is still running; it must call
// pdl_wait() before touching anything the predecessor writes. pdl_trigger() lets the successor's
// CTAs be scheduled as early as possible.
__device__ __forceinline__ void pdl_trigger() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
__device__ __forceinline__ void pdl_wait() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
}

// word_vecs row of (time t, global image g): segment g / N, row t*N + (g % N)
__device__ __forceinline__ const float* word_vec_row(const DevModel& md, int t, int g) {
  const int seg = g / md.N;
  return md.wv_seg[seg] + ((size_t)t * md.N + (g - seg * md.N)) * md.Dt;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Block-wide reductions for kNodeThreads threads; `red` is >= 32 floats of shared scratch.
// All threads get the result. Contains __syncthreads.
template <int MODE>  // 0 sum, 1 max, 2 min
__device__ __forceinline__ float block_reduce(float v, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (MODE == 0) v = warp_sum(v);
  else if (MODE == 1) v = warp_max(v);
  else v = warp_min(v);
  __syncthreads();   // protect `red` from the previous use
  if (lane == 0) red[warp] = v;
  __syncthreads();
  const int nw = blockDim.x >> 5;
  float r = (lane < nw) ? red[lane] : (MODE == 0 ? 0.f : (MODE == 1 ? -INFINITY : INFINITY));
  if (MODE == 0) r = warp_sum(r);
  else if (MODE == 1) r = warp_max(r);
  else r = warp_min(r);
  return r;
}

}  // namespace n2nmn
