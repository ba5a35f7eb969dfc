// SURVEY.md §8 (f1): the attentional seq2seq layout generator of the reference,
// AttentionSeq2Seq (models_clevr/nmn3_netgen_att.py:46-322; the VQA and SHAPES copies are the
// same code), inference configuration: encoder = embedding + multi-layer LSTM under
// dynamic_rnn (:73-120), decoder = raw_rnn loop with tanh attention over the encoder outputs,
// token scores, the Assembler's validity masks, greedy decoding or teacher forcing (:122-322).
// Produces on the device what nmn3_model.py consumes: predicted_tokens, token_probs (whose logs
// sum to log_seq_prob), neg_entropy, word_vecs and the attention maps.
//
// Data layout (fp32, time-major like the reference's tensors):
//   table_enc [V_txt][4L]    = embedding_mat · W_x of encoder layer 0 (the embedding lookup and
//   table_dec [V_nmn+1][4L]    the layer-0 input product fold into ONE row gather per token;
//                              row V_nmn of table_dec is go_embedding)
//   w_cell[side][l] [(in + L)][4L], b_cell [4L]: the BasicLSTMCell matrix (rows of the layer
//       input, then rows of the recurrent state — TF's order) with the gate columns REGROUPED per
//       8 units (regroup_gates_kernel) so that the cell update happens in the GEMM epilogue;
//   h[l] double buffered [2][N][L] (every CTA reads all of h_prev while others write h_next),
//   c[l] [N][L] in place; enc_out / enc_ht [T][N][L]; atts [T_dec][T_enc][N].
// Kernels: lstm_step (one launch per layer per time step: [x, h_prev]·W on mma.sync m16n8k8 with
// error-compensated TF32 = fp32 parity, 32 or 64 questions x 8 units per CTA, K streamed through
// a cp.async ring, LSTM cell in the epilogue), s2s_gemm (same tile engine: h-transform, attention
// query, table precompute), dec_attn (one CTA per question and step: attention, context vector,
// token scores, validity mask, argmax / forcing, probabilities, entropy, stack-state update),
// word_vecs. The whole call is a chain of (T_enc + layers - 1) + layers·T_dec + 2·T_dec + 3
// dependent launches on the caller's stream (the encoder layers run as a wavefront), linked by
// programmatic dependent launch: each kernel requests what does not depend on its predecessor
// (weights, tables) before griddepcontrol.wait.
// At N = 64 an LSTM launch costs the issue time of its mma.sync instructions (three passes for fp32
// parity; DESIGN.md §4c).
// Dropout (n2nmn_seq2seq_set_dropout): the training scripts' DropoutWrapper on the layers below the
// top one, applied to given uniforms in the LSTM step epilogue (lstm_step_kernel's kDrop variant).
// Training: with n2nmn_seq2seq_set_record on, the forward also stores what the backward pass
// (n2nmn_seq2seq_backward, kernels in seq2seq_bwd.cuh) reads; n2nmn_seq2seq_adam_step runs the
// module network's clip + Adam kernels (optim.cuh) over the flat variable layout.
#include <cuda_runtime.h>

#include <cmath>
#include <algorithm>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "../../include/n2nmn_b200.h"
#include "launch.cuh"
#include "mma_tile.cuh"
#include "optim.cuh"

using namespace n2nmn;

namespace {

constexpr int kMaxLayers = 4;
constexpr int kAttnThreads = 512;
constexpr int kMaxVocabNmn = 64;    // token scores / masks live in one warp's reach
constexpr int kMaxTEnc = 128;

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

// Gate columns regrouped per 8 units: dst column (u/8)*32 + g*8 + u%8 = src column g*L + u
// (gate g = i, j, f, o of unit u). A CTA of the step kernel owns 32 such columns = all four gates
// of 8 units, and inside it n-tile g of the mma holds gate g: one thread's accumulators across
// the four n-tiles are the four gates of its two units.
__global__ void regroup_gates_kernel(const float* __restrict__ src, float* __restrict__ dst,
                                     int rows, int L) {
  const int n = rows * 4 * L;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int r = i / (4 * L), c = i - r * 4 * L;
    const int blk = c >> 5, g = (c >> 3) & 3, u = blk * 8 + (c & 7);
    dst[i] = src[(size_t)r * 4 * L + g * L + u];
  }
}

__global__ void transpose_kernel(const float* __restrict__ src, float* __restrict__ dst, int rows,
                                 int cols) {   // dst[c][r] = src[r][c]
  const int n = rows * cols;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int c = i / rows, r = i - c * rows;
    dst[i] = src[(size_t)r * cols + c];
  }
}

// out[r][c] = Σ_k A[r][k] B[k][c] + bias[c];  grid = (ceil(C/32), ceil(R/(16 WM)))
template <int WM, bool kExact>
__global__ void __launch_bounds__(kMmaThreads)
s2s_gemm_kernel(GemmOperands p, const float* __restrict__ bias, float* __restrict__ out, int ldo) {
  pdl_trigger();
  extern __shared__ __align__(16) float mma_smem[];
  const int row0 = blockIdx.y * 16 * WM, c0 = blockIdx.x * kMmaCols;
  float acc[4][4];
  if (!mma_tile<WM, kExact>(mma_smem, p, row0, c0, acc, [] {})) return;
  const int lane = threadIdx.x & 31, wm = (threadIdx.x >> 5) % WM, g = lane >> 2, tig = lane & 3;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int r = row0 + wm * 16 + g + 8 * hh;
    if (r >= p.R) continue;
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int c = c0 + nt * 8 + 2 * tig + j;
        if (c < p.C) out[(size_t)r * ldo + c] = acc[nt][hh * 2 + j] + (bias ? bias[c] : 0.f);
      }
  }
}

struct LstmStep {
  const float* x;        // [N][L] output of the layer below at this step, or nullptr (layer 0)
  const float* h_prev;   // [N][L]
  const float* w;        // [(L +) L][4L] regrouped: rows of x (layer >= 1) then rows of h_prev
  const float* table;    // layer 0: [V][4L] regrouped input products, else nullptr
  const int32_t* tok;    // layer 0: token of question n at this step
  const float* bias;     // [4L] regrouped
  float* c;              // [N][L] in place
  float* h_out;          // [N][L]
  float* out_seq;        // encoder top layer: encoder_outputs[t] (zero past the end) or nullptr
  const int32_t* seq_len;   // encoder: [N]; nullptr in the decoder (every row live)
  int t, N, L;
  // recording forward only (kRecord): activated gates i, j, f, o [N][4L] in TF's column order,
  // c_t and h_t [N][L] (the carried state past the sequence end)
  float *rec_gates, *rec_c, *rec_h;
  // dropout of this layer's output (kDrop; nullptr on the top layer or with dropout off): this
  // step's uniforms [N][L]; the dropped output [N][L] that the layer above reads as its x; the
  // keep-mask [N][L] (recording forward only)
  const float* drop_u;
  float* drop_out;
  uint8_t* drop_keep;
};

// BasicLSTMCell(forget_bias=1) step (gate order i, j, f, o) with dynamic_rnn's masking: past the
// sequence end the state is carried through and the output is zero (nmn3_netgen_att.py:95-99).
// grid = (4L/32, ceil(N/(16 WM))): one CTA = 8 units x 64 (WM = 4) or 32 (WM = 2) questions; the
// narrow variant is used while it is what it takes to put a CTA on most SMs (N <= 64 at L = 512).
// The encoder runs as a WAVEFRONT: layer l of time step t and layer l-1 of step t+1 only depend on
// the previous launch, so one launch carries up to kMaxLayers steps (blockIdx.z = layer; a slot with
// N == 0 is idle) and the encoder takes T + layers - 1 launches instead of T * layers. With the
// 3-stage ring two CTAs share an SM, which keeps as many bytes in flight as the 5-stage ring of
// the single-step launches.
// kDrop: DropoutWrapper(output_keep_prob=0.5) on the layers below the top (nmn3_netgen_att.py:17-44)
// as tf.nn.dropout computes it: kept iff floor(0.5 + u) = 1 in fp32, a kept element is 2·h. Only the
// copy the layer above reads is dropped; h_out, c, out_seq and the record keep the undropped values.
struct LstmWave { LstmStep s[kMaxLayers]; };
template <int WM, bool kExact, int ST, bool kRecord = false, bool kDrop = false>
__global__ void __launch_bounds__(kMmaThreads) lstm_step_kernel(const LstmWave wave) {
  pdl_trigger();
  const LstmStep& p = wave.s[blockIdx.z];
  if (p.N == 0) return;
  extern __shared__ __align__(16) float mma_smem[];
  const int row0 = blockIdx.y * 16 * WM, c0 = blockIdx.x * kMmaCols;
  const int L = p.L, C = 4 * L;
  GemmOperands op;
  if (p.x != nullptr) { op.a0 = p.x; op.k0 = L; op.lda0 = L; op.a1 = p.h_prev; op.k1 = L; op.lda1 = L; }
  else { op.a0 = p.h_prev; op.k0 = L; op.lda0 = L; op.a1 = nullptr; op.k1 = 0; op.lda1 = 0; }
  op.R = p.N; op.B = p.w; op.ldb = C; op.C = C;
  float acc[4][4];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wm = warp % WM, g = lane >> 2,
            tig = lane & 3;
  // epilogue inputs, requested as soon as the previous step is complete (they ride under the GEMM)
  float gt[2][4][2], c_prev[2][2], h_keep[2][2], du[2][2];
  bool live[2];
  auto prefetch = [&] {
    if (warp / WM != 0) return;
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int n = row0 + wm * 16 + g + 8 * hh;
#pragma unroll
      for (int gate = 0; gate < 4; ++gate) {
        const float2 b2 = *reinterpret_cast<const float2*>(p.bias + c0 + gate * 8 + 2 * tig);
        gt[hh][gate][0] = b2.x; gt[hh][gate][1] = b2.y;
      }
      live[hh] = false;
      if (n >= p.N) continue;
      if (p.table != nullptr) {
        const float* row = p.table + (size_t)p.tok[n] * C + c0 + 2 * tig;
#pragma unroll
        for (int gate = 0; gate < 4; ++gate) {
          const float2 e = *reinterpret_cast<const float2*>(row + gate * 8);
          gt[hh][gate][0] += e.x; gt[hh][gate][1] += e.y;
        }
      }
      live[hh] = p.seq_len == nullptr || p.t < p.seq_len[n];
      const size_t idx = (size_t)n * L + (c0 >> 2) + 2 * tig;
      const float2 cp = *reinterpret_cast<const float2*>(p.c + idx);
      const float2 hp = *reinterpret_cast<const float2*>(p.h_prev + idx);
      c_prev[hh][0] = cp.x; c_prev[hh][1] = cp.y;
      h_keep[hh][0] = hp.x; h_keep[hh][1] = hp.y;
      if constexpr (kDrop)
        if (p.drop_u != nullptr) {
          const float2 u2 = *reinterpret_cast<const float2*>(p.drop_u + idx);
          du[hh][0] = u2.x; du[hh][1] = u2.y;
        }
    }
  };
  if (!mma_tile<WM, kExact, ST>(mma_smem, op, row0, c0, acc, prefetch)) return;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int n = row0 + wm * 16 + g + 8 * hh;
    if (n >= p.N) continue;
    float c_new[2], h_new[2], o_new[2];
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const float gi = gt[hh][0][j] + acc[0][hh * 2 + j], gj = gt[hh][1][j] + acc[1][hh * 2 + j];
      const float gf = gt[hh][2][j] + acc[2][hh * 2 + j], go = gt[hh][3][j] + acc[3][hh * 2 + j];
      const float c2 = c_prev[hh][j] * sigmoidf_(gf + 1.0f) + sigmoidf_(gi) * tanhf(gj);
      const float h2 = tanhf(c2) * sigmoidf_(go);
      c_new[j] = live[hh] ? c2 : c_prev[hh][j];
      h_new[j] = live[hh] ? h2 : h_keep[hh][j];
      o_new[j] = live[hh] ? h2 : 0.f;
    }
    const size_t idx = (size_t)n * L + (c0 >> 2) + 2 * tig;
    *reinterpret_cast<float2*>(p.c + idx) = make_float2(c_new[0], c_new[1]);
    *reinterpret_cast<float2*>(p.h_out + idx) = make_float2(h_new[0], h_new[1]);
    if (p.out_seq != nullptr)
      *reinterpret_cast<float2*>(p.out_seq + idx) = make_float2(o_new[0], o_new[1]);
    if constexpr (kDrop)
      if (p.drop_u != nullptr) {
        const bool k0 = 0.5f + du[hh][0] >= 1.f, k1 = 0.5f + du[hh][1] >= 1.f;
        *reinterpret_cast<float2*>(p.drop_out + idx) =
            make_float2(k0 ? 2.f * h_new[0] : 0.f, k1 ? 2.f * h_new[1] : 0.f);
        if constexpr (kRecord)
          *reinterpret_cast<uchar2*>(p.drop_keep + idx) = make_uchar2(k0 ? 1 : 0, k1 ? 1 : 0);
      }
    if constexpr (kRecord) {
      const size_t gi0 = (size_t)n * C + (c0 >> 2) + 2 * tig;
      float2 act[4];
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const float a0 = sigmoidf_(gt[hh][0][j] + acc[0][hh * 2 + j]);
        const float a1 = tanhf(gt[hh][1][j] + acc[1][hh * 2 + j]);
        const float a2 = sigmoidf_(gt[hh][2][j] + acc[2][hh * 2 + j] + 1.0f);
        const float a3 = sigmoidf_(gt[hh][3][j] + acc[3][hh * 2 + j]);
        (j == 0 ? act[0].x : act[0].y) = a0; (j == 0 ? act[1].x : act[1].y) = a1;
        (j == 0 ? act[2].x : act[2].y) = a2; (j == 0 ? act[3].x : act[3].y) = a3;
      }
#pragma unroll
      for (int gate = 0; gate < 4; ++gate)
        *reinterpret_cast<float2*>(p.rec_gates + gi0 + (size_t)gate * L) = act[gate];
      *reinterpret_cast<float2*>(p.rec_c + idx) = make_float2(c_new[0], c_new[1]);
      *reinterpret_cast<float2*>(p.rec_h + idx) = make_float2(h_new[0], h_new[1]);
    }
  }
}

struct AttnStep {
  const float* q;         // [N][L] h_top · W_a + b_a
  const float* h_top;     // [N][L]
  const float* enc_ht;    // [T][N][L]
  const float* enc_out;   // [T][N][L]
  const float* v;         // [L]
  const float* wy_t;      // [V][2L] token_prediction weights, transposed
  const float* by;        // [V]
  const int32_t* seq_len; // [N]
  const int32_t* P;       // [V][3]
  const int32_t* W;       // [3][V][4]
  const int32_t* b;       // [V][4]
  int32_t* X;             // [N][3] decoding state (nmn3_netgen_att.py:288-293)
  const int32_t* gt;      // [N] this step's ground-truth tokens or nullptr
  const float* u;         // [N] this step's uniform numbers (decoder_sampling) or nullptr
  int32_t* tokens;        // [N] this step's predicted tokens (row t of predicted_tokens)
  int32_t* cur_tok;       // [N] input token of the next step
  float* probs;           // [N] row t of token_probs
  float* neg_entropy;     // [N] accumulated
  float* atts;            // [T][N] this step's attention
  int T, N, L, V;
  // recording forward only (kRecord): context vector [N][L], token scores [N][V], validity bits
  // [N][2], attention [T][N], chosen token [N]
  float *rec_d2, *rec_sc, *rec_att;
  int32_t *rec_valid, *rec_tok;
};

// One CTA per question: nmn3_netgen_att.py:205-293 for one decoding step. Everything that does
// not depend on the previous kernel (W_y^T, v, b_y and the Assembler tables) is staged in shared
// memory BEFORE griddepcontrol.wait, i.e. under the tail of the kernels before it. The step is a
// chain of short phases, each bound by the latency of its global loads, so every phase keeps as
// many independent 16-byte loads in flight per thread as registers allow.
__host__ __device__ inline size_t attn_smem_floats(int L, int T, int V) {
  const int part = L > 4 * kAttnThreads ? L : 4 * kAttnThreads;
  return (size_t)V * 2 * L + 4 * L + part + ((T + 3) & ~3) + 2 * ((V + 3) & ~3) + 3 * V + 12 * V +
         4 * V + 8;
}
template <bool kRecord = false>
__global__ void __launch_bounds__(kAttnThreads) dec_attn_kernel(AttnStep p) {
  pdl_trigger();
  extern __shared__ __align__(16) float sm[];
  const int n = blockIdx.x, L = p.L, T = p.T, V = p.V;
  const int part = L > 4 * kAttnThreads ? L : 4 * kAttnThreads;
  float* s_wy = sm;                    // [V][2L]
  float* s_x = s_wy + (size_t)V * 2 * L;   // [2L] = [h_top, d2]
  float* s_q = s_x + 2 * L;            // [L]
  float* s_v = s_q + L;                // [L]
  float* s_part = s_v + L;             // [G][L] partial context vectors
  float* s_att = s_part + part;        // [T]
  float* s_sc = s_att + ((T + 3) & ~3);   // [V] scores
  float* s_by = s_sc + ((V + 3) & ~3);    // [V]
  int32_t* s_P = reinterpret_cast<int32_t*>(s_by + ((V + 3) & ~3));   // [V][3]
  int32_t* s_W = s_P + 3 * V;          // [3][V][4]
  int32_t* s_b = s_W + 12 * V;         // [V][4]
  int32_t* s_valid = s_b + 4 * V;      // [2]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, nw = kAttnThreads / 32;
  for (int i = tid; i < V * 2 * L / 4; i += kAttnThreads) tp_cp16(s_wy + 4 * i, p.wy_t + 4 * i);
  tp_commit();
  for (int d = tid; d < L; d += kAttnThreads) s_v[d] = p.v[d];
  for (int i = tid; i < V; i += kAttnThreads) s_by[i] = p.by[i];
  for (int i = tid; i < 3 * V; i += kAttnThreads) s_P[i] = p.P[i];
  for (int i = tid; i < 12 * V; i += kAttnThreads) s_W[i] = p.W[i];
  for (int i = tid; i < 4 * V; i += kAttnThreads) s_b[i] = p.b[i];
  pdl_wait();
  for (int d = tid; d < L; d += kAttnThreads) {
    s_x[d] = p.h_top[(size_t)n * L + d];
    s_q[d] = p.q[(size_t)n * L + d];
  }
  __syncthreads();
  const int ncol = L >> 2;
  const size_t tstride = (size_t)p.N * L;
  // att_raw[te] = Σ_d tanh(q + enc_ht[te]) v   (:208-212): a warp takes 4 time steps at once
  for (int tb = warp * 4; tb < T; tb += nw * 4) {
    float s[4] = {0.f, 0.f, 0.f, 0.f};
    const float* ht = p.enc_ht + (size_t)tb * tstride + (size_t)n * L;
#pragma unroll 2
    for (int c4 = lane; c4 < ncol; c4 += 32) {
      const float4 q4 = reinterpret_cast<const float4*>(s_q)[c4];
      const float4 v4 = reinterpret_cast<const float4*>(s_v)[c4];
      float4 h4[4];
#pragma unroll
      for (int i = 0; i < 4; ++i)
        h4[i] = tb + i < T ? __ldg(reinterpret_cast<const float4*>(ht + i * tstride) + c4)
                           : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int i = 0; i < 4; ++i)
        s[i] += tanhf(q4.x + h4[i].x) * v4.x + tanhf(q4.y + h4[i].y) * v4.y +
                tanhf(q4.z + h4[i].z) * v4.z + tanhf(q4.w + h4[i].w) * v4.w;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
      for (int o = 16; o; o >>= 1) s[i] += __shfl_xor_sync(0xffffffffu, s[i], o);
      if (lane == 0 && tb + i < T) s_att[tb + i] = s[i];
    }
  }
  __syncthreads();
  // softmax over ALL time steps, then mask by the sequence length and renormalise (:213-216)
  if (warp == 0) {
    float m = -INFINITY;
    for (int te = lane; te < T; te += 32) m = fmaxf(m, s_att[te]);
#pragma unroll
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float s = 0.f;
    for (int te = lane; te < T; te += 32) { const float e = expf(s_att[te] - m); s_att[te] = e; s += e; }
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const int len = p.seq_len[n];
    float s2 = 0.f;
    for (int te = lane; te < T; te += 32) {
      const float a = te < len ? s_att[te] / s : 0.f;
      s_att[te] = a; s2 += a;
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    for (int te = lane; te < T; te += 32) {
      const float a = s_att[te] / s2;
      s_att[te] = a;
      p.atts[(size_t)te * p.N + n] = a;
      if constexpr (kRecord) p.rec_att[(size_t)te * p.N + n] = a;
    }
  } else if (warp == 1) {
    // validity of every token from the decoding state (:8-11); all ones under forcing (:230-233)
    const int32_t x0 = p.X[n * 3], x1 = p.X[n * 3 + 1], x2 = p.X[n * 3 + 2];
    uint32_t lo = 0, hi = 0;
    for (int base = 0; base < V; base += 32) {
      const int vv = base + lane;
      bool ok = vv < V;
      if (ok && p.gt == nullptr) {
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const int32_t lhs = x0 * s_W[(0 * V + vv) * 4 + c] + x1 * s_W[(1 * V + vv) * 4 + c] +
                              x2 * s_W[(2 * V + vv) * 4 + c];
          ok = ok && (lhs - s_b[vv * 4 + c] >= 0);
        }
      }
      const uint32_t bal = __ballot_sync(0xffffffffu, ok);
      if (base == 0) lo = bal; else hi = bal;
    }
    if (lane == 0) { s_valid[0] = (int32_t)lo; s_valid[1] = (int32_t)hi; }
    if constexpr (kRecord)
      if (lane == 0) { p.rec_valid[2 * n] = (int32_t)lo; p.rec_valid[2 * n + 1] = (int32_t)hi; }
  }
  __syncthreads();
  // d2 = Σ_te att[te] encoder_outputs[te]   (:218): G groups of threads split the time steps of
  // each 4-channel column, partial sums meet in shared memory
  {
    const int G = ncol >= kAttnThreads ? 1 : kAttnThreads / ncol;
    for (int item = tid; item < ncol * G; item += kAttnThreads) {
      const int c4 = item % ncol, gi = item / ncol;
      const float4* eo = reinterpret_cast<const float4*>(p.enc_out + (size_t)n * L) + c4;
      float4 acc4 = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 8
      for (int te = gi; te < T; te += G) {
        const float4 e = __ldg(eo + (size_t)te * (tstride >> 2));
        const float a = s_att[te];
        acc4.x += a * e.x; acc4.y += a * e.y; acc4.z += a * e.z; acc4.w += a * e.w;
      }
      reinterpret_cast<float4*>(s_part + (size_t)gi * L)[c4] = acc4;
    }
    __syncthreads();
    for (int d = tid; d < L; d += kAttnThreads) {
      float s = 0.f;
      for (int gi = 0; gi < G; ++gi) s += s_part[(size_t)gi * L + d];
      s_x[L + d] = s;
      if constexpr (kRecord) p.rec_d2[(size_t)n * L + d] = s;
    }
  }
  tp_wait<0>();
  __syncthreads();
  // token_scores = [h_top, d2] · W_y + b_y   (:221-223)
  for (int vv = warp; vv < V; vv += nw) {
    const float4* wr = reinterpret_cast<const float4*>(s_wy + (size_t)vv * 2 * L);
    float s = 0.f;
    for (int k4 = lane; k4 < 2 * ncol; k4 += 32) {
      const float4 x4 = reinterpret_cast<const float4*>(s_x)[k4], w4 = wr[k4];
      s += x4.x * w4.x + x4.y * w4.y + x4.z * w4.z + x4.w * w4.w;
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) s_sc[vv] = s + s_by[vv];
    if constexpr (kRecord)
      if (lane == 0) p.rec_sc[(size_t)n * V + vv] = s + s_by[vv];
  }
  __syncthreads();
  if (warp == 0) {   // lane handles tokens lane and lane + 32 (V <= 64)
    const uint32_t vlo = (uint32_t)s_valid[0], vhi = (uint32_t)s_valid[1];
    const int v0 = lane, v1 = lane + 32;
    const bool in0 = v0 < V, in1 = v1 < V;
    const bool ok0 = in0 && ((vlo >> lane) & 1), ok1 = in1 && ((vhi >> lane) & 1);
    const float sc0 = in0 ? s_sc[v0] : -INFINITY, sc1 = in1 ? s_sc[v1] : -INFINITY;
    float mx = fmaxf(sc0, sc1);
#pragma unroll
    for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    // greedy token: invalid scores are replaced by (global min - 1) before the argmax (:259-261),
    // i.e. the first best VALID token, or token 0 if none is valid
    float best = ok0 ? sc0 : -INFINITY;
    int pred = ok0 ? v0 : 0x7fffffff;
    if (ok1 && sc1 > best) { best = sc1; pred = v1; }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int op = __shfl_xor_sync(0xffffffffu, pred, o);
      if (ob > best || (ob == best && op < pred)) { best = ob; pred = op; }
    }
    if (pred == 0x7fffffff) pred = 0;
    if (p.u != nullptr) {
      // decoder_sampling (:234-256): one draw from softmax(scores - 50·invalid) by inverse CDF
      // over the tokens in vocabulary order — the first token whose cumulative probability
      // exceeds u — kept when it is valid, else the greedy token above
      const float z0 = in0 ? sc0 - (ok0 ? 0.f : 50.f) : -INFINITY;
      const float z1 = in1 ? sc1 - (ok1 ? 0.f : 50.f) : -INFINITY;
      float zm = fmaxf(z0, z1);
#pragma unroll
      for (int o = 16; o; o >>= 1) zm = fmaxf(zm, __shfl_xor_sync(0xffffffffu, zm, o));
      float c0 = in0 ? expf(z0 - zm) : 0.f, c1 = in1 ? expf(z1 - zm) : 0.f;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {   // inclusive scans over the lanes
        const float t0 = __shfl_up_sync(0xffffffffu, c0, o), t1 = __shfl_up_sync(0xffffffffu, c1, o);
        if (lane >= o) { c0 += t0; c1 += t1; }
      }
      c1 += __shfl_sync(0xffffffffu, c0, 31);
      const float thr = p.u[n] * __shfl_sync(0xffffffffu, c1, 31);
      const uint32_t m0 = __ballot_sync(0xffffffffu, in0 && c0 > thr);
      const uint32_t m1 = __ballot_sync(0xffffffffu, in1 && c1 > thr);
      const int samp = m0 ? __ffs(m0) - 1 : (m1 ? 31 + __ffs(m1) : V - 1);
      if (((samp < 32 ? vlo >> samp : vhi >> (samp - 32)) & 1u) != 0u) pred = samp;
    }
    if (p.gt != nullptr) pred = p.gt[n];   // :264-266
    const float e0 = in0 ? expf(sc0 - mx) : 0.f, e1 = in1 ? expf(sc1 - mx) : 0.f;
    float se = e0 + e1;
#pragma unroll
    for (int o = 16; o; o >>= 1) se += __shfl_xor_sync(0xffffffffu, se, o);
    const float a0 = ok0 ? e0 / se : 0.f, a1 = ok1 ? e1 / se : 0.f;      // :270
    float sv = a0 + a1;
#pragma unroll
    for (int o = 16; o; o >>= 1) sv += __shfl_xor_sync(0xffffffffu, sv, o);
    const float p0 = a0 / sv, p1 = a1 / sv;                               // :272
    float ent = 0.f;
    if (in0) ent += p0 * logf(fmaxf(1e-5f, p0 + (ok0 ? 0.f : 1.f)));      // :283-285
    if (in1) ent += p1 * logf(fmaxf(1e-5f, p1 + (ok1 ? 0.f : 1.f)));
#pragma unroll
    for (int o = 16; o; o >>= 1) ent += __shfl_xor_sync(0xffffffffu, ent, o);
    const float pp = __shfl_sync(0xffffffffu, pred < 32 ? p0 : p1, pred & 31);
    if (lane == 0) {
      p.probs[n] = pp;                                                    // :281
      p.neg_entropy[n] += ent;
      p.X[n * 3] += s_P[pred * 3];                                        // :288-289
      p.X[n * 3 + 1] += s_P[pred * 3 + 1];
      p.X[n * 3 + 2] += s_P[pred * 3 + 2];
      p.tokens[n] = pred;
      p.cur_tok[n] = pred;
      if constexpr (kRecord) p.rec_tok[n] = pred;
    }
  }
}

// word_vecs[td][n][:] = Σ_te atts[td][te][n] · embedding_mat[input_seq[te][n]]   (:312)
// grid = (N, T_dec)
__global__ void word_vecs_kernel(const float* __restrict__ atts, const int32_t* __restrict__ seq,
                                 const float* __restrict__ emb, float* __restrict__ out, int T,
                                 int N, int E) {
  const int n = blockIdx.x, td = blockIdx.y;
  extern __shared__ float s_a[];   // [T] weights then [T] token ids (as int)
  int32_t* s_tok = reinterpret_cast<int32_t*>(s_a + T);
  for (int te = threadIdx.x; te < T; te += blockDim.x) {
    s_a[te] = atts[((size_t)td * T + te) * N + n];
    s_tok[te] = seq[(size_t)te * N + n];
  }
  __syncthreads();
  for (int e = threadIdx.x; e < E; e += blockDim.x) {
    float s = 0.f;
    for (int te = 0; te < T; ++te) s += s_a[te] * emb[(size_t)s_tok[te] * E + e];
    out[((size_t)td * N + n) * E + e] = s;
  }
}

__global__ void init_state_kernel(int32_t* X, int32_t* cur_tok, float* neg_entropy, int N,
                                  int T_dec, int go_row) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  X[n * 3] = 0; X[n * 3 + 1] = 0; X[n * 3 + 2] = T_dec;   // :293
  cur_tok[n] = go_row;
  neg_entropy[n] = 0.f;
}

struct S2SVar {
  std::string name;
  std::vector<int64_t> shape;
  float* dev;       // raw copy as given (TF layout), inside the context's flat variable buffer
  size_t count;
  int64_t offset;   // in the flat layout (16-byte aligned)
  bool loaded;
};

}  // namespace

#include "seq2seq_bwd.cuh"

struct n2nmn_seq2seq {
  n2nmn_seq2seq_config cfg;
  int num_sms = 0;
  std::vector<void*> allocs;   // every device buffer below (dmalloc), freed by destroy
  std::vector<S2SVar> vars;
  bool dirty = true, tables_set = false;
  const float* sample_u = nullptr;   // [T_decoder][N] uniforms of the following forward calls
  // dropout uniforms of the following forward calls (n2nmn_seq2seq_set_dropout), per side
  // [T][layers-1][N][L]; nullptr = no dropout on that side
  const float* drop_u[2] = {};
  // derived weights
  float *table_enc = nullptr, *table_dec = nullptr, *dec_rows = nullptr;   // dec_rows = [emb; go]
  float* w_cell[2][kMaxLayers] = {};   // interleaved full matrices [(in+L)][4L]
  float* b_cell[2][kMaxLayers] = {};
  float* wy_t = nullptr;
  // state / workspaces
  float* h[kMaxLayers][2] = {};
  float* c[kMaxLayers] = {};
  float *enc_out = nullptr, *enc_ht = nullptr, *q = nullptr, *atts = nullptr;
  int32_t *X = nullptr, *cur_tok = nullptr, *P = nullptr, *W = nullptr, *b = nullptr;
  int64_t launches = 0;
  float* wstore = nullptr;   // every variable, flat layout (n2nmn_seq2seq_flat_offset)
  int64_t flat_size = 0;
  // recording forward (n2nmn_seq2seq_set_record): what the backward pass reads. Slots are sized
  // for max_batch and T_encoder; inside a (side, layer) block the rows are [t][N] with the
  // recorded N, so that all steps of a layer form one [T·N] matrix.
  bool record = false;
  bool rec_ready = false;    // workspace allocated (all of it)
  bool rec_valid = false;    // the last forward recorded and no weight changed since
  int rec_N = 0, rec_T = 0;
  float *rec_gates[2] = {}, *rec_c[2] = {}, *rec_h[2] = {};   // [layers][T_cap][N][4L | L]
  float *rec_q = nullptr, *rec_d2 = nullptr, *rec_sc = nullptr, *rec_att = nullptr;
  int32_t *rec_valid_bits = nullptr, *rec_tok = nullptr, *rec_seq = nullptr, *rec_len = nullptr;
  // dropout (allocated on first use): the dropped outputs the layer above reads, one slot per
  // step (the encoder wavefront writes step t+1 of a layer while the layer above reads step t; the
  // backward reads them as that layer's x), and the recording forward's keep-masks;
  // [layers-1][T_cap][max_batch][L] each, rows [t][N] as in the recording
  float* drop_x[2] = {};
  uint8_t* drop_keep[2] = {};
  bool rec_drop[2] = {};     // the recorded forward ran dropout on that side
  // backward workspace, allocated with the recording
  float *dgates[2] = {};     // [layers][T_cap][N][4L]
  float *d_h[4] = {};        // drec, dup, hcarry, dc: [layers][N][L] each
  float *ds = nullptr, *dh_top = nullptr, *dq = nullptr, *dv_part = nullptr;
  float *d_enc_out = nullptr, *d_enc_ht = nullptr, *dx0 = nullptr;
  float *w_t[2][kMaxLayers] = {};   // transposed cell matrices [4L][in + L] (TF layout)
  float *wa_t = nullptr, *wh_t = nullptr;
  bool bwd_dirty = true;     // transposes stale
  VarSeg* d_segs = nullptr;  // Adam segment table, ready with d_sumsq
  float* d_sumsq = nullptr;
  bool segs_ready = false;
  int var(const std::string& n) const {
    for (size_t i = 0; i < vars.size(); ++i) if (vars[i].name == n) return (int)i;
    return -1;
  }
  const float* v(const std::string& n) const { return vars[var(n)].dev; }
};

namespace {

// The kernels that call griddepcontrol.wait (s2s_gemm, lstm_step, dec_attn, s2s_bwd_gemm,
// s2s_cell_bwd) launch with programmatic dependent launch; every other launch is plain.
constexpr LaunchAttrs kPdl{true};

// Tile geometry of the mma_tile kernels for R rows, C columns and nz slots: 32-row tiles (WM = 2)
// while 64-row tiles would leave SMs without a CTA.
struct Tiles {
  bool narrow;
  dim3 grid;
};
Tiles tiles(int R, int C, int nz, int num_sms) {
  const int cb = (C + kMmaCols - 1) / kMmaCols;
  const bool narrow = R > 16 && cb * nz * ((R + 63) / 64) < num_sms;
  return {narrow, dim3(cb, narrow ? (R + 31) / 32 : (R + 63) / 64, nz)};
}

// Kernel variants, chosen in one place for the attribute setup and the launch.
auto gemm_variant(bool narrow, bool exact) {
  if (narrow) return exact ? &s2s_gemm_kernel<2, true> : &s2s_gemm_kernel<2, false>;
  return exact ? &s2s_gemm_kernel<4, true> : &s2s_gemm_kernel<4, false>;
}
auto bwd_gemm_variant(bool narrow, bool exact) {
  if (narrow) return exact ? &s2s_bwd_gemm_kernel<2, true> : &s2s_bwd_gemm_kernel<2, false>;
  return exact ? &s2s_bwd_gemm_kernel<4, true> : &s2s_bwd_gemm_kernel<4, false>;
}
// 64-row tiles run the 3-stage ring; 32-row tiles the 5-stage ring, or the 3-stage one where two
// CTAs share an SM (the encoder wavefront)
template <bool kRec, bool kDrop>
auto lstm_variant(bool narrow, bool shared_sm, bool exact) {
  if (!narrow)
    return exact ? &lstm_step_kernel<4, true, 3, kRec, kDrop> : &lstm_step_kernel<4, false, 3, kRec, kDrop>;
  if (shared_sm)
    return exact ? &lstm_step_kernel<2, true, 3, kRec, kDrop> : &lstm_step_kernel<2, false, 3, kRec, kDrop>;
  return exact ? &lstm_step_kernel<2, true, 5, kRec, kDrop> : &lstm_step_kernel<2, false, 5, kRec, kDrop>;
}
auto lstm_variant(bool narrow, bool shared_sm, bool exact, bool rec, bool drop) {
  if (drop)
    return rec ? lstm_variant<true, true>(narrow, shared_sm, exact)
               : lstm_variant<false, true>(narrow, shared_sm, exact);
  return rec ? lstm_variant<true, false>(narrow, shared_sm, exact)
             : lstm_variant<false, false>(narrow, shared_sm, exact);
}
auto cell_bwd_variant(bool drop) { return drop ? &s2s_cell_bwd_kernel<true> : &s2s_cell_bwd_kernel<false>; }
size_t lstm_smem(bool narrow, bool shared_sm) {
  return mma_smem_bytes(narrow ? 2 : 4, narrow && !shared_sm ? 5 : 3);
}

GemmOperands gemm_ops(const float* A, int lda, int R, int K, const float* B, int ldb, int C) {
  GemmOperands op;
  op.a0 = A; op.k0 = K; op.lda0 = lda; op.a1 = nullptr; op.k1 = 0; op.lda1 = 0;
  op.R = R; op.B = B; op.ldb = ldb; op.C = C;
  return op;
}

int launch_gemm(n2nmn_seq2seq* s, cudaStream_t st, const float* A, int lda, int R, int K,
                const float* B, int ldb, int C, const float* bias, float* out, int ldo,
                bool force_exact = false) {
  const Tiles t = tiles(R, C, 1, s->num_sms);
  const bool exact = !(s->cfg.flags & N2NMN_SEQ2SEQ_FLAG_TF32) || force_exact;
  return launch(s->launches, gemm_variant(t.narrow, exact), t.grid, kMmaThreads,
                mma_smem_bytes(t.narrow ? 2 : 4), st, kPdl, gemm_ops(A, lda, R, K, B, ldb, C), bias,
                out, ldo);
}

std::string cell_prefix(int side, int l) {
  return std::string(side == 0 ? "encoder" : "decoder") + "/lstm/multi_rnn_cell/cell_" +
         std::to_string(l) + "/basic_lstm_cell/";
}

// Re-derive the packed weights after a set_weight (once; on the caller's stream).
int prepare(n2nmn_seq2seq* s, cudaStream_t st) {
  const auto& g = s->cfg;
  const int L = g.lstm_dim, C = 4 * L;
  for (auto& v : s->vars)
    if (!v.loaded) return fail_with(N2NMN_ERR_STATE, "seq2seq weight not set: " + v.name);
  for (int side = 0; side < 2; ++side) {
    for (int l = 0; l < g.num_layers; ++l) {
      const int in = l == 0 ? (side == 0 ? g.embed_dim_txt : g.embed_dim_nmn) : L;
      TRY(launch(s->launches, regroup_gates_kernel, s->num_sms, 256, 0, st, {},
                 s->v(cell_prefix(side, l) + "weights"), s->w_cell[side][l], in + L, L));
      TRY(launch(s->launches, regroup_gates_kernel, 8, 256, 0, st, {},
                 s->v(cell_prefix(side, l) + "biases"), s->b_cell[side][l], 1, L));
    }
  }
  CUDA_TRY(cudaMemcpyAsync(s->dec_rows, s->v("decoder/embedding_mat"),
                           sizeof(float) * g.num_vocab_nmn * g.embed_dim_nmn,
                           cudaMemcpyDeviceToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(s->dec_rows + (size_t)g.num_vocab_nmn * g.embed_dim_nmn,
                           s->v("decoder/go_embedding"), sizeof(float) * g.embed_dim_nmn,
                           cudaMemcpyDeviceToDevice, st));
  TRY(launch_gemm(s, st, s->v("encoder/embedding_mat"), g.embed_dim_txt, g.num_vocab_txt,
                  g.embed_dim_txt, s->w_cell[0][0], C, C, nullptr, s->table_enc, C, true));
  TRY(launch_gemm(s, st, s->dec_rows, g.embed_dim_nmn, g.num_vocab_nmn + 1, g.embed_dim_nmn,
                  s->w_cell[1][0], C, C, nullptr, s->table_dec, C, true));
  TRY(launch(s->launches, transpose_kernel, 64, 256, 0, st, {},
             s->v("decoder/token_prediction/weights"), s->wy_t, 2 * L, g.num_vocab_nmn));
  s->dirty = false;
  return N2NMN_OK;
}

// Every device buffer of the context is allocated here and recorded for n2nmn_seq2seq_destroy.
template <class T>
cudaError_t dmalloc(n2nmn_seq2seq* s, T** p, size_t n) {
  const cudaError_t e = cudaMalloc(reinterpret_cast<void**>(p), n * sizeof(T));
  if (e == cudaSuccess) s->allocs.push_back(*p);
  return e;
}
// Lazy workspaces: a retry after a failed attempt allocates only what is still missing.
template <class T>
cudaError_t dmalloc_once(n2nmn_seq2seq* s, T** p, size_t n) {
  return *p ? cudaSuccess : dmalloc(s, p, n);
}

int t_cap(const n2nmn_seq2seq* s, int side) { return side == 0 ? s->cfg.T_encoder : s->cfg.T_decoder; }
// recorded rows of (side, layer) from step t on, with the recorded batch size N
float* rec_gates_at(n2nmn_seq2seq* s, int side, int l, int t, int N) {
  const size_t L4 = 4 * (size_t)s->cfg.lstm_dim;
  return s->rec_gates[side] + ((size_t)l * t_cap(s, side) * s->cfg.max_batch + (size_t)t * N) * L4;
}
float* dgates_at(n2nmn_seq2seq* s, int side, int l, int t, int N) {
  const size_t L4 = 4 * (size_t)s->cfg.lstm_dim;
  return s->dgates[side] + ((size_t)l * t_cap(s, side) * s->cfg.max_batch + (size_t)t * N) * L4;
}
template <class T>
T* rec_state_at(n2nmn_seq2seq* s, T* base, int side, int l, int t, int N) {
  const size_t L = s->cfg.lstm_dim;
  return base + ((size_t)l * t_cap(s, side) * s->cfg.max_batch + (size_t)t * N) * L;
}

// The recording and backward workspace, allocated on first use. Ready only when all of it is:
// a failed attempt leaves rec_ready false and the next call allocates what is still missing.
int ensure_record(n2nmn_seq2seq* s) {
  if (s->rec_ready) return N2NMN_OK;
  const auto& g = s->cfg;
  const size_t L = g.lstm_dim, N = g.max_batch, NL = g.num_layers, Td = g.T_decoder;
  const size_t Te = g.T_encoder, Vn = g.num_vocab_nmn, Vp = (Vn + 3) & ~size_t(3);
  for (int side = 0; side < 2; ++side) {
    const size_t rows = NL * (size_t)t_cap(s, side) * N;
    CUDA_TRY(dmalloc_once(s, &s->rec_gates[side], rows * 4 * L));
    CUDA_TRY(dmalloc_once(s, &s->rec_c[side], rows * L));
    CUDA_TRY(dmalloc_once(s, &s->rec_h[side], rows * L));
    CUDA_TRY(dmalloc_once(s, &s->dgates[side], rows * 4 * L));
    for (size_t l = 0; l < NL; ++l) {
      const size_t in = l == 0 ? (side == 0 ? g.embed_dim_txt : g.embed_dim_nmn) : L;
      CUDA_TRY(dmalloc_once(s, &s->w_t[side][l], 4 * L * (in + L)));
    }
  }
  CUDA_TRY(dmalloc_once(s, &s->rec_q, Td * N * L));
  CUDA_TRY(dmalloc_once(s, &s->rec_d2, Td * N * L));
  CUDA_TRY(dmalloc_once(s, &s->rec_sc, Td * N * Vn));
  CUDA_TRY(dmalloc_once(s, &s->rec_att, Td * Te * N));
  CUDA_TRY(dmalloc_once(s, &s->rec_valid_bits, Td * N * 2));
  CUDA_TRY(dmalloc_once(s, &s->rec_tok, Td * N));
  CUDA_TRY(dmalloc_once(s, &s->rec_seq, Te * N));
  CUDA_TRY(dmalloc_once(s, &s->rec_len, N));
  for (auto*& p : s->d_h) CUDA_TRY(dmalloc_once(s, &p, NL * N * L));
  CUDA_TRY(dmalloc_once(s, &s->ds, Td * N * Vp));
  CUDA_TRY(dmalloc_once(s, &s->dh_top, Td * N * L));
  CUDA_TRY(dmalloc_once(s, &s->dq, Td * N * L));
  CUDA_TRY(dmalloc_once(s, &s->dv_part, N * L));
  CUDA_TRY(dmalloc_once(s, &s->d_enc_out, Te * N * L));
  CUDA_TRY(dmalloc_once(s, &s->d_enc_ht, Te * N * L));
  const size_t E = std::max(g.embed_dim_txt * Te, g.embed_dim_nmn * Td);
  CUDA_TRY(dmalloc_once(s, &s->dx0, E * N));
  CUDA_TRY(dmalloc_once(s, &s->wa_t, L * L));
  CUDA_TRY(dmalloc_once(s, &s->wh_t, L * L));
  s->rec_ready = true;
  return N2NMN_OK;
}

// The dropout buffers of `side`, allocated on the first forward that drops there; the keep-masks
// on the first such forward that records.
int ensure_dropout(n2nmn_seq2seq* s, int side, bool rec) {
  const auto& g = s->cfg;
  const size_t n = (size_t)(g.num_layers - 1) * t_cap(s, side) * g.max_batch * g.lstm_dim;
  CUDA_TRY(dmalloc_once(s, &s->drop_x[side], n));
  if (rec) CUDA_TRY(dmalloc_once(s, &s->drop_keep[side], n));
  return N2NMN_OK;
}

// ---- backward helpers ---------------------------------------------------------------------------
// The transposed matrices of the backward products, re-made after a weight changed.
int prepare_backward(n2nmn_seq2seq* s, cudaStream_t st) {
  const auto& g = s->cfg;
  const int L = g.lstm_dim;
  for (int side = 0; side < 2; ++side)
    for (int l = 0; l < g.num_layers; ++l) {
      const int in = l == 0 ? (side == 0 ? g.embed_dim_txt : g.embed_dim_nmn) : L;
      TRY(launch(s->launches, transpose_kernel, s->num_sms, 256, 0, st, {},
                 s->v(cell_prefix(side, l) + "weights"), s->w_t[side][l], in + L, 4 * L));
    }
  TRY(launch(s->launches, transpose_kernel, 64, 256, 0, st, {},
             s->v("decoder/att_prediction/weights"), s->wa_t, L, L));
  TRY(launch(s->launches, transpose_kernel, 64, 256, 0, st, {},
             s->v("encoder/encoder_h_transform/weights"), s->wh_t, L, L));
  s->bwd_dirty = false;
  return N2NMN_OK;
}

// One launch of s2s_bwd_gemm_kernel over `nz` slots; exact = the error-compensated 3xTF32 path.
int launch_bwd_gemm(n2nmn_seq2seq* s, cudaStream_t st, const BwdGemmWave& w, int nz) {
  int R = 0, C = 0;
  for (int z = 0; z < nz; ++z) { R = std::max(R, w.s[z].op.R); C = std::max(C, w.s[z].op.C); }
  const Tiles t = tiles(R, C, nz, s->num_sms);
  const bool exact = !(s->cfg.flags & N2NMN_SEQ2SEQ_FLAG_TF32);
  return launch(s->launches, bwd_gemm_variant(t.narrow, exact), t.grid, kMmaThreads,
                mma_smem_bytes(t.narrow ? 2 : 4), st, kPdl, w);
}

BwdGemm bwd_gemm(GemmOperands op, float* out0, int ldo0, float* out1, int ldo1, int split,
                 bool accumulate) {
  BwdGemm b;
  b.op = op; b.out0 = out0; b.ldo0 = ldo0; b.out1 = out1; b.ldo1 = ldo1; b.split = split;
  b.accumulate = accumulate ? 1 : 0;
  return b;
}

int one_gemm(n2nmn_seq2seq* s, cudaStream_t st, const BwdGemm& g) {
  BwdGemmWave w;
  std::memset(&w, 0, sizeof(w));
  w.s[0] = g;
  return launch_bwd_gemm(s, st, w, 1);
}

int launch_xtb(n2nmn_seq2seq* s, cudaStream_t st, const XtbSrc& x) {
  const int K = x.kx + x.kh;
  const dim3 grid0((x.C + kXtbTile - 1) / kXtbTile, (K + kXtbTile - 1) / kXtbTile);
  const int tiles = grid0.x * grid0.y;
  // split the rows while the tiles alone leave SMs idle, keeping >= 128 rows per split
  int splits = std::max(1, std::min((2 * s->num_sms + tiles - 1) / tiles, x.R / 128));
  return launch(s->launches, s2s_xtb_kernel, dim3(grid0.x, grid0.y, splits), 256, 0, st, {}, x);
}

int launch_colsum(n2nmn_seq2seq* s, cudaStream_t st, const float* in, int R, int ld, int C, float* out) {
  const int cb = (C + 255) / 256;
  const int splits = std::max(1, std::min((2 * s->num_sms + cb - 1) / cb, R / 64));
  return launch(s->launches, s2s_colsum_kernel, dim3(cb, splits), 256, 0, st, {}, in, R, ld, C, out);
}

XtbSrc xtb_src() { XtbSrc x; std::memset(&x, 0, sizeof(x)); return x; }

int backward_impl(n2nmn_seq2seq* s, const float* dlp, const float* dne, const float* dwv,
                  const float* dstates, float* gflat, cudaStream_t st) {
  const auto& g = s->cfg;
  const int L = g.lstm_dim, L4 = 4 * L, NL = g.num_layers, Vn = g.num_vocab_nmn;
  const int Vp = (Vn + 3) & ~3, Et = g.embed_dim_txt, En = g.embed_dim_nmn, Td = g.T_decoder;
  const int N = s->rec_N, T = s->rec_T;
  auto off = [&](const std::string& name) { return gflat + s->vars[s->var(name)].offset; };
  if (s->bwd_dirty) TRY(prepare_backward(s, st));
  CUDA_TRY(cudaMemsetAsync(gflat, 0, sizeof(float) * s->flat_size, st));
  for (auto* p : s->d_h) CUDA_TRY(cudaMemsetAsync(p, 0, sizeof(float) * NL * g.max_batch * L, st));
  CUDA_TRY(cudaMemsetAsync(s->d_enc_out, 0, sizeof(float) * T * N * L, st));
  CUDA_TRY(cudaMemsetAsync(s->d_enc_ht, 0, sizeof(float) * T * N * L, st));
  float *drec = s->d_h[0], *dup = s->d_h[1], *hcarry = s->d_h[2], *dc = s->d_h[3];
  const size_t NLs = (size_t)g.max_batch * L;   // per-layer stride of the dh buffers
  // ---- 1. decoder head, every step at once
  HeadBwd hb;
  hb.sc = s->rec_sc; hb.valid = s->rec_valid_bits; hb.tok = s->rec_tok; hb.att = s->rec_att;
  hb.q = s->rec_q; hb.enc_ht = s->enc_ht; hb.enc_out = s->enc_out;
  hb.emb_txt = s->v("encoder/embedding_mat"); hb.seq = s->rec_seq; hb.seq_len = s->rec_len;
  hb.v = s->v("decoder/att_prediction/v"); hb.wy = s->v("decoder/token_prediction/weights");
  hb.dlp = dlp; hb.dne = dne; hb.dwv = dwv;
  hb.ds = s->ds; hb.dh_top = s->dh_top; hb.dq = s->dq; hb.d_enc_out = s->d_enc_out;
  hb.d_enc_ht = s->d_enc_ht; hb.dv_part = s->dv_part; hb.d_emb_txt = off("encoder/embedding_mat");
  hb.T = T; hb.N = N; hb.L = L; hb.V = Vn; hb.Vp = Vp; hb.Td = Td; hb.E = Et;
  TRY(launch(s->launches, s2s_head_bwd_kernel, N, kHeadBwdThreads,
             head_bwd_smem_floats(L, T) * sizeof(float), st, {}, hb));
  // dh_top += dq · W_aᵀ over all T_dec·N rows; att_prediction, token_prediction and v gradients
  const int Rd = Td * N;
  const float* h_top = rec_state_at(s, s->rec_h[1], 1, NL - 1, 0, N);   // [Td·N][L]
  TRY(one_gemm(s, st, bwd_gemm(gemm_ops(s->dq, L, Rd, L, s->wa_t, L, L), s->dh_top, L, nullptr, 0,
                               L, true)));
  XtbSrc x = xtb_src();
  x.x = h_top; x.ldx = L; x.kx = L; x.G = s->dq; x.ldg = L; x.C = L; x.R = Rd;
  x.out = off("decoder/att_prediction/weights"); x.ldo = L;
  TRY(launch_xtb(s, st, x));
  TRY(launch_colsum(s, st, s->dq, Rd, L, L, off("decoder/att_prediction/biases")));
  x = xtb_src();
  x.x = h_top; x.ldx = L; x.kx = L; x.hb = s->rec_d2; x.ldh = L; x.kh = L;
  x.G = s->ds; x.ldg = Vp; x.C = Vn; x.R = Rd;
  x.out = off("decoder/token_prediction/weights"); x.ldo = Vn;
  TRY(launch_xtb(s, st, x));
  TRY(launch_colsum(s, st, s->ds, Rd, Vp, Vn, off("decoder/token_prediction/biases")));
  TRY(launch_colsum(s, st, s->dv_part, N, L, L, off("decoder/att_prediction/v")));
  // ---- 2. decoder BPTT, one cell backward and one [dx, dh_prev] product per layer and step
  auto in_dim = [&](int side, int l) { return l == 0 ? (side == 0 ? Et : En) : L; };
  auto cell_slot = [&](int side, int l, int t) {
    CellBwd c;
    c.gates = rec_gates_at(s, side, l, t, N);
    c.c_prev = t > 0 ? rec_state_at(s, s->rec_c[side], side, l, t - 1, N)
                     : (side == 1 ? rec_state_at(s, s->rec_c[0], 0, l, T - 1, N) : nullptr);
    c.c_new = rec_state_at(s, s->rec_c[side], side, l, t, N);
    c.drec = drec + l * NLs;
    c.dup = l < NL - 1 ? dup + l * NLs : nullptr;
    c.dup_keep = l < NL - 1 && s->rec_drop[side] ? rec_state_at(s, s->drop_keep[side], side, l, t, N)
                                                  : nullptr;
    c.dtop = l == NL - 1 ? (side == 1 ? s->dh_top : s->d_enc_out) + (size_t)t * N * L : nullptr;
    c.hcarry = side == 0 ? hcarry + l * NLs : nullptr;
    c.dc = dc + l * NLs;
    c.dgates = dgates_at(s, side, l, t, N);
    c.seq_len = side == 0 ? s->rec_len : nullptr;
    c.t = t; c.N = N; c.L = L;
    return c;
  };
  auto gemm_slot = [&](int side, int l, int t) {   // [dx, dh_prev] = dgates · Wᵀ (layer 0: dh only)
    const int in = in_dim(side, l);
    const float* B = s->w_t[side][l] + (l == 0 ? in : 0);
    return bwd_gemm(gemm_ops(dgates_at(s, side, l, t, N), L4, N, L4, B, in + L, l == 0 ? L : in + L),
                    l == 0 ? nullptr : dup + (l - 1) * NLs, L, drec + l * NLs, L, l == 0 ? 0 : in,
                    false);
  };
  auto launch_cells = [&](int side, const CellBwdWave& w, int nz) {
    return launch(s->launches, cell_bwd_variant(s->rec_drop[side]), dim3((N * L + 255) / 256, 1, nz),
                  256, 0, st, kPdl, w);
  };
  for (int t = Td - 1; t >= 0; --t)
    for (int l = NL - 1; l >= 0; --l) {
      CellBwdWave cw;
      std::memset(&cw, 0, sizeof(cw));
      cw.s[0] = cell_slot(1, l, t);
      TRY(launch_cells(1, cw, 1));
      BwdGemmWave gw;
      std::memset(&gw, 0, sizeof(gw));
      gw.s[0] = gemm_slot(1, l, t);
      TRY(launch_bwd_gemm(s, st, gw, 1));
    }
  // drec / dc now hold the gradient of the encoder's final state from the decoder; the caller's
  // gradient of that state (the question-prior net's input) joins it
  if (dstates != nullptr)
    TRY(launch(s->launches, s2s_add_state_grad_kernel, dim3((N * L + 255) / 256, NL), 256, 0, st, {},
               dstates, dc, drec, NLs, N, L));
  // ---- 3. encoder: d enc_out += d enc_ht · W_hᵀ, encoder_h_transform gradients
  const int Re = T * N;
  TRY(one_gemm(s, st, bwd_gemm(gemm_ops(s->d_enc_ht, L, Re, L, s->wh_t, L, L), s->d_enc_out, L,
                               nullptr, 0, L, true)));
  x = xtb_src();
  x.x = s->enc_out; x.ldx = L; x.kx = L; x.G = s->d_enc_ht; x.ldg = L; x.C = L; x.R = Re;
  x.out = off("encoder/encoder_h_transform/weights"); x.ldo = L;
  TRY(launch_xtb(s, st, x));
  TRY(launch_colsum(s, st, s->d_enc_ht, Re, L, L, off("encoder/encoder_h_transform/biases")));
  // reverse wavefront: tick k runs layer l at step t = T - 1 - k + (layers - 1 - l)
  for (int k = 0; k < T + NL - 1; ++k) {
    CellBwdWave cw;
    BwdGemmWave gw;
    std::memset(&cw, 0, sizeof(cw));
    std::memset(&gw, 0, sizeof(gw));
    for (int l = 0; l < NL; ++l) {
      const int t = T - 1 - k + (NL - 1 - l);
      if (t < 0 || t >= T) continue;   // idle slot (N = 0, R = 0)
      cw.s[l] = cell_slot(0, l, t);
      gw.s[l] = gemm_slot(0, l, t);
    }
    TRY(launch_cells(0, cw, NL));
    TRY(launch_bwd_gemm(s, st, gw, NL));
  }
  // ---- 4. cell weight and bias gradients over all steps; layer-0 input rows
  for (int side = 0; side < 2; ++side) {
    const int Ts = side == 0 ? T : Td, R = Ts * N;
    for (int l = 0; l < NL; ++l) {
      const int in = in_dim(side, l);
      x = xtb_src();
      if (l == 0) {
        x.table = side == 0 ? s->v("encoder/embedding_mat") : s->dec_rows;
        x.idx = side == 0 ? s->rec_seq : s->rec_tok;
        x.shift = side == 0 ? 0 : N;   // decoder step 0 reads go_embedding (row V of dec_rows)
        x.first_idx = Vn;
      } else {   // the layer below's output as this layer read it: dropped, or h
        x.x = rec_state_at(s, s->rec_drop[side] ? s->drop_x[side] : s->rec_h[side], side, l - 1, 0, N);
        x.ldx = L;
      }
      x.kx = in;
      x.h0 = side == 0 ? nullptr : rec_state_at(s, s->rec_h[0], 0, l, T - 1, N);
      x.hb = rec_state_at(s, s->rec_h[side], side, l, 0, N);
      x.h0_rows = N; x.ldh = L; x.kh = L;
      x.G = dgates_at(s, side, l, 0, N); x.ldg = L4; x.C = L4; x.R = R;
      x.out = off(cell_prefix(side, l) + "weights"); x.ldo = L4;
      TRY(launch_xtb(s, st, x));
      TRY(launch_colsum(s, st, dgates_at(s, side, l, 0, N), R, L4, L4,
                        off(cell_prefix(side, l) + "biases")));
    }
    // embedding rows: d x0 = dgates · W_xᵀ, scattered into the looked-up rows
    TRY(one_gemm(s, st, bwd_gemm(gemm_ops(dgates_at(s, side, 0, 0, N), L4, R, L4, s->w_t[side][0],
                                          in_dim(side, 0) + L, in_dim(side, 0)),
                                 s->dx0, in_dim(side, 0), nullptr, 0, in_dim(side, 0), false)));
    if (side == 0)
      TRY(launch(s->launches, s2s_scatter_rows_kernel, R, 128, 0, st, {}, s->dx0, Et, s->rec_seq, 0,
                 0, off("encoder/embedding_mat"), g.num_vocab_txt, nullptr));
    else
      TRY(launch(s->launches, s2s_scatter_rows_kernel, R, 128, 0, st, {}, s->dx0, En, s->rec_tok, N,
                 Vn, off("decoder/embedding_mat"), Vn, off("decoder/go_embedding")));
  }
  return N2NMN_OK;
}

}  // namespace

extern "C" {

int n2nmn_seq2seq_create(const n2nmn_seq2seq_config* cfg, n2nmn_seq2seq** out) {
  if (!cfg || !out) return fail_with(N2NMN_ERR_ARG, "null argument");
  if (cfg->abi_version != N2NMN_ABI_VERSION) return fail_with(N2NMN_ERR_ARG, "ABI version mismatch");
  const int L = cfg->lstm_dim;
  // lstm_dim: a multiple of 8, the units of one step-kernel CTA (8 units x 4 gates = 32 columns)
  if (cfg->num_vocab_txt <= 0 || cfg->embed_dim_txt <= 0 || cfg->embed_dim_nmn <= 0 ||
      cfg->embed_dim_txt % 4 != 0 || cfg->embed_dim_nmn % 4 != 0 ||
      cfg->num_vocab_nmn <= 0 || cfg->num_vocab_nmn > kMaxVocabNmn || L <= 0 || L % 8 != 0 ||
      cfg->num_layers <= 0 || cfg->num_layers > kMaxLayers || cfg->T_encoder <= 0 ||
      cfg->T_encoder > kMaxTEnc || cfg->T_decoder <= 0 || cfg->max_batch <= 0)
    return fail_with(N2NMN_ERR_ARG,
                     "bad seq2seq config (lstm_dim must be a multiple of 8, embed dims of 4, num_vocab_nmn <= 64, "
                     "num_layers <= 4, T_encoder <= 128)");
  CUDA_TRY(cudaSetDevice(cfg->device));
  cudaDeviceProp prop;
  CUDA_TRY(cudaGetDeviceProperties(&prop, cfg->device));
  if (prop.major != 9)
    return fail_with(N2NMN_ERR_DEVICE, std::string("n2nmn_b200 needs an sm_90 GPU, found sm_") +
                                           std::to_string(prop.major) + std::to_string(prop.minor));
  const size_t smem_max = prop.sharedMemPerBlockOptin;
  if (head_bwd_smem_floats(L, cfg->T_encoder) * sizeof(float) > smem_max)
    return fail_with(N2NMN_ERR_ARG, "lstm_dim too large for the backward head kernel's shared memory");
  const size_t attn_bytes = attn_smem_floats(L, cfg->T_encoder, cfg->num_vocab_nmn) * sizeof(float);
  if (attn_bytes > 200 * 1024 || attn_bytes > smem_max)
    return fail_with(N2NMN_ERR_ARG, "num_vocab_nmn * lstm_dim too large for the decoder step kernel");
  // Kernel attributes belong to the process, not the context, so every context sets the same
  // values: the mma_tile kernels' fixed sizes, and the device's limit for dec_attn and the head
  // backward, whose size follows the config (checked above; neither has static shared memory).
  for (bool exact : {false, true})
    for (bool narrow : {false, true}) {
      TRY(set_smem(gemm_variant(narrow, exact), (int)mma_smem_bytes(narrow ? 2 : 4)));
      TRY(set_smem(bwd_gemm_variant(narrow, exact), (int)mma_smem_bytes(narrow ? 2 : 4)));
      for (bool shared_sm : {false, true})
        for (bool rec : {false, true})
          for (bool drop : {false, true})
            TRY(set_smem(lstm_variant(narrow, shared_sm, exact, rec, drop),
                         (int)lstm_smem(narrow, shared_sm), narrow && shared_sm ? 100 : -1));
    }
  for (bool rec : {false, true})
    TRY(set_smem(rec ? &dec_attn_kernel<true> : &dec_attn_kernel<false>, (int)smem_max));
  TRY(set_smem(s2s_head_bwd_kernel, (int)smem_max));
  // every failure below frees what was built so far (n2nmn_seq2seq_destroy takes a partial context)
  std::unique_ptr<n2nmn_seq2seq, decltype(&n2nmn_seq2seq_destroy)> owner(new n2nmn_seq2seq,
                                                                          n2nmn_seq2seq_destroy);
  n2nmn_seq2seq* s = owner.get();
  s->cfg = *cfg;
  s->num_sms = prop.multiProcessorCount;
  const int C = 4 * L, N = cfg->max_batch, Vt = cfg->num_vocab_txt, Vn = cfg->num_vocab_nmn;
  const int Et = cfg->embed_dim_txt, En = cfg->embed_dim_nmn;
  auto add = [&](const std::string& name, std::vector<int64_t> shape) {
    size_t cnt = 1;
    for (auto d : shape) cnt *= (size_t)d;
    s->vars.push_back({name, shape, nullptr, cnt, false});
  };
  // variables of `encoder_decoder/` in creation order (nmn3_netgen_att.py:73-240)
  add("encoder/embedding_mat", {Vt, Et});
  for (int l = 0; l < cfg->num_layers; ++l) {
    add(cell_prefix(0, l) + "weights", {(l == 0 ? Et : L) + L, C});
    add(cell_prefix(0, l) + "biases", {C});
  }
  add("encoder/encoder_h_transform/weights", {L, L});
  add("encoder/encoder_h_transform/biases", {L});
  add("decoder/embedding_mat", {Vn, En});
  add("decoder/go_embedding", {1, En});
  add("decoder/att_prediction/v", {L});
  add("decoder/att_prediction/weights", {L, L});
  add("decoder/att_prediction/biases", {L});
  add("decoder/token_prediction/weights", {2 * L, Vn});
  add("decoder/token_prediction/biases", {Vn});
  for (int l = 0; l < cfg->num_layers; ++l) {
    add(cell_prefix(1, l) + "weights", {(l == 0 ? En : L) + L, C});
    add(cell_prefix(1, l) + "biases", {C});
  }
  for (auto& v : s->vars) {
    v.offset = s->flat_size;
    s->flat_size += (int64_t)((v.count + 3) & ~size_t(3));
  }
  CUDA_TRY(dmalloc(s, &s->wstore, (size_t)s->flat_size));
  CUDA_TRY(cudaMemset(s->wstore, 0, sizeof(float) * s->flat_size));
  for (auto& v : s->vars) v.dev = s->wstore + v.offset;
  CUDA_TRY(dmalloc(s, &s->table_enc, (size_t)Vt * C));
  CUDA_TRY(dmalloc(s, &s->table_dec, (size_t)(Vn + 1) * C));
  CUDA_TRY(dmalloc(s, &s->dec_rows, (size_t)(Vn + 1) * En));
  CUDA_TRY(dmalloc(s, &s->wy_t, (size_t)Vn * 2 * L));
  for (int side = 0; side < 2; ++side)
    for (int l = 0; l < cfg->num_layers; ++l) {
      const int in = l == 0 ? (side == 0 ? Et : En) : L;
      CUDA_TRY(dmalloc(s, &s->w_cell[side][l], (size_t)(in + L) * C));
      CUDA_TRY(dmalloc(s, &s->b_cell[side][l], (size_t)C));
    }
  for (int l = 0; l < cfg->num_layers; ++l) {
    CUDA_TRY(dmalloc(s, &s->h[l][0], (size_t)N * L));
    CUDA_TRY(dmalloc(s, &s->h[l][1], (size_t)N * L));
    CUDA_TRY(dmalloc(s, &s->c[l], (size_t)N * L));
  }
  const size_t TNL = (size_t)cfg->T_encoder * N * L;
  CUDA_TRY(dmalloc(s, &s->enc_out, TNL));
  CUDA_TRY(dmalloc(s, &s->enc_ht, TNL));
  CUDA_TRY(dmalloc(s, &s->q, (size_t)N * L));
  CUDA_TRY(dmalloc(s, &s->atts, (size_t)cfg->T_decoder * cfg->T_encoder * N));
  CUDA_TRY(dmalloc(s, &s->X, (size_t)N * 3));
  CUDA_TRY(dmalloc(s, &s->cur_tok, (size_t)N));
  CUDA_TRY(dmalloc(s, &s->P, (size_t)Vn * 3));
  CUDA_TRY(dmalloc(s, &s->W, (size_t)3 * Vn * 4));
  CUDA_TRY(dmalloc(s, &s->b, (size_t)Vn * 4));
  *out = owner.release();
  return N2NMN_OK;
}

int n2nmn_seq2seq_destroy(n2nmn_seq2seq* s) {
  if (!s) return N2NMN_OK;
  for (void* p : s->allocs) cudaFree(p);
  delete s;
  return N2NMN_OK;
}

int n2nmn_seq2seq_num_variables(const n2nmn_seq2seq* s) { return s ? (int)s->vars.size() : 0; }

int n2nmn_seq2seq_variable_info(const n2nmn_seq2seq* s, int index, const char** name,
                                int64_t shape[4], int* ndim) {
  if (!s || index < 0 || index >= (int)s->vars.size()) return fail_with(N2NMN_ERR_ARG, "bad variable index");
  const auto& v = s->vars[index];
  if (name) *name = v.name.c_str();
  if (ndim) *ndim = (int)v.shape.size();
  if (shape) for (size_t i = 0; i < v.shape.size() && i < 4; ++i) shape[i] = v.shape[i];
  return N2NMN_OK;
}

int n2nmn_seq2seq_set_weight(n2nmn_seq2seq* s, const char* name, const float* src_dev,
                             const int64_t* shape, int ndim, void* stream) {
  if (!s || !name || !src_dev || !shape) return fail_with(N2NMN_ERR_ARG, "null argument");
  const int i = s->var(name);
  if (i < 0) return fail_with(N2NMN_ERR_ARG, std::string("unknown seq2seq variable: ") + name);
  auto& v = s->vars[i];
  bool same = ndim == (int)v.shape.size();
  for (int d = 0; same && d < ndim; ++d) same = shape[d] == v.shape[d];
  if (!same) return fail_with(N2NMN_ERR_ARG, std::string("shape mismatch for ") + name);
  CUDA_TRY(cudaMemcpyAsync(v.dev, src_dev, v.count * sizeof(float), cudaMemcpyDeviceToDevice,
                           (cudaStream_t)stream));
  v.loaded = true;
  s->dirty = true;
  s->bwd_dirty = true;
  s->rec_valid = false;
  return N2NMN_OK;
}

int n2nmn_seq2seq_set_assembler(n2nmn_seq2seq* s, const int32_t* P, const int32_t* W,
                                const int32_t* b, void* stream) {
  if (!s || !P || !W || !b) return fail_with(N2NMN_ERR_ARG, "null argument");
  const int Vn = s->cfg.num_vocab_nmn;
  auto st = (cudaStream_t)stream;
  CUDA_TRY(cudaMemcpyAsync(s->P, P, sizeof(int32_t) * Vn * 3, cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(s->W, W, sizeof(int32_t) * 3 * Vn * 4, cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(s->b, b, sizeof(int32_t) * Vn * 4, cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaStreamSynchronize(st));   // the host arrays may be temporaries
  s->tables_set = true;
  return N2NMN_OK;
}

int n2nmn_seq2seq_forward(n2nmn_seq2seq* s, const int32_t* input_seq_dev,
                          const int32_t* seq_len_dev, int T_enc, int N,
                          const int32_t* gt_layout_dev, int32_t* tokens_dev,
                          float* token_probs_dev, float* neg_entropy_dev, float* word_vecs_dev,
                          float* atts_dev, void* stream) {
  return n2nmn_seq2seq_forward_ex(s, input_seq_dev, seq_len_dev, T_enc, N, gt_layout_dev, tokens_dev,
                                  token_probs_dev, neg_entropy_dev, word_vecs_dev, atts_dev, stream,
                                  nullptr);
}

int n2nmn_seq2seq_forward_ex(n2nmn_seq2seq* s, const int32_t* input_seq_dev,
                             const int32_t* seq_len_dev, int T_enc, int N,
                             const int32_t* gt_layout_dev, int32_t* tokens_dev,
                             float* token_probs_dev, float* neg_entropy_dev, float* word_vecs_dev,
                             float* atts_dev, void* stream, float* encoder_states_dev) {
  if (!s || !input_seq_dev || !seq_len_dev || !tokens_dev || !token_probs_dev ||
      !neg_entropy_dev || !word_vecs_dev)
    return fail_with(N2NMN_ERR_ARG, "null argument");
  const auto& g = s->cfg;
  if (T_enc <= 0 || T_enc > g.T_encoder || N <= 0 || N > g.max_batch)
    return fail_with(N2NMN_ERR_CAPACITY, "T_enc / N exceed what the seq2seq was created for");
  if (!s->tables_set) return fail_with(N2NMN_ERR_STATE, "assembler tables (P, W, b) not set");
  auto st = (cudaStream_t)stream;
  s->rec_valid = false;
  const bool rec = s->record;
  if (rec) TRY(ensure_record(s));
  const int L = g.lstm_dim, C = 4 * L, NL = g.num_layers, Vn = g.num_vocab_nmn;
  // with one layer there is nothing below the top layer to drop
  const bool drop[2] = {s->drop_u[0] != nullptr && NL > 1, s->drop_u[1] != nullptr && NL > 1};
  for (int side = 0; side < 2; ++side)
    if (drop[side]) TRY(ensure_dropout(s, side, rec));
  if (s->dirty) TRY(prepare(s, st));
  const int Et = g.embed_dim_txt, En = g.embed_dim_nmn, T_dec = g.T_decoder;
  float* atts = atts_dev ? atts_dev : s->atts;
  for (int l = 0; l < NL; ++l) {
    CUDA_TRY(cudaMemsetAsync(s->h[l][0], 0, sizeof(float) * N * L, st));
    CUDA_TRY(cudaMemsetAsync(s->c[l], 0, sizeof(float) * N * L, st));
  }
  TRY(launch(s->launches, init_state_kernel, (N + 127) / 128, 128, 0, st, {}, s->X, s->cur_tok,
             neg_entropy_dev, N, T_dec, Vn));
  const Tiles tl = tiles(N, C, 1, s->num_sms);
  int cur = 0;   // h[l][cur] holds every layer's h_{t-1}
  const bool exact = !(g.flags & N2NMN_SEQ2SEQ_FLAG_TF32);
  // one LSTM cell evaluation: layer l of `side` at step t; `par` = parity of the h buffer that
  // holds the layer's previous state (its own and the layer below's run in lock step)
  auto cell = [&](int side, int l, int t, int par, const int32_t* tok, const int32_t* seq_len,
                  float* out_seq) {
    const int in = l == 0 ? (side == 0 ? Et : En) : L;
    const bool dr = drop[side] && l < NL - 1;
    LstmStep p;
    p.x = l == 0 ? nullptr
                 : drop[side] ? rec_state_at(s, s->drop_x[side], side, l - 1, t, N) : s->h[l - 1][par ^ 1];
    p.h_prev = s->h[l][par];
    p.w = s->w_cell[side][l] + (l == 0 ? (size_t)in * C : 0);
    p.table = l == 0 ? (side == 0 ? s->table_enc : s->table_dec) : nullptr;
    p.tok = tok;
    p.bias = s->b_cell[side][l];
    p.c = s->c[l];
    p.h_out = s->h[l][par ^ 1];
    p.out_seq = l == NL - 1 ? out_seq : nullptr;
    p.seq_len = seq_len;
    p.t = t; p.N = N; p.L = L;
    p.rec_gates = rec ? rec_gates_at(s, side, l, t, N) : nullptr;
    p.rec_c = rec ? rec_state_at(s, s->rec_c[side], side, l, t, N) : nullptr;
    p.rec_h = rec ? rec_state_at(s, s->rec_h[side], side, l, t, N) : nullptr;
    p.drop_u = dr ? s->drop_u[side] + ((size_t)t * (NL - 1) + l) * N * L : nullptr;
    p.drop_out = dr ? rec_state_at(s, s->drop_x[side], side, l, t, N) : nullptr;
    p.drop_keep = dr && rec ? rec_state_at(s, s->drop_keep[side], side, l, t, N) : nullptr;
    return p;
  };
  auto launch_wave = [&](int side, const LstmWave& w, int nz, bool shared_sm) {
    return launch(s->launches, lstm_variant(tl.narrow, shared_sm, exact, rec, drop[side]),
                  dim3(tl.grid.x, tl.grid.y, nz), kMmaThreads, lstm_smem(tl.narrow, shared_sm), st,
                  kPdl, w);
  };
  // encoder, dynamic_rnn (:95-99): tick k runs layer l at step t = k - l
  for (int k = 0; k < T_enc + NL - 1; ++k) {
    LstmWave w;
    std::memset(&w, 0, sizeof(w));
    for (int l = 0; l < NL; ++l) {
      const int t = k - l;
      if (t < 0 || t >= T_enc) continue;    // idle slot (N = 0)
      w.s[l] = cell(0, l, t, t & 1, input_seq_dev + (size_t)t * N, seq_len_dev,
                    s->enc_out + (size_t)t * N * L);
    }
    TRY(launch_wave(0, w, NL, NL > 1));
  }
  cur = T_enc & 1;
  // dynamic_rnn's final state (:95-99), (c, h) per layer: the decoder's initial state, which its
  // first step overwrites in place
  if (encoder_states_dev != nullptr)
    for (int l = 0; l < NL; ++l) {
      float* dst = encoder_states_dev + (size_t)l * 2 * N * L;
      CUDA_TRY(cudaMemcpyAsync(dst, s->c[l], sizeof(float) * N * L, cudaMemcpyDeviceToDevice, st));
      CUDA_TRY(cudaMemcpyAsync(dst + (size_t)N * L, s->h[l][cur], sizeof(float) * N * L,
                               cudaMemcpyDeviceToDevice, st));
    }
  TRY(launch_gemm(s, st, s->enc_out, L, T_enc * N, L, s->v("encoder/encoder_h_transform/weights"),
                  L, L, s->v("encoder/encoder_h_transform/biases"), s->enc_ht, L));   // :104-108
  const size_t attn_smem = attn_smem_floats(L, T_enc, Vn) * sizeof(float);
  for (int t = 0; t < T_dec; ++t) {   // raw_rnn loop (:199-305)
    // decoder step: the layers of one step depend on each other, one launch each
    for (int l = 0; l < NL; ++l) {
      LstmWave w;
      std::memset(&w, 0, sizeof(w));
      w.s[0] = cell(1, l, t, cur, s->cur_tok, nullptr, nullptr);
      TRY(launch_wave(1, w, 1, false));
    }
    cur ^= 1;
    const float* h_top = s->h[NL - 1][cur];
    float* q = rec ? s->rec_q + (size_t)t * N * L : s->q;   // the recording keeps every query
    TRY(launch_gemm(s, st, h_top, L, N, L, s->v("decoder/att_prediction/weights"), L, L,
                    s->v("decoder/att_prediction/biases"), q, L));
    AttnStep a;
    a.q = q; a.h_top = h_top; a.enc_ht = s->enc_ht; a.enc_out = s->enc_out;
    a.v = s->v("decoder/att_prediction/v");
    a.wy_t = s->wy_t; a.by = s->v("decoder/token_prediction/biases");
    a.seq_len = seq_len_dev; a.P = s->P; a.W = s->W; a.b = s->b; a.X = s->X;
    a.gt = gt_layout_dev ? gt_layout_dev + (size_t)t * N : nullptr;
    a.u = s->sample_u ? s->sample_u + (size_t)t * N : nullptr;
    a.tokens = tokens_dev + (size_t)t * N;
    a.cur_tok = s->cur_tok;
    a.probs = token_probs_dev + (size_t)t * N;
    a.neg_entropy = neg_entropy_dev;
    a.atts = atts + (size_t)t * T_enc * N;
    a.T = T_enc; a.N = N; a.L = L; a.V = Vn;
    a.rec_d2 = rec ? s->rec_d2 + (size_t)t * N * L : nullptr;
    a.rec_sc = rec ? s->rec_sc + (size_t)t * N * Vn : nullptr;
    a.rec_att = rec ? s->rec_att + (size_t)t * T_enc * N : nullptr;
    a.rec_valid = rec ? s->rec_valid_bits + (size_t)t * N * 2 : nullptr;
    a.rec_tok = rec ? s->rec_tok + (size_t)t * N : nullptr;
    TRY(launch(s->launches, rec ? &dec_attn_kernel<true> : &dec_attn_kernel<false>, N, kAttnThreads,
               attn_smem, st, kPdl, a));
  }
  TRY(launch(s->launches, word_vecs_kernel, dim3(N, T_dec), 128, sizeof(float) * 2 * T_enc, st, {},
             atts, input_seq_dev, s->v("encoder/embedding_mat"), word_vecs_dev, T_enc, N, Et));
  if (rec) {   // the inputs may be temporaries of the caller
    CUDA_TRY(cudaMemcpyAsync(s->rec_seq, input_seq_dev, sizeof(int32_t) * T_enc * N,
                             cudaMemcpyDeviceToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(s->rec_len, seq_len_dev, sizeof(int32_t) * N, cudaMemcpyDeviceToDevice, st));
    s->rec_N = N;
    s->rec_T = T_enc;
    s->rec_drop[0] = drop[0];
    s->rec_drop[1] = drop[1];
    s->rec_valid = true;
  }
  return N2NMN_OK;
}

int n2nmn_seq2seq_set_sampling(n2nmn_seq2seq* s, const float* uniforms_dev) {
  if (!s) return fail_with(N2NMN_ERR_ARG, "null argument");
  s->sample_u = uniforms_dev;
  return N2NMN_OK;
}

int n2nmn_seq2seq_set_dropout(n2nmn_seq2seq* s, const float* enc_uniforms_dev,
                              const float* dec_uniforms_dev) {
  if (!s) return fail_with(N2NMN_ERR_ARG, "null argument");
  s->drop_u[0] = enc_uniforms_dev;
  s->drop_u[1] = dec_uniforms_dev;
  return N2NMN_OK;
}

int64_t n2nmn_seq2seq_launch_count(const n2nmn_seq2seq* s) { return s ? s->launches : 0; }

int n2nmn_seq2seq_set_record(n2nmn_seq2seq* s, int on) {
  if (!s) return fail_with(N2NMN_ERR_ARG, "null argument");
  s->record = on != 0;
  return N2NMN_OK;
}

int64_t n2nmn_seq2seq_flat_size(const n2nmn_seq2seq* s) { return s ? s->flat_size : 0; }

int n2nmn_seq2seq_flat_offset(const n2nmn_seq2seq* s, int index, int64_t* offset, int64_t* count) {
  if (!s || index < 0 || index >= (int)s->vars.size()) return fail_with(N2NMN_ERR_ARG, "bad variable index");
  if (offset) *offset = s->vars[index].offset;
  if (count) *count = (int64_t)s->vars[index].count;
  return N2NMN_OK;
}

int n2nmn_seq2seq_backward(n2nmn_seq2seq* s, const float* d_log_seq_prob_dev,
                           const float* d_neg_entropy_dev, const float* d_word_vecs_dev,
                           float* grad_flat_dev, void* stream) {
  return n2nmn_seq2seq_backward_ex(s, d_log_seq_prob_dev, d_neg_entropy_dev, d_word_vecs_dev,
                                   grad_flat_dev, stream, nullptr);
}

int n2nmn_seq2seq_backward_ex(n2nmn_seq2seq* s, const float* d_log_seq_prob_dev,
                              const float* d_neg_entropy_dev, const float* d_word_vecs_dev,
                              float* grad_flat_dev, void* stream,
                              const float* d_encoder_states_dev) {
  if (!s || !grad_flat_dev) return fail_with(N2NMN_ERR_ARG, "null argument");
  if (!s->rec_valid)
    return fail_with(N2NMN_ERR_STATE,
                     "seq2seq backward needs a recording forward of this batch (n2nmn_seq2seq_set_record) "
                     "with no weight set since");
  return backward_impl(s, d_log_seq_prob_dev, d_neg_entropy_dev, d_word_vecs_dev,
                       d_encoder_states_dev, grad_flat_dev, (cudaStream_t)stream);
}

int n2nmn_seq2seq_load_flat_weights(n2nmn_seq2seq* s, const float* wflat_dev, void* stream) {
  if (!s || !wflat_dev) return fail_with(N2NMN_ERR_ARG, "null argument");
  CUDA_TRY(cudaMemcpyAsync(s->wstore, wflat_dev, sizeof(float) * s->flat_size,
                           cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  for (auto& v : s->vars) v.loaded = true;
  s->dirty = true;
  s->bwd_dirty = true;
  s->rec_valid = false;
  return N2NMN_OK;
}

int n2nmn_seq2seq_get_flat_weights(const n2nmn_seq2seq* s, float* wflat_dev, void* stream) {
  if (!s || !wflat_dev) return fail_with(N2NMN_ERR_ARG, "null argument");
  CUDA_TRY(cudaMemcpyAsync(wflat_dev, s->wstore, sizeof(float) * s->flat_size,
                           cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return N2NMN_OK;
}

int n2nmn_seq2seq_adam_step(n2nmn_seq2seq* s, float* wflat_dev, float* gflat_dev, float* m_dev,
                            float* v_dev, int step, float lr, float beta1, float beta2, float eps,
                            float max_norm, float weight_decay, void* stream) {
  if (!s || !wflat_dev || !gflat_dev || !m_dev || !v_dev || step < 1)
    return fail_with(N2NMN_ERR_ARG, "bad argument");
  auto st = (cudaStream_t)stream;
  const int nv = (int)s->vars.size();
  if (!s->segs_ready) {
    std::vector<VarSeg> segs(nv);
    for (int i = 0; i < nv; ++i) {
      segs[i].offset = (int)s->vars[i].offset;
      segs[i].count = (int)s->vars[i].count;
      const std::string& n = s->vars[i].name;   // l2_reg covers ".../weights" only (nmn3_model.py:161-166)
      segs[i].decay = n.size() >= 8 && n.compare(n.size() - 8, 8, "/weights") == 0;
    }
    CUDA_TRY(dmalloc_once(s, &s->d_segs, (size_t)nv));
    CUDA_TRY(cudaMemcpy(s->d_segs, segs.data(), nv * sizeof(VarSeg), cudaMemcpyHostToDevice));
    CUDA_TRY(dmalloc_once(s, &s->d_sumsq, (size_t)nv));
    s->segs_ready = true;
  }
  CUDA_TRY(cudaMemsetAsync(s->d_sumsq, 0, nv * sizeof(float), st));
  const dim3 grid(32, nv);
  TRY(launch(s->launches, grad_norm_kernel, grid, 256, 0, st, {}, wflat_dev, gflat_dev, s->d_segs,
             weight_decay, 1.f, s->d_sumsq, nullptr));
  const double lr_t = (double)lr * std::sqrt(1.0 - std::pow((double)beta2, step)) /
                      (1.0 - std::pow((double)beta1, step));
  TRY(launch(s->launches, adam_clip_kernel<false>, grid, 256, 0, st, {}, wflat_dev, gflat_dev,
             m_dev, v_dev, s->d_segs, s->d_sumsq, (float)lr_t, beta1, beta2, eps, max_norm,
             nullptr, nullptr, 0));
  return n2nmn_seq2seq_load_flat_weights(s, wflat_dev, stream);
}

}  // extern "C"
