// Backward pass of the layout generator (seq2seq.cu, n2nmn_seq2seq_backward): the kernels. The
// gradients are TF 1.0's registered gradients of nmn3_netgen_att.py's graph (DESIGN.md §4c):
//   s2s_head_bwd_kernel : one CTA per question, looping over the decoding steps: token scores
//                         (log-prob and entropy terms), d[h_top, d2] = ds·W_yᵀ, attention and
//                         context vector, word_vecs; d enc_out / d enc_ht rows of the question are
//                         owned by its CTA (deterministic sums)
//   s2s_cell_bwd_kernel : LSTM cell backward of one (layer, step) per z slot -> dgates [N][4L]
//   s2s_bwd_gemm_kernel : [dx, dh_prev] = dgates·Wᵀ (and the bulk products dq·W_aᵀ, d enc_ht·W_hᵀ,
//                         dgates·W_xᵀ) on the mma_tile engine, one product per z slot
//   s2s_xtb_kernel      : weight gradients out += Σ_r [x_r, h_r]ᵀ·g_r over all T·N rows (fp32)
//   s2s_colsum_kernel   : bias gradients (column sums); s2s_scatter_rows_kernel: embedding rows
//   s2s_add_state_grad_kernel: the caller's gradient of the encoder's final state (backward_ex)
#pragma once
#include "mma_tile.cuh"

namespace {

constexpr int kHeadBwdThreads = 512;

struct HeadBwd {
  const float* sc;          // [Td][N][V] token scores
  const int32_t* valid;     // [Td][N][2] validity bits
  const int32_t* tok;       // [Td][N] chosen tokens
  const float* att;         // [Td][T][N]
  const float* q;           // [Td][N][L] attention queries
  const float* enc_ht;      // [T][N][L]
  const float* enc_out;     // [T][N][L]
  const float* emb_txt;     // [V_txt][E]
  const int32_t* seq;       // [T][N]
  const int32_t* seq_len;   // [N]
  const float* v;           // [L]
  const float* wy;          // [2L][V] token_prediction weights (TF layout)
  const float* dlp;         // [N] d / d log_seq_prob or nullptr
  const float* dne;         // [N] d / d neg_entropy or nullptr
  const float* dwv;         // [Td][N][E] d / d word_vecs or nullptr
  float* ds;                // [Td][N][Vp] d token scores (zero in the padding)
  float* dh_top;            // [Td][N][L] = ds·W_y[:L]ᵀ (the attention query part is added later)
  float* dq;                // [Td][N][L]
  float* d_enc_out;         // [T][N][L] +=, zeroed by the caller
  float* d_enc_ht;          // [T][N][L] +=, zeroed by the caller
  float* dv_part;           // [N][L] this question's d v
  float* d_emb_txt;         // [V_txt][E] += (atomics), from word_vecs
  int T, N, L, V, Vp, Td, E;
};

__host__ __device__ inline size_t head_bwd_smem_floats(int L, int T) {
  return 2 * (size_t)L + 2 * (size_t)((T + 3) & ~3) + 64 + 32;
}

__global__ void __launch_bounds__(kHeadBwdThreads) s2s_head_bwd_kernel(const HeadBwd p) {
  extern __shared__ __align__(16) float smb[];
  const int n = blockIdx.x, L = p.L, T = p.T, V = p.V, N = p.N;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, nw = kHeadBwdThreads / 32;
  float* s_dv = smb;                        // [L]
  float* s_dd2 = s_dv + L;                  // [L]
  float* s_att = s_dd2 + L;                 // [T]
  float* s_dr = s_att + ((T + 3) & ~3);     // [T]
  float* s_ds = s_dr + ((T + 3) & ~3);      // [64]
  float* s_red = s_ds + 64;                 // [32]
  const int len = p.seq_len[n];
  const size_t tstride = (size_t)N * L;
  for (int d = tid; d < L; d += kHeadBwdThreads) s_dv[d] = 0.f;
  const float g_lp = p.dlp ? p.dlp[n] : 0.f, g_ne = p.dne ? p.dne[n] : 0.f;
  for (int t = 0; t < p.Td; ++t) {
    const size_t tn = (size_t)t * N + n;
    // ---- token scores (:270-285): ds_k = g_lp([k = pred] - p_k) + g_ne p_k (e_k - Σ p e) on
    // valid k, 0 elsewhere; e_k = d(p log max(1e-5, p + 1 - valid)) / dp, TF's Maximum gradient
    // reaching p only where p + 1 - valid > 1e-5
    if (warp == 0) {
      const uint32_t vlo = (uint32_t)p.valid[2 * tn], vhi = (uint32_t)p.valid[2 * tn + 1];
      const int v0 = lane, v1 = lane + 32;
      const bool in0 = v0 < V, in1 = v1 < V;
      const bool ok0 = in0 && ((vlo >> lane) & 1), ok1 = in1 && ((vhi >> lane) & 1);
      const float sc0 = in0 ? p.sc[tn * V + v0] : -INFINITY, sc1 = in1 ? p.sc[tn * V + v1] : -INFINITY;
      const float mx = warp_max(fmaxf(sc0, sc1));
      const float e0 = in0 ? expf(sc0 - mx) : 0.f, e1 = in1 ? expf(sc1 - mx) : 0.f;
      const float se = warp_sum(e0 + e1);
      const float a0 = ok0 ? e0 / se : 0.f, a1 = ok1 ? e1 / se : 0.f;
      const float sv = warp_sum(a0 + a1);
      const float p0 = a0 / sv, p1 = a1 / sv;
      const int pred = p.tok[tn];
      auto ent = [](float pk, bool ok) {
        const float y = pk + (ok ? 0.f : 1.f);
        return logf(fmaxf(1e-5f, y)) + (y > 1e-5f ? pk / y : 0.f);
      };
      const float en0 = in0 ? ent(p0, ok0) : 0.f, en1 = in1 ? ent(p1, ok1) : 0.f;
      const float spe = warp_sum(p0 * en0 + p1 * en1);
      const float ds0 = ok0 ? g_lp * ((v0 == pred ? 1.f : 0.f) - p0) + g_ne * p0 * (en0 - spe) : 0.f;
      const float ds1 = ok1 ? g_lp * ((v1 == pred ? 1.f : 0.f) - p1) + g_ne * p1 * (en1 - spe) : 0.f;
      s_ds[v0] = ds0; s_ds[v1] = ds1;
      if (v0 < p.Vp) p.ds[tn * p.Vp + v0] = ds0;
      if (v1 < p.Vp) p.ds[tn * p.Vp + v1] = ds1;
    }
    for (int te = tid; te < T; te += kHeadBwdThreads) s_att[te] = p.att[((size_t)t * T + te) * N + n];
    __syncthreads();
    // ---- d[h_top, d2] = ds · W_yᵀ (:221-223)
    for (int j = tid; j < 2 * L; j += kHeadBwdThreads) {
      const float* wr = p.wy + (size_t)j * V;
      float x = 0.f;
      for (int k = 0; k < V; ++k) x = fmaf(s_ds[k], wr[k], x);
      if (j < L) p.dh_top[tn * L + j] = x;
      else s_dd2[j - L] = x;
    }
    __syncthreads();
    // ---- d att[te] = dd2 · enc_out[te] + dwv · emb[seq[te]] (:218, :312), te < len
    for (int te = warp; te < len; te += nw) {
      const float* eo = p.enc_out + (size_t)te * tstride + (size_t)n * L;
      float s = 0.f;
      for (int d = lane; d < L; d += 32) s = fmaf(s_dd2[d], eo[d], s);
      if (p.dwv != nullptr) {
        const float* er = p.emb_txt + (size_t)p.seq[(size_t)te * N + n] * p.E;
        const float* gw = p.dwv + tn * p.E;
        for (int e = lane; e < p.E; e += 32) s = fmaf(gw[e], er[e], s);
      }
      s = warp_sum(s);
      if (lane == 0) s_dr[te] = s;
    }
    for (int d = tid; d < L; d += kHeadBwdThreads) {   // d enc_out[te] += att[te]·dd2 (live te)
      const float g = s_dd2[d];
      for (int te = 0; te < len; ++te) p.d_enc_out[(size_t)te * tstride + (size_t)n * L + d] += s_att[te] * g;
    }
    __syncthreads();
    // ---- masked, renormalised softmax over the encoder steps (:213-216): d att_raw = att (datt -
    // Σ att·datt) for te < len, 0 beyond
    if (warp == 0) {
      float s = 0.f;
      for (int te = lane; te < len; te += 32) s += s_att[te] * s_dr[te];
      s = warp_sum(s);
      for (int te = lane; te < T; te += 32) s_dr[te] = te < len ? s_att[te] * (s_dr[te] - s) : 0.f;
    }
    __syncthreads();
    // ---- att_raw = Σ_d tanh(q + enc_ht) v (:208-212)
    for (int d = tid; d < L; d += kHeadBwdThreads) {
      const float qd = p.q[tn * L + d], vd = p.v[d];
      float dqd = 0.f, dvd = 0.f;
      for (int te = 0; te < len; ++te) {
        const size_t o = (size_t)te * tstride + (size_t)n * L + d;
        const float tau = tanhf(qd + p.enc_ht[o]), dr = s_dr[te];
        dvd = fmaf(dr, tau, dvd);
        const float dz = dr * vd * (1.f - tau * tau);
        dqd += dz;
        p.d_enc_ht[o] += dz;
      }
      s_dv[d] += dvd;
      p.dq[tn * L + d] = dqd;
    }
    __syncthreads();
  }
  for (int d = tid; d < L; d += kHeadBwdThreads) p.dv_part[(size_t)n * L + d] = s_dv[d];
  // ---- word_vecs = Σ_te att · embedding_mat[input_seq] (:312): scatter into the embedding rows
  if (p.dwv != nullptr)
    for (int te = 0; te < len; ++te) {
      float* dst = p.d_emb_txt + (size_t)p.seq[(size_t)te * N + n] * p.E;
      for (int e = tid; e < p.E; e += kHeadBwdThreads) {
        float s = 0.f;
        for (int t = 0; t < p.Td; ++t)
          s = fmaf(p.att[((size_t)t * T + te) * N + n], p.dwv[((size_t)t * N + n) * p.E + e], s);
        atomicAdd(dst + e, s);
      }
    }
  (void)s_red;
}

// BasicLSTMCell backward of one (layer, step) per z slot, one thread per (question, unit).
// dh = drec (next step's recurrent product) + dup (the layer above's input product) + hcarry
// (state carried through a later step past the sequence end) + dtop (head / encoder output, live
// rows only). Past the sequence end (encoder) the gates get nothing and dh, dc pass straight
// through (dynamic_rnn's carry, :95-99). kDrop: the layer above read this layer's output through
// dropout, so its input product reaches dh as dup·2·keep (tf.nn.dropout's gradient).
struct CellBwd {
  const float* gates;    // [N][4L] activated i, j, f, o (TF column order)
  const float* c_prev;   // [N][L] or nullptr (zero initial state)
  const float* c_new;    // [N][L]
  const float* drec;     // [N][L]
  const float* dup;      // [N][L] or nullptr
  const uint8_t* dup_keep;   // kDrop: [N][L] keep-mask of the dropout on this layer's output
  const float* dtop;     // [N][L] or nullptr
  float* hcarry;         // [N][L] in/out or nullptr (decoder: no carry)
  float* dc;             // [N][L] in: d c_t; out: d c_{t-1}
  float* dgates;         // [N][4L] out, TF column order (pre-activation gradients)
  const int32_t* seq_len;   // [N] or nullptr
  int t, N, L;
};
struct CellBwdWave { CellBwd s[kMaxLayers]; };

template <bool kDrop = false>
__global__ void __launch_bounds__(256) s2s_cell_bwd_kernel(const CellBwdWave w) {
  pdl_trigger();
  const CellBwd& p = w.s[blockIdx.z];
  pdl_wait();
  if (p.N == 0) return;
  const int L = p.L;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.N * L) return;
  const int n = i / L, u = i - n * L;
  const bool live = p.seq_len == nullptr || p.t < p.seq_len[n];
  float dh = p.drec[i];
  if constexpr (kDrop) {
    if (p.dup) dh += p.dup_keep[i] ? 2.f * p.dup[i] : 0.f;
  } else {
    if (p.dup) dh += p.dup[i];
  }
  if (p.hcarry) dh += p.hcarry[i];
  if (p.dtop && live) dh += p.dtop[i];
  const float dcin = p.dc[i];
  float* dg = p.dgates + (size_t)n * 4 * L + u;
  if (!live) {
    dg[0] = 0.f; dg[L] = 0.f; dg[2 * L] = 0.f; dg[3 * L] = 0.f;
    p.hcarry[i] = dh;   // (seq_len set only in the encoder, which always has a carry buffer)
    return;
  }
  const float* g = p.gates + (size_t)n * 4 * L + u;
  const float gi = g[0], gj = g[L], gf = g[2 * L], go = g[3 * L];
  const float tc = tanhf(p.c_new[i]);
  const float cp = p.c_prev ? p.c_prev[i] : 0.f;
  const float dcc = dcin + dh * go * (1.f - tc * tc);
  dg[0] = dcc * gj * gi * (1.f - gi);
  dg[L] = dcc * gi * (1.f - gj * gj);
  dg[2 * L] = dcc * cp * gf * (1.f - gf);
  dg[3 * L] = dh * tc * go * (1.f - go);
  p.dc[i] = dcc * gf;
  if (p.hcarry) p.hcarry[i] = 0.f;
}

// dc[l] += d_states[l][0], dh[l] += d_states[l][1]: the caller's gradient of the encoder's final
// (c, h) [layers][2][N][L] added to the decoder's; grid = (ceil(N·L / 256), layers)
__global__ void __launch_bounds__(256) s2s_add_state_grad_kernel(const float* __restrict__ d_states,
                                                                 float* __restrict__ dc,
                                                                 float* __restrict__ dh,
                                                                 size_t layer_stride, int N, int L) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x, l = blockIdx.y;
  if (i >= N * L) return;
  const float* src = d_states + (size_t)l * 2 * N * L;
  dc[l * layer_stride + i] += src[i];
  dh[l * layer_stride + i] += src[(size_t)N * L + i];
}

// out = [accumulate ? out : 0] + A·B on the mma_tile engine, columns [0, split) to out0 and
// [split, C) to out1 (the input and recurrent parts of [dx, dh_prev] = dgates·Wᵀ).
struct BwdGemm {
  GemmOperands op;
  float* out0; int ldo0;
  float* out1; int ldo1;
  int split, accumulate;
};
struct BwdGemmWave { BwdGemm s[kMaxLayers]; };

template <int WM, bool kExact>
__global__ void __launch_bounds__(kMmaThreads) s2s_bwd_gemm_kernel(const BwdGemmWave w) {
  pdl_trigger();
  const BwdGemm& p = w.s[blockIdx.z];
  extern __shared__ __align__(16) float mma_smem[];
  const int row0 = blockIdx.y * 16 * WM, c0 = blockIdx.x * kMmaCols;
  if (p.op.R == 0 || c0 >= p.op.C || row0 >= p.op.R) { pdl_wait(); return; }
  float acc[4][4];
  if (!mma_tile<WM, kExact>(mma_smem, p.op, row0, c0, acc, [] {})) return;
  const int lane = threadIdx.x & 31, wm = (threadIdx.x >> 5) % WM, g = lane >> 2, tig = lane & 3;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int r = row0 + wm * 16 + g + 8 * hh;
    if (r >= p.op.R) continue;
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int c = c0 + nt * 8 + 2 * tig + j;
        if (c >= p.op.C) continue;
        float* o = c < p.split ? p.out0 + (size_t)r * p.ldo0 + c
                               : p.out1 + (size_t)r * p.ldo1 + (c - p.split);
        *o = (p.accumulate ? *o : 0.f) + acc[nt][hh * 2 + j];
      }
  }
}

// out[k][c] += Σ_r A[r][k] G[r][c], A = [x | h]: columns [0, kx) are x rows (dense x + r·ldx, or
// the gathered table row idx(r) with idx(r) = first_idx for r < shift, else idx[r - shift]),
// columns [kx, kx + kh) are h rows (the first h0_rows rows from h0, nullptr = zeros, then
// hb + (r - h0_rows)·ldh). 64 x 64 output tile per CTA, 4 x 4 per thread, rows in chunks of 16;
// grid.z splits the rows (atomics into the zeroed gradient buffer).
struct XtbSrc {
  const float* x; int ldx;
  const float* table; const int32_t* idx; int shift, first_idx;
  int kx;
  const float* h0; const float* hb; int h0_rows, ldh, kh;
  const float* G; int ldg, C, R;
  float* out; int ldo;
};
constexpr int kXtbTile = 64, kXtbRows = 16;

__global__ void __launch_bounds__(256) s2s_xtb_kernel(const XtbSrc p) {
  __shared__ float As[kXtbRows][kXtbTile], Gs[kXtbRows][kXtbTile + 4];
  const int k0 = blockIdx.y * kXtbTile, c0 = blockIdx.x * kXtbTile;
  const int K = p.kx + p.kh, tid = threadIdx.x, tk = (tid >> 4) * 4, tc = (tid & 15) * 4;
  const int chunk = (p.R + gridDim.z - 1) / gridDim.z;
  const int rb = blockIdx.z * chunk, re = min(p.R, rb + chunk);
  float acc[4][4] = {};
  for (int r0 = rb; r0 < re; r0 += kXtbRows) {
    for (int e = tid; e < kXtbRows * kXtbTile; e += 256) {
      const int rr = e / kXtbTile, kk = e - rr * kXtbTile, r = r0 + rr, k = k0 + kk;
      float a = 0.f, gv = 0.f;
      if (r < re) {
        if (k < p.kx) {
          if (p.table != nullptr) {
            const int ix = r < p.shift ? p.first_idx : p.idx[r - p.shift];
            a = p.table[(size_t)ix * p.kx + k];
          } else {
            a = p.x[(size_t)r * p.ldx + k];
          }
        } else if (k < K) {
          const int kh = k - p.kx;
          if (r < p.h0_rows) a = p.h0 ? p.h0[(size_t)r * p.ldh + kh] : 0.f;
          else a = p.hb[(size_t)(r - p.h0_rows) * p.ldh + kh];
        }
        if (c0 + kk < p.C) gv = p.G[(size_t)r * p.ldg + c0 + kk];
      }
      As[rr][kk] = a;
      Gs[rr][kk] = gv;
    }
    __syncthreads();
#pragma unroll
    for (int rr = 0; rr < kXtbRows; ++rr) {
      const float4 a4 = *reinterpret_cast<const float4*>(&As[rr][tk]);
      const float4 g4 = *reinterpret_cast<const float4*>(&Gs[rr][tc]);
      const float av[4] = {a4.x, a4.y, a4.z, a4.w}, gvv[4] = {g4.x, g4.y, g4.z, g4.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], gvv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int k = k0 + tk + i, c = c0 + tc + j;
      if (k < K && c < p.C) {
        float* o = p.out + (size_t)k * p.ldo + c;
        if (gridDim.z == 1) *o += acc[i][j];
        else atomicAdd(o, acc[i][j]);
      }
    }
}

// out[c] += Σ_r in[r][c]; grid = (ceil(C / 256), row splits)
__global__ void __launch_bounds__(256) s2s_colsum_kernel(const float* __restrict__ in, int R, int ld,
                                                         int C, float* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const int chunk = (R + gridDim.y - 1) / gridDim.y, rb = blockIdx.y * chunk, re = min(R, rb + chunk);
  float s = 0.f;
  for (int r = rb; r < re; ++r) s += in[(size_t)r * ld + c];
  if (gridDim.y == 1) out[c] += s;
  else atomicAdd(out + c, s);
}

// Embedding rows: dst row idx(r) += src[r] (idx as in XtbSrc); rows >= rows_main go to `extra`
// (the decoder's go_embedding, the row after its embedding_mat). One CTA per source row.
__global__ void __launch_bounds__(128) s2s_scatter_rows_kernel(const float* __restrict__ src, int E,
                                                               const int32_t* __restrict__ idx,
                                                               int shift, int first_idx,
                                                               float* __restrict__ dst, int rows_main,
                                                               float* __restrict__ extra) {
  const int r = blockIdx.x;
  const int ix = r < shift ? first_idx : idx[r - shift];
  float* d = ix < rows_main ? dst + (size_t)ix * E : extra + (size_t)(ix - rows_main) * E;
  for (int e = threadIdx.x; e < E; e += blockDim.x) {
    const float v = src[(size_t)r * E + e];
    if (v != 0.f) atomicAdd(d + e, v);
  }
}

}  // namespace
