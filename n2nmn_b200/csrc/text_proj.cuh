// K1: text projection for every node that takes a text vector, and the quadratic-form
// coefficients of the Transform nodes.
//   tau[r, :] = word_vecs[t_r, b_r, :] · W_txt[set] + b_txt[set]
// (fc('fc_text') / fc('text_fc'): models_clevr/nmn3_modules.py:104,167,209,429,478 through
//  util/cnn.py:116). The gather of _slice_word_vecs (nmn3_modules.py:53-57) is folded into the
// load: row (t*N + b) of the segment's time-major word_vecs.
//
// Both are small dense products  C[r, c] = Σ_k A[r, k] · B[k, c]  with a few hundred to a few
// thousand rows per launch, done with fp32 parity on the tensor cores by the shared tile engine
// (mma_tile.cuh: mma.sync m16n8k8, error-compensated TF32, operands streamed by cp.async): 64 rows
// x 32 columns per CTA.
//   History: round 1 gave every group of 8 rows its own CTA, which streamed the whole weight
//   matrix from L2 with a handful of loads in flight (~1000 SM-cycles per row). Round 2 first used
//   a 64 x 64 FFMA tile with both operands whole in shared memory: ncu (profiles/r2g.md) showed it
//   bound by shared-memory wavefronts — an LDS.128 is four wavefronts whatever it broadcasts, so
//   a 2 x 4 register tile pays 24 wavefronts per 32 FMAs — 24.3 K wavefronts in 26 K active cycles
//   per tile, 27 us per launch of 8 batches. Fragments need a fifth of that traffic.
//   text_proj_kernel : A = gathered word vectors (K = Dt), B = W_txt [Dt][Mp]; emits tau,
//                      tau∘w_eltwise and tau² so the consumers' epilogues are pure FMAs.
//   quad_kernel      : A = tau (first n outputs) or tau² (the rest) of the Transform rows, K = Mp,
//                      B = conv_quad^T [Mp][quad_pitch] (common.cuh); emits (u, Q) per node.
// Weights are stored with row pitch Mp (zero padded), so padded columns come out as exact zeros.
#pragma once
#include "common.cuh"
#include "mma_tile.cuh"

namespace n2nmn {

constexpr int kTextStages = 2;   // K = 300 / Mp: 2-3 chunks; 108 KB of ring, two CTAs per SM

// Rows of each text weight set, by value: a CTA finds its group without touching global memory.
struct TextSetRows { int32_t start[NUM_TEXT_SETS + 1]; };

// grid = (Mp / 32, groups); one group = <= 64 text rows of ONE weight set (schedule.cpp)
__global__ void __launch_bounds__(kMmaThreads)
text_proj_kernel(DevModel md, TextBufs tb, TextSetRows rows,
                 const int32_t* __restrict__ text_t, const int32_t* __restrict__ text_b) {
  pdl_trigger();   // the contraction kernel only needs our output in its epilogue
  const int M = md.M, Mp = md.Mp;
  TextGroup g;   // blockIdx.y-th group, groups never straddle weight sets
  {
    int gi = blockIdx.y, set = 0;
    for (; set < NUM_TEXT_SETS; ++set) {
      const int ng = (rows.start[set + 1] - rows.start[set] + kTextRowsPerCta - 1) / kTextRowsPerCta;
      if (gi < ng) break;
      gi -= ng;
    }
    g.set = set;
    g.start = rows.start[set] + gi * kTextRowsPerCta;
    g.count = min(kTextRowsPerCta, rows.start[set + 1] - g.start);
  }
  const int es = (g.set == TS_FIND) ? ES_FIND : (g.set == TS_FSP) ? ES_FSP
               : (g.set == TS_TRANSFORM) ? ES_TRANSFORM : -1;
  const int c0 = blockIdx.x * kMmaCols;
  __shared__ const float* s_rows[kTextRowsPerCta];   // the gather of _slice_word_vecs
  if (threadIdx.x < kTextRowsPerCta)
    s_rows[threadIdx.x] = (int)threadIdx.x < g.count
        ? word_vec_row(md, text_t[g.start + threadIdx.x], text_b[g.start + threadIdx.x]) : nullptr;
  __syncthreads();
  GemmOperands op;
  op.a0 = nullptr; op.k0 = md.Dt; op.lda0 = 0; op.a1 = nullptr; op.k1 = 0; op.lda1 = 0;
  op.R = kTextRowsPerCta; op.B = md.txt_w[g.set]; op.ldb = Mp; op.C = Mp; op.a_rows = s_rows;
  extern __shared__ __align__(16) float mma_smem[];
  float acc[4][4];
  if (!mma_tile<4, true, kTextStages>(mma_smem, op, 0, c0, acc, [] {})) return;
  const int lane = threadIdx.x & 31, wm = (threadIdx.x >> 5) & 3, gq = lane >> 2, tig = lane & 3;
#pragma unroll
  for (int nt = 0; nt < 4; ++nt) {
    const int c = c0 + nt * 8 + 2 * tig;   // this thread's two adjacent columns of n-tile nt
    float bias[2], w2[2];
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const bool live = c + j < M;
      bias[j] = live ? md.txt_b[g.set][c + j] : 0.f;
      w2[j] = (live && es >= 0) ? md.elt_w[es][c + j] : 1.f;
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int r = wm * 16 + gq + 8 * hh;
      if (r >= g.count) continue;
      const float t0 = (c < M) ? acc[nt][2 * hh] + bias[0] : 0.f;
      const float t1 = (c + 1 < M) ? acc[nt][2 * hh + 1] + bias[1] : 0.f;
      const size_t idx = (size_t)(g.start + r) * Mp + c;
      *reinterpret_cast<float2*>(tb.tau + idx) = make_float2(t0, t1);
      *reinterpret_cast<float2*>(tb.tauw + idx) = make_float2(t0 * w2[0], t1 * w2[1]);
      *reinterpret_cast<float2*>(tb.tau2 + idx) = make_float2(t0 * t0, t1 * t1);
    }
  }
}

// (u, Q) of the Transform nodes (common.cuh): tq[row, o] = Σ_c (o < n ? tau : tau²)[row, c] ·
// conv_quad^T[c, o] for the text rows [row0, row0 + nrows) of the Transform weight set.
// Column block 0 = the u columns [0, quad_u_pitch) against tau; block b >= 1 = 32 Q columns from
// quad_u_pitch + 32 (b - 1) against tau² (which the text kernel already stored).
// grid = (1 + ceil((quad_pitch - quad_u_pitch) / 32), ceil(nrows / 64)).
__global__ void __launch_bounds__(kMmaThreads)
quad_kernel(DevModel md, TextBufs tb, int row0, int nrows) {
  pdl_trigger();
  const int Mp = md.Mp, qp = quad_pitch(md.ksize), nu = quad_u_pitch(md.ksize);
  const int r0 = row0 + blockIdx.y * 64, cnt = min(64, row0 + nrows - r0);
  const bool upart = blockIdx.x == 0;
  const int c0 = upart ? 0 : nu + kMmaCols * ((int)blockIdx.x - 1);
  GemmOperands op;
  op.a0 = (upart ? tb.tau : tb.tau2) + (size_t)r0 * Mp; op.k0 = Mp; op.lda0 = Mp;
  op.a1 = nullptr; op.k1 = 0; op.lda1 = 0;
  op.R = cnt; op.B = md.conv_quad; op.ldb = qp; op.C = upart ? nu : qp;
  extern __shared__ __align__(16) float mma_smem[];
  float acc[4][4];
  // (the tile routine waits for the text kernel — tau, tau² — after requesting the weights)
  if (!mma_tile<4, true, kTextStages>(mma_smem, op, 0, c0, acc, [] {})) return;
  const int lane = threadIdx.x & 31, wm = (threadIdx.x >> 5) & 3, gq = lane >> 2, tig = lane & 3;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int r = wm * 16 + gq + 8 * hh;
    if (r >= cnt) continue;
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      const int c = c0 + nt * 8 + 2 * tig;
      if (c + 1 < op.C)
        *reinterpret_cast<float2*>(tb.tq + (size_t)(r0 + r) * qp + c) =
            make_float2(acc[nt][2 * hh], acc[nt][2 * hh + 1]);
      else if (c < op.C)
        tb.tq[(size_t)(r0 + r) * qp + c] = acc[nt][2 * hh];
    }
  }
}

}  // namespace n2nmn
