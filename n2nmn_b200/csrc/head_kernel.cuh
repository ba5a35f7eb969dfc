// K4: batched answer heads of the attention-pooled root modules (evaluation schedules with
// pooled_direct, schedule.hpp).
//
// DescribeModule / SamePropertyModule (models_clevr/nmn3_modules.py:402-495, VQA
// models_vqa/nmn3_modules.py:193-240) are
//     f   = Σ_p softmax(att)_p · X_b[p,:]                      (pooled feature, D values)
//     φ   = f · W_att + b_att            (fc_att; SameProperty: φ0, φ1 with their own W_att)
//     e   = τ ∘ φ (∘ φ1),  ê = l2_normalize(e),  scores = ê · W_out + b_out.
// Round 1 computed φ from a stored per-image map G = X_b·W_att + b made by the contraction kernel
// (Σ_p s_p = 1): that made HALF of the contraction kernel's tiles serve these few root nodes
// (two 128-row tiles of 16.8 MFMA each per image and layer, against 0.2 MFMA for f and φ done
// directly). Now the tree kernel only writes the softmaxed attention weights of such a root;
//   pool_kernel : f for every (root, 128-channel chunk) — one CTA each, every load of the 150
//                 feature rows independent (a single memory round trip, not a chain inside the
//                 question's CTA);
//   head_kernel : the two small dense products for up to 16 roots of one type per CTA, so every
//                 weight matrix is read once per 16 nodes instead of once per node (VQA: W_out is
//                 12 MB).
// Exact fp32 on the CUDA cores: 100 nodes x 512 x 250 MACs per launch is microseconds of work, and
// fp32 here is tighter than the TF32 maps it replaces.
#pragma once
#include "node_eval.cuh"

namespace n2nmn {

constexpr int kHeadThreads = 512;    // 16 warps x 48 weight loads per lane in flight
constexpr int kPoolQuads = 32;      // channel quads (128 channels) per pool-kernel CTA
constexpr int kPoolSlices = 8;      // pixel slices = warps

// f[row, chunk] = Σ_p s_p · X_b[p, chunk] (reduce_sum(image_feat_grid * att_softmax, [1,2]),
// models_clevr/nmn3_modules.py:432-440, 482-487). grid = (pool rows, channel chunks).
__global__ void __launch_bounds__(kPoolQuads * kPoolSlices)
pool_kernel(const NodeCtx c, const int32_t* __restrict__ pool_img, int HWp) {
  extern __shared__ __align__(16) float pool_smem[];   // [HWp] weights + [slices][quads] float4
  const DevModel& md = c.md;
  const int HW = md.HW, quads = md.feat_pitch >> 2;
  float* s_w = pool_smem;
  float4* s_red = reinterpret_cast<float4*>(pool_smem + HWp);
  const int row = blockIdx.x;
  const int q = threadIdx.x & (kPoolQuads - 1), sl = threadIdx.x / kPoolQuads;
  const int qb = blockIdx.y * kPoolQuads + q;
  const int g = pool_img[row];                       // launch table (uploaded before the step)
  const int seg = g / md.N;
  const float4* __restrict__ X = reinterpret_cast<const float4*>(
      md.feat_seg[seg] + (size_t)(g - seg * md.N) * HW * md.feat_pitch);
  pdl_trigger();
  pdl_wait();                                        // the weights come from the tree kernel
  for (int p = threadIdx.x; p < HW; p += blockDim.x) s_w[p] = c.pool_att[(size_t)row * HWp + p];
  __syncthreads();
  float4 A = make_float4(0.f, 0.f, 0.f, 0.f);
  if (qb < quads) {
    constexpr int kB = 10;   // feature rows in flight per thread (all loads issued before any use)
    for (int p0 = sl; p0 < HW; p0 += kPoolSlices * kB) {
      float4 x[kB];
#pragma unroll
      for (int i = 0; i < kB; ++i) {
        const int p = p0 + i * kPoolSlices;
        x[i] = (p < HW) ? __ldg(X + (size_t)p * quads + qb) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int i = 0; i < kB; ++i) {
        const int p = p0 + i * kPoolSlices;
        const float w = (p < HW) ? s_w[p] : 0.f;
        A.x = fmaf(w, x[i].x, A.x); A.y = fmaf(w, x[i].y, A.y);
        A.z = fmaf(w, x[i].z, A.z); A.w = fmaf(w, x[i].w, A.w);
      }
    }
  }
  s_red[sl * kPoolQuads + q] = A;
  __syncthreads();
  if (sl == 0 && qb < quads) {
#pragma unroll
    for (int j = 1; j < kPoolSlices; ++j) {
      const float4 t = s_red[j * kPoolQuads + q];
      A.x += t.x; A.y += t.y; A.z += t.z; A.w += t.w;
    }
    reinterpret_cast<float4*>(c.pooled + (size_t)row * c.pool_pitch)[qb] = A;
  }
}

struct HeadSmem { int f, phi, scratch, total; };
__host__ __device__ inline HeadSmem head_smem_layout(int nn, int pitch, int Mp) {
  HeadSmem s;
  s.f = 2 * nn * (pitch + 4);        // pooled rows of the chunk (nn = nodes per CTA), padded
                                     // pitch, as two planes: TF32 hi part, TF32 lo part
  s.phi = 2 * nn * Mp;               // φ0 / φ1 (ê is written over φ0)
  s.scratch = 8 * kHeadNodesMax * 32;
  s.total = s.f + s.phi + s.scratch;   // == head_smem_floats(nn, pitch, Mp)
  return s;
}

// phi[n][c] = bias[c] + Σ_k F[n][k]·W[k*M + c] for the chunk's <= 16 rows (rows >= cnt are zeros).
// A 16 x Mp x Dk product: on the CUDA cores it is bound by the shared-memory reads of F (every
// FMA needs one F value per lane: 8 MB of smem->register traffic per CTA, measured 34 us), so it
// runs on mma.sync m16n8k8 fragments instead — the 16 nodes are exactly one M tile, each warp owns
// Mp/8 columns, the B fragments come straight from the TF-layout weight matrix in global memory
// (4 rows x 32 B per load instruction), A fragments from the padded F rows in shared memory.
// Precision: the pooled features enter as a TF32 hi + lo pair (split once when they are staged, so
// they lose nothing), the weights are rounded to TF32 (cvt.rna) as they are loaded — the same
// operand rounding the stored maps this replaces had on BOTH operands. (Splitting the weights as
// well made the loop issue-bound: cvt.rna.tf32 is a multi-instruction sequence.)
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hi) : "f"(x));
  const float r = x - __uint_as_float(hi);
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lo) : "f"(r));
}
__device__ __forceinline__ void mma_16x8x8_tf32(float (&d)[4], const uint32_t (&a)[4],
                                                uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
      "{%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// Fs: [NN][fp] (fp = pitch + 4: rows g and g+8 of a fragment then fall in different banks); rows
// >= NN of the 16-row M tile are zeros and are never stored. Each of the 16 warps owns Mp/16
// columns = NT n-tiles of 8 (NT = 2 for Mp = 256 ... 8 for Mp = 1024) and keeps 48 weight loads per
// lane in flight: the product is a stream of the weight matrix through one SM (512 KB ... 8 MB),
// so memory-level parallelism is what sets its duration.
template <int NN, int NT>
__device__ __forceinline__ void head_fc_att_nt(const float* __restrict__ Fs, int fp, int Dk,
                                               const float* __restrict__ W, int M, int Mp,
                                               const float* __restrict__ bias, float* phi) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int ksteps = (Dk + 7) >> 3;
  const int n0 = warp * (8 * NT);
  if (n0 >= Mp) return;
  float acc[NT][4];
#pragma unroll
  for (int j = 0; j < NT; ++j)
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[j][i] = 0.f;
  // B fragment values of k-step ks, n-tile j: W[8ks + t (+4)][n0 + 8j + g]
  auto loadB = [&](int ks, float (&b)[NT][2]) {
#pragma unroll
    for (int j = 0; j < NT; ++j) {
      const int col = n0 + 8 * j + g;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int k = 8 * ks + t + 4 * h;
        b[j][h] = (col < M && k < Dk) ? __ldg(W + (size_t)k * M + col) : 0.f;
      }
    }
  };
  constexpr int PF = 24 / NT;      // k-steps of B values in flight (48 loads per lane)
  float bq[PF][NT][2];
#pragma unroll
  for (int u = 0; u < PF; ++u) loadB(u, bq[u]);
  for (int ks0 = 0; ks0 < ksteps; ks0 += PF) {
#pragma unroll
    for (int u = 0; u < PF; ++u) {
      const int ks = ks0 + u;
      float bcur[NT][2];
#pragma unroll
      for (int j = 0; j < NT; ++j) { bcur[j][0] = bq[u][j][0]; bcur[j][1] = bq[u][j][1]; }
      loadB(ks + PF, bq[u]);     // (guards make loads beyond Dk zeros)
      if (ks < ksteps) {
        const int k = 8 * ks + t;
        uint32_t ah[4], al[4];
        const bool r0 = g < NN, r1 = g + 8 < NN;
        const uint32_t* Fh = reinterpret_cast<const uint32_t*>(Fs);
        const uint32_t* Fl = Fh + NN * fp;
        ah[0] = r0 ? Fh[g * fp + k] : 0u;           al[0] = r0 ? Fl[g * fp + k] : 0u;
        ah[1] = r1 ? Fh[(g + 8) * fp + k] : 0u;     al[1] = r1 ? Fl[(g + 8) * fp + k] : 0u;
        ah[2] = r0 ? Fh[g * fp + k + 4] : 0u;       al[2] = r0 ? Fl[g * fp + k + 4] : 0u;
        ah[3] = r1 ? Fh[(g + 8) * fp + k + 4] : 0u; al[3] = r1 ? Fl[(g + 8) * fp + k + 4] : 0u;
#pragma unroll
        for (int j = 0; j < NT; ++j) {
          uint32_t b0, b1;
          asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(b0) : "f"(bcur[j][0]));
          asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(b1) : "f"(bcur[j][1]));
          mma_16x8x8_tf32(acc[j], al, b0, b1);
          mma_16x8x8_tf32(acc[j], ah, b0, b1);
        }
      }
    }
  }
  // C fragment: (row g, cols 2t, 2t+1), (row g+8, same cols)
#pragma unroll
  for (int j = 0; j < NT; ++j) {
    const int col = n0 + 8 * j + 2 * t;
    const float b0 = col < M ? bias[col] : 0.f, b1 = col + 1 < M ? bias[col + 1] : 0.f;
    if (g < NN) {
      phi[g * Mp + col] = col < M ? acc[j][0] + b0 : 0.f;
      phi[g * Mp + col + 1] = col + 1 < M ? acc[j][1] + b1 : 0.f;
    }
    if (g + 8 < NN) {
      phi[(g + 8) * Mp + col] = col < M ? acc[j][2] + b0 : 0.f;
      phi[(g + 8) * Mp + col + 1] = col + 1 < M ? acc[j][3] + b1 : 0.f;
    }
  }
}
template <int NN>
__device__ __forceinline__ void head_fc_att(const float* __restrict__ Fs, int fp, int Dk,
                                            const float* __restrict__ W, int M, int Mp,
                                            const float* __restrict__ bias, float* phi) {
  if (Mp <= 256) head_fc_att_nt<NN, 2>(Fs, fp, Dk, W, M, Mp, bias, phi);
  else if (Mp <= 512) head_fc_att_nt<NN, 4>(Fs, fp, Dk, W, M, Mp, bias, phi);
  else head_fc_att_nt<NN, 8>(Fs, fp, Dk, W, M, Mp, bias, phi);
}

template <int NN>
__global__ void __launch_bounds__(kHeadThreads)
head_kernel(const NodeCtx c, const NodeRec* __restrict__ nodes,
            const HeadWork* __restrict__ work, const int32_t* __restrict__ list) {
  extern __shared__ __align__(16) float head_smem[];
  const DevModel& md = c.md;
  const int M = md.M, Mp = md.Mp, C = md.C, Dk = md.Dk, HW = md.HW;
  const int HWp = (HW + 3) & ~3;
  const float* __restrict__ pooled = c.pooled;
  const int pool_pitch = c.pool_pitch;
  const HeadSmem L = head_smem_layout(NN, pool_pitch, Mp);
  float* Fs = head_smem;
  float* phi0 = Fs + L.f;
  float* phi1 = phi0 + NN * Mp;
  float* scratch = phi1 + NN * Mp;
  __shared__ int s_node[kHeadNodesMax];
  __shared__ const float* s_rowp[2][kHeadNodesMax];   // input rows of the chunk's nodes
  __shared__ const float* s_taup[kHeadNodesMax];
  __shared__ float* s_outp[kHeadNodesMax];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

  const HeadWork wk = work[blockIdx.x];   // launch tables: uploaded before any kernel of the step
  const int cnt = wk.count;
  const bool feat = (wk.op == OP_DESCRIBE || wk.op == OP_SAME_PROPERTY);
  const bool two = (wk.op == OP_SAME_PROPERTY || wk.op == OP_EQUAL_NUM ||
                    wk.op == OP_MORE_NUM || wk.op == OP_LESS_NUM);
  if (threadIdx.x < kHeadNodesMax)
    s_node[threadIdx.x] = threadIdx.x < cnt ? list[wk.first + threadIdx.x] : -1;
  __syncthreads();
  if (threadIdx.x < cnt) {   // node records -> pointers (one dependent round trip, not one per use)
    const NodeRec nd = nodes[s_node[threadIdx.x]];
    const float* base = feat ? pooled : c.pool_att;
    const size_t pitch = feat ? (size_t)pool_pitch : (size_t)HWp;
    s_rowp[0][threadIdx.x] = base + (size_t)nd.aux * pitch;
    s_rowp[1][threadIdx.x] = base + (size_t)(two ? nd.aux2 : nd.aux) * pitch;
    s_taup[threadIdx.x] = feat ? c.tb.tau + (size_t)nd.text * Mp : nullptr;
    s_outp[threadIdx.x] = score_row(c, nd.out);
  }
  pdl_wait();            // inputs come from the pool / tree kernel, tau from the text kernel
  __syncthreads();

  const float* fin;       // [cnt][fpitch] input of the final fc, fL values each
  int fpitch, fL;
  const float* __restrict__ Wo;
  const float* __restrict__ bo;
  if (feat) {
    for (int which = 0; which < (two ? 2 : 1); ++which) {
      // ---- the chunk's pooled rows -> shared memory as TF32 hi / lo planes (unused rows = 0)
      for (int i = threadIdx.x; i < NN * (pool_pitch >> 2); i += kHeadThreads) {
        const int n = i / (pool_pitch >> 2), q = i - n * (pool_pitch >> 2);
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (n < cnt && 4 * q < md.feat_pitch)   // (columns beyond the feature pitch: zeros)
          v = __ldg(reinterpret_cast<const float4*>(s_rowp[which][n]) + q);
        uint4 hi, lo;
        split_tf32(v.x, hi.x, lo.x); split_tf32(v.y, hi.y, lo.y);
        split_tf32(v.z, hi.z, lo.z); split_tf32(v.w, hi.w, lo.w);
        reinterpret_cast<uint4*>(Fs + n * (pool_pitch + 4))[q] = hi;
        reinterpret_cast<uint4*>(Fs + (NN + n) * (pool_pitch + 4))[q] = lo;
      }
      __syncthreads();
      const int set = two ? (which ? PS_SP_ATT1 : PS_SP_ATT0) : PS_DESC_ATT;
      head_fc_att<NN>(Fs, pool_pitch + 4, Dk, md.proj_w[set], M, Mp, md.proj_b[set],
                      which ? phi1 : phi0);
      __syncthreads();
    }
    // ---- e = τ∘φ0(∘φ1), l2_normalize over the M channels (nmn3_modules.py:448, 491)
    for (int n = warp; n < cnt; n += kHeadThreads / 32) {
      const float* tau = s_taup[n];
      float ss = 0.f;
      for (int ch = lane; ch < Mp; ch += 32) {
        float e = 0.f;
        if (ch < M) {
          e = tau[ch] * phi0[n * Mp + ch];
          if (two) e *= phi1[n * Mp + ch];
        }
        phi0[n * Mp + ch] = e;
        ss = fmaf(e, e, ss);
      }
      ss = warp_sum(ss);
      const float inv = rsqrtf(fmaxf(ss, kEps));
      for (int ch = lane; ch < Mp; ch += 32) phi0[n * Mp + ch] *= inv;
    }
    const int os = two ? OS_SAMEPROP : OS_DESCRIBE;
    fin = phi0; fpitch = Mp; fL = M; Wo = md.out_w[os]; bo = md.out_b[os];
    if (c.ehat != nullptr) {   // many classes: the product runs as a GEMM over all roots
      __syncthreads();
      for (int i = threadIdx.x; i < cnt * Mp; i += kHeadThreads) {
        const int n = i / Mp, ch = i - n * Mp;
        const float v = phi0[n * Mp + ch];
        c.ehat[(size_t)(wk.first + n) * Mp + ch] = v;
        if (c.ehat_lo != nullptr)
          c.ehat_lo[(size_t)(wk.first + n) * Mp + ch] =
              v - __uint_as_float(__float_as_uint(v) & 0xffffe000u);
      }
      if (threadIdx.x < cnt) c.ehat_dst[wk.first + threadIdx.x] = s_outp[threadIdx.x];
      return;
    }
  } else {
    // ---- Exist / Count / EqualNum / MoreNum / LessNum (nmn3_modules.py:258-400; SHAPES Answer):
    //      z = [min, mean, max] or [att(HW), min, max] (x2) from the root's input maps
    float* z = Fs;
    const int zp = (2 * (HW + 2) + 3) & ~3;
    const bool exist = (wk.op == OP_EXIST);
    for (int n = warp; n < cnt; n += kHeadThreads / 32) {
      for (int which = 0; which < (two ? 2 : 1); ++which) {
        const float* a = s_rowp[which][n];
        float* zo = z + n * zp + which * (HW + 2);
        float mn = INFINITY, mx = -INFINITY, sm = 0.f;
        for (int p = lane; p < HW; p += 32) {
          const float v = __ldg(a + p);
          if (!exist) zo[p] = v;
          mn = fminf(mn, v); mx = fmaxf(mx, v); sm += v;
        }
        mn = warp_min(mn); mx = warp_max(mx); sm = warp_sum(sm);
        if (lane == 0) {
          if (exist) { zo[0] = mn; zo[1] = sm / (float)HW; zo[2] = mx; }
          else { zo[HW] = mn; zo[HW + 1] = mx; }
        }
      }
    }
    const int set = exist ? SS_EXIST : (wk.op == OP_COUNT) ? SS_COUNT
                  : (wk.op == OP_EQUAL_NUM) ? SS_EQUAL : (wk.op == OP_MORE_NUM) ? SS_MORE : SS_LESS;
    fin = z; fpitch = zp; fL = exist ? 3 : (two ? 2 * (HW + 2) : HW + 2);
    Wo = md.sc_w[set]; bo = md.sc_b[set];
  }
  __syncthreads();

  // ---- scores = in·W + b (fc_eltwise / fc_scores)
  if (C <= 32) {
    // warp w < 8 takes the rows k ≡ w (mod 8), lane = class; partial sums meet in `scratch`
    if (warp < 8) {
      float acc[NN];
#pragma unroll
      for (int n = 0; n < NN; ++n) acc[n] = 0.f;
      if (lane < C) {
#pragma unroll 4
        for (int k = warp; k < fL; k += 8) {
          const float w = __ldg(Wo + (size_t)k * C + lane);
#pragma unroll
          for (int n = 0; n < NN; ++n) acc[n] = fmaf(fin[n * fpitch + k], w, acc[n]);
        }
      }
#pragma unroll
      for (int n = 0; n < NN; ++n) scratch[(warp * kHeadNodesMax + n) * 32 + lane] = acc[n];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < cnt * 32; i += kHeadThreads) {
      const int n = i >> 5, cl = i & 31;
      if (cl < C) {
        float v = bo[cl];
#pragma unroll
        for (int w = 0; w < 8; ++w) v += scratch[(w * kHeadNodesMax + n) * 32 + cl];
        s_outp[n][cl] = v;
      }
    }
  } else {
    for (int cl = threadIdx.x; cl < C; cl += kHeadThreads) {
      float acc[NN];
#pragma unroll
      for (int n = 0; n < NN; ++n) acc[n] = 0.f;
#pragma unroll 16
      for (int k = 0; k < fL; ++k) {
        const float w = __ldg(Wo + (size_t)k * C + cl);
#pragma unroll
        for (int n = 0; n < NN; ++n) acc[n] = fmaf(fin[n * fpitch + k], w, acc[n]);
      }
      const float b = bo[cl];
#pragma unroll
      for (int n = 0; n < NN; ++n)
        if (n < cnt) s_outp[n][cl] = acc[n] + b;
    }
  }
}

}  // namespace n2nmn
