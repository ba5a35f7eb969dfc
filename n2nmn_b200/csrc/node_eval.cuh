// K3, wave form: evaluation of ONE expression-tree node by one CTA through the global attention
// arena, and wave_kernel = one CTA per node of one tree depth across the whole batch — the
// depth-bucketed waves that replace TF Fold's dynamic batching (models_clevr/nmn3_model.py:49-159,
// SURVEY.md §3.5). Also backs the per-module entry point (n2nmn_module_fwd). The default executor
// (tree_kernel.cuh) shares the building blocks below.
//
// Find / Filter reach these kernels with their "find" map already in the arena (fused epilogue
// of the projection kernel); FindSameProperty / Describe / SameProperty with their stored
// tensor-core maps in mbuf.
#pragma once
#include <cooperative_groups.h>

#include "common.cuh"

namespace n2nmn {

namespace cg = cooperative_groups;

struct NodeCtx {
  DevModel md;
  TextBufs tb;
  float* arena;        // [slots][HW]
  float* scores;       // segment 0: [rows][C]
  float* scores_seg[kMaxSeg];
  int score_rows;      // score rows per segment (a huge value when there is one segment)
  const float* mbuf;   // [mslots][HW][Mp]
  // schedules with pooled_direct (Describe / SameProperty roots): tree kernel -> pool_att
  // [rows][HWp] softmaxed attention weights -> pool kernel -> pooled [rows][pool_pitch] feature
  // vectors -> head kernel -> scores
  float* pool_att;
  float* pooled;
  int pool_pitch;
  // training: the attended feature vectors phi of the Describe / SameProperty roots, kept for the
  // backward pass, [score row][2][Mp] (nullptr outside training)
  float* phi_out;
  // answer heads with many classes (VQA: 3001): head_kernel leaves the normalised vector ê of
  // root r (its position in the head list) in ehat[r][Mp] and the address of its score row in
  // ehat_dst[r]; head_tail_wgmma_kernel does the fc_eltwise product as one GEMM (nullptr otherwise)
  float* ehat;
  float* ehat_lo;      // ê - trunc_tf32(ê) for the wgmma tail (head_tail_wgmma.cuh), or nullptr
  float** ehat_dst;
};

// score row of question / call row q (numbered across the segments)
__device__ __forceinline__ float* score_row(const NodeCtx& c, int q) {
  const int seg = q / c.score_rows;
  return c.scores_seg[seg] + (size_t)(q - seg * c.score_rows) * c.md.C;
}

constexpr int kNodeScratch = 2048;   // floats

// Shared-memory carve-up (floats); the host computes the same layout to size the launch.
constexpr int kHeadCapFloats = 12288;   // answer-head weights are staged in smem up to 48 KB

struct NodeSmem {
  int HWp, pad, v, z, k, head, total;
};
__host__ __device__ inline NodeSmem node_smem_layout(int H, int W, int Mp, int ksize, int M,
                                                     int C) {
  NodeSmem s;
  const int HW = H * W;
  s.HWp = (HW + 3) & ~3;
  s.pad = ((H + ksize - 1) * (W + ksize - 1) + 3) & ~3;
  s.v = 5 * Mp;                      // v0 v1 v2 + two partial-sum buffers
  s.z = (2 * (HW + 2) + 3) & ~3;
  s.k = ksize * ksize * Mp;
  const int rows = (2 * (HW + 2) > M) ? 2 * (HW + 2) : M;
  s.head = (rows * C <= kHeadCapFloats) ? ((rows * C + 3) & ~3) : 0;
  s.total = 2 * s.HWp + s.pad + kNodeScratch + s.v + 64 + s.z + s.k + s.head;
  return s;
}

struct SmemPtrs {
  float *a0, *a1, *pad, *scratch, *v0, *v1, *v2, *part0, *part1, *red, *z, *k, *head;
  bool k_ready;        // conv filter bank already staged in k
  const float* head_w; // staged answer-head weights (nullptr: read them from global memory)
};
__device__ __forceinline__ SmemPtrs carve(float* base, const DevModel& md) {
  const NodeSmem L = node_smem_layout(md.H, md.W, md.Mp, md.ksize, md.M, md.C);
  SmemPtrs s;
  s.a0 = base;
  s.a1 = s.a0 + L.HWp;
  s.pad = s.a1 + L.HWp;
  s.scratch = s.pad + L.pad;
  s.v0 = s.scratch + kNodeScratch;
  s.v1 = s.v0 + md.Mp;
  s.v2 = s.v1 + md.Mp;
  s.part0 = s.v2 + md.Mp;
  s.part1 = s.part0 + md.Mp;
  s.red = s.part1 + md.Mp;
  s.z = s.red + 64;
  s.k = s.z + L.z;
  s.head = L.head ? s.k + L.k : nullptr;
  s.k_ready = false;
  s.head_w = nullptr;
  return s;
}

// ---- asynchronous global -> shared staging (cp.async; completes behind other work) --------------
__device__ __forceinline__ void cp_async_4(float* dst, const float* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;"
               ::"r"((uint32_t)__cvta_generic_to_shared(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_16(float* dst, const float* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;"
               ::"r"((uint32_t)__cvta_generic_to_shared(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit_wait_all() {
  asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
}
// n floats, issued by the whole CTA; 16-byte chunks when both sides allow it.
__device__ __forceinline__ void stage_async(float* dst, const float* src, int n) {
  const bool wide = ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0
                    && (n & 3) == 0;
  if (wide) {
    for (int i = threadIdx.x * 4; i < n; i += blockDim.x * 4) cp_async_16(dst + i, src + i);
  } else {
    for (int i = threadIdx.x; i < n; i += blockDim.x) cp_async_4(dst + i, src + i);
  }
}

// Position of this CTA inside the cluster that evaluates the node.
struct Coop {
  int rank, size;
  __device__ __forceinline__ void sync() const {
    if (size > 1) cg::this_cluster().sync();   // also orders global + distributed-smem traffic
    else __syncthreads();
  }
  __device__ __forceinline__ const float* peer(const float* p, int r) const {
    return (size > 1) ? cg::this_cluster().map_shared_rank(const_cast<float*>(p), r) : p;
  }
};

// ---- building blocks ---------------------------------------------------------------------------
__device__ __forceinline__ void load_att(float* dst, const float* arena, int slot, int HW) {
  const float* src = arena + (size_t)slot * HW;
  for (int p = threadIdx.x; p < HW; p += blockDim.x) dst[p] = src[p];
}

// tf.nn.softmax over the flattened map (models_clevr/nmn3_modules.py:170-172), in place.
__device__ __forceinline__ void softmax_inplace(float* a, int HW, float* red) {
  float mx = -INFINITY;
  for (int p = threadIdx.x; p < HW; p += blockDim.x) mx = fmaxf(mx, a[p]);
  mx = block_reduce<1>(mx, red);
  float sum = 0.f;
  for (int p = threadIdx.x; p < HW; p += blockDim.x) {
    const float e = expf(a[p] - mx);
    a[p] = e;
    sum += e;
  }
  sum = block_reduce<0>(sum, red);
  for (int p = threadIdx.x; p < HW; p += blockDim.x) a[p] = a[p] / sum;
  __syncthreads();
}

// This CTA's share [q0, q1) of `n` items split evenly over the cluster.
__device__ __forceinline__ void coop_range(const Coop& co, int n, int& q0, int& q1) {
  const int per = (n + co.size - 1) / co.size;
  q0 = min(n, co.rank * per);
  q1 = min(n, q0 + per);
}

// part[c] = Σ_{k in [k0,k1)} in[k-k0] · W[k*Mp + c] for all c < Mp (W has row pitch Mp, zero
// padded). Threads form a (column quad, row slice) grid; row slices are reduced through scratch.
__device__ __forceinline__ void gemv_partial(const float* in, int k0, int k1,
                                             const float* __restrict__ W, int Mp, float* part,
                                             float* scratch) {
  const int quads = Mp >> 2, nthreads = blockDim.x;
  if (quads >= nthreads) {
    for (int q = threadIdx.x; q < quads; q += nthreads) {
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      const float4* w = reinterpret_cast<const float4*>(W) + q;
#pragma unroll 8
      for (int k = k0; k < k1; ++k) {
        const float4 wv = __ldg(w + (size_t)k * quads);
        const float x = in[k - k0];
        acc.x = fmaf(x, wv.x, acc.x); acc.y = fmaf(x, wv.y, acc.y);
        acc.z = fmaf(x, wv.z, acc.z); acc.w = fmaf(x, wv.w, acc.w);
      }
      reinterpret_cast<float4*>(part)[q] = acc;
    }
    __syncthreads();
    return;
  }
  int slices = nthreads / quads;
  if (slices * Mp > kNodeScratch) slices = kNodeScratch / Mp;
  const int q = threadIdx.x % quads, sl = threadIdx.x / quads;
  if (sl < slices) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    const float4* w = reinterpret_cast<const float4*>(W) + q;
#pragma unroll 8
    for (int k = k0 + sl; k < k1; k += slices) {
      const float4 wv = __ldg(w + (size_t)k * quads);
      const float x = in[k - k0];
      acc.x = fmaf(x, wv.x, acc.x); acc.y = fmaf(x, wv.y, acc.y);
      acc.z = fmaf(x, wv.z, acc.z); acc.w = fmaf(x, wv.w, acc.w);
    }
    reinterpret_cast<float4*>(scratch)[sl * quads + q] = acc;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < Mp; c += nthreads) {
    float s = 0.f;
    for (int k = 0; k < slices; ++k) s += scratch[k * Mp + c];
    part[c] = s;
  }
  __syncthreads();
}

// phi = fc_att(reduce_sum(image_feat_grid * softmax(att), [1,2])) (nmn3_modules.py:170-176) for one
// attention input, cooperatively over the cluster. The projection kernel has already stored
// G = X_b·W_att + b_att for the node's image, and Σ_p s_p = 1, so phi = Σ_p s_p·G[p,:]: the pixel
// rows of G are split over the CTAs and `part` receives this CTA's partial sums (all Mp columns).
// The caller exchanges the partials after a cluster sync (sum_partials).
__device__ __forceinline__ void pooled_fc_partial(const DevModel& md, const Coop& co,
                                                  const float* G, float* soft, float* part,
                                                  const SmemPtrs& s) {
  softmax_inplace(soft, md.HW, s.red);
  int p0, p1;
  coop_range(co, md.HW, p0, p1);
  gemv_partial(soft + p0, p0, p1, G, md.Mp, part, s.scratch);
}

// out[c] = bias[c] + Σ_ranks part_r[c] (c < M; zero beyond), reading the peers' partial buffers
// through distributed shared memory. Must be called after co.sync().
__device__ __forceinline__ void sum_partials(const Coop& co, const float* part,
                                             const float* __restrict__ bias, float* out, int M,
                                             int Mp) {
  for (int c = threadIdx.x; c < Mp; c += blockDim.x) {
    float v = 0.f;
    if (c < M) {
      v = bias ? bias[c] : 0.f;
      for (int r = 0; r < co.size; ++r) v += co.peer(part, r)[c];
    }
    out[c] = v;
  }
  __syncthreads();
}

// scores[c] = b[c] + Σ_k z[k]·W[k*C + c]: the fc('fc_scores') / fc('fc_eltwise') heads
// (nmn3_modules.py:278,302,334,450,493). Thread groups split k, 32 lanes span c.
__device__ __forceinline__ void small_fc(const float* z, int L, const float* __restrict__ W,
                                         const float* __restrict__ bias, int C, float* out,
                                         float* scratch) {
  const int lane = threadIdx.x & 31, g = threadIdx.x >> 5, G = blockDim.x >> 5;
  for (int c0 = 0; c0 < C; c0 += 32) {
    const int c = c0 + lane;
    float acc = 0.f;
    if (c < C) {
#pragma unroll 4
      for (int k = g; k < L; k += G) acc = fmaf(z[k], W[(size_t)k * C + c], acc);
    }
    scratch[g * 32 + lane] = acc;
    __syncthreads();
    if (g == 0 && c < C) {
      float s = bias[c];
      for (int j = 0; j < G; ++j) s += scratch[j * 32 + lane];
      out[c] = s;
    }
    __syncthreads();
  }
}

__device__ __forceinline__ void minmax(const float* a, int HW, float* red, float& mn, float& mx,
                                       float& sum) {
  float lmn = INFINITY, lmx = -INFINITY, ls = 0.f;
  for (int p = threadIdx.x; p < HW; p += blockDim.x) {
    const float v = a[p];
    lmn = fminf(lmn, v); lmx = fmaxf(lmx, v); ls += v;
  }
  mn = block_reduce<2>(lmn, red);
  mx = block_reduce<1>(lmx, red);
  sum = block_reduce<0>(ls, red);
}

// ---- the modules -------------------------------------------------------------------------------
template <int KS>
__device__ __forceinline__ void eval_transform(const NodeCtx& c, const NodeRec& nd,
                                               const SmemPtrs& s, const Coop& co) {
  // TransformModule, conv variant (models_clevr/nmn3_modules.py:185-216, SHAPES :71-101):
  // SAME cross-correlation of the 1-channel map with [KS,KS,1,M], ∘ text, l2norm over M, ·w2 + b2
  // Pixels are split over the cluster's warps; every CTA stages the (small) filter bank itself.
  const DevModel& md = c.md;
  const int H = md.H, W = md.W, HW = md.HW, M = md.M;
  const int PW = W + KS - 1, PH = H + KS - 1, R = (KS - 1) / 2;
  const int Mq = md.Mp;   // filter bank and vectors are padded to the row pitch (zeros)
  for (int i = threadIdx.x; i < PH * PW; i += blockDim.x) s.pad[i] = 0.f;
  __syncthreads();
  const float* src = c.arena + (size_t)nd.in0 * HW;
  for (int p = threadIdx.x; p < HW; p += blockDim.x) {
    const int y = p / W, x = p - y * W;
    s.pad[(y + R) * PW + x + R] = src[p];
  }
  if (!s.k_ready) stage_async(s.k, md.conv_k, KS * KS * Mq);
  const float* tau = c.tb.tau + (size_t)nd.text * md.Mp;
  for (int ch = threadIdx.x; ch < Mq; ch += blockDim.x) {
    const bool live = ch < M;
    s.v0[ch] = live ? tau[ch] : 0.f;
    s.v1[ch] = live ? md.elt_w[ES_TRANSFORM][ch] : 0.f;
    s.v2[ch] = live ? md.conv_b[ch] : 0.f;
  }
  cp_async_commit_wait_all();
  __syncthreads();
  const int lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  const int gwarp = co.rank * nwarps + (threadIdx.x >> 5), gwarps = co.size * nwarps;
  const float b2 = md.elt_b[ES_TRANSFORM][0];
  float* dst = c.arena + (size_t)nd.out * HW;
  for (int p = gwarp; p < HW; p += gwarps) {
    const int y = p / W, x = p - y * W;
    float win[KS * KS];
#pragma unroll
    for (int dy = 0; dy < KS; ++dy)
#pragma unroll
      for (int dx = 0; dx < KS; ++dx) win[dy * KS + dx] = s.pad[(y + dy) * PW + x + dx];
    float num = 0.f, den = 0.f;
    for (int c0 = lane * 4; c0 < Mq; c0 += 128) {
      float4 A = *reinterpret_cast<const float4*>(s.v2 + c0);
#pragma unroll
      for (int tap = 0; tap < KS * KS; ++tap) {
        const float4 k4 = *reinterpret_cast<const float4*>(s.k + tap * Mq + c0);
        A.x = fmaf(win[tap], k4.x, A.x); A.y = fmaf(win[tap], k4.y, A.y);
        A.z = fmaf(win[tap], k4.z, A.z); A.w = fmaf(win[tap], k4.w, A.w);
      }
      const float4 t4 = *reinterpret_cast<const float4*>(s.v0 + c0);
      const float4 w4 = *reinterpret_cast<const float4*>(s.v1 + c0);
      const float ex = A.x * t4.x, ey = A.y * t4.y, ez = A.z * t4.z, ew = A.w * t4.w;
      num = fmaf(ex, w4.x, num); num = fmaf(ey, w4.y, num);
      num = fmaf(ez, w4.z, num); num = fmaf(ew, w4.w, num);
      den = fmaf(ex, ex, den); den = fmaf(ey, ey, den);
      den = fmaf(ez, ez, den); den = fmaf(ew, ew, den);
    }
    num = warp_sum(num);
    den = warp_sum(den);
    if (lane == 0) dst[p] = num * rsqrtf(fmaxf(den, kEps)) + b2;
  }
}

__device__ __forceinline__ void eval_find_same_property(const NodeCtx& c, const NodeRec& nd,
                                                        const SmemPtrs& s, const Coop& co) {
  // FindSamePropertyModule (models_clevr/nmn3_modules.py:134-183) and the VQA TransformModule
  // (models_vqa/nmn3_modules.py:123-171): l2norm_c(m ∘ τ ∘ φ)·w2 + b2 with φ = fc_att(pooled).
  const DevModel& md = c.md;
  const int HW = md.HW, Mp = md.Mp, M = md.M;
  load_att(s.a0, c.arena, nd.in0, HW);
  __syncthreads();
  pooled_fc_partial(md, co, c.mbuf + (size_t)nd.aux2 * HW * Mp, s.a0, s.part0, s);
  co.sync();
  sum_partials(co, s.part0, nullptr, s.v0, M, Mp);
  const float* tauw = c.tb.tauw + (size_t)nd.text * Mp;   // τ∘w2
  const float* tau = c.tb.tau + (size_t)nd.text * Mp;
  for (int ch = threadIdx.x; ch < Mp; ch += blockDim.x) {
    const float phi = s.v0[ch];
    const float tp = tau[ch] * phi;
    s.v1[ch] = tauw[ch] * phi;   // coefficient of m in the numerator
    s.v2[ch] = tp * tp;          // coefficient of m² in the squared norm
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  const int gwarp = co.rank * nwarps + (threadIdx.x >> 5), gwarps = co.size * nwarps;
  const float b2 = md.elt_b[ES_FSP][0];
  const float* mimg = c.mbuf + (size_t)nd.aux * HW * Mp;
  float* dst = c.arena + (size_t)nd.out * HW;
  for (int p = gwarp; p < HW; p += gwarps) {
    const float4* mrow = reinterpret_cast<const float4*>(mimg + (size_t)p * Mp);
    float num = 0.f, den = 0.f;
    for (int q = lane; q < (Mp >> 2); q += 32) {
      const float4 m = __ldg(mrow + q);
      const float4 a = reinterpret_cast<const float4*>(s.v1)[q];
      const float4 d = reinterpret_cast<const float4*>(s.v2)[q];
      num = fmaf(m.x, a.x, num); num = fmaf(m.y, a.y, num);
      num = fmaf(m.z, a.z, num); num = fmaf(m.w, a.w, num);
      den = fmaf(m.x * m.x, d.x, den); den = fmaf(m.y * m.y, d.y, den);
      den = fmaf(m.z * m.z, d.z, den); den = fmaf(m.w * m.w, d.w, den);
    }
    num = warp_sum(num);
    den = warp_sum(den);
    if (lane == 0) dst[p] = num * rsqrtf(fmaxf(den, kEps)) + b2;
  }
}

__device__ __forceinline__ void normalize_and_score(const NodeCtx& c, const NodeRec& nd,
                                                    const SmemPtrs& s, float* e, int out_set) {
  // tf.nn.l2_normalize(e, 1) then fc('fc_eltwise') (nmn3_modules.py:448-450, 491-493)
  const DevModel& md = c.md;
  float ss = 0.f;
  for (int ch = threadIdx.x; ch < md.M; ch += blockDim.x) ss = fmaf(e[ch], e[ch], ss);
  ss = block_reduce<0>(ss, s.red);
  const float inv = rsqrtf(fmaxf(ss, kEps));
  for (int ch = threadIdx.x; ch < md.M; ch += blockDim.x) e[ch] *= inv;
  __syncthreads();
  small_fc(e, md.M, s.head_w ? s.head_w : md.out_w[out_set], md.out_b[out_set], md.C,
           score_row(c, nd.out), s.scratch);
}

__device__ __forceinline__ void eval_describe(const NodeCtx& c, const NodeRec& nd,
                                              const SmemPtrs& s, const Coop& co) {
  // DescribeModule (models_clevr/nmn3_modules.py:454-495, VQA models_vqa/nmn3_modules.py:193-240)
  const DevModel& md = c.md;
  load_att(s.a0, c.arena, nd.in0, md.HW);
  __syncthreads();
  pooled_fc_partial(md, co, c.mbuf + (size_t)nd.aux * md.HW * md.Mp, s.a0, s.part0, s);
  co.sync();
  if (co.rank != 0) return;   // the tail is tiny: one CTA finishes it
  sum_partials(co, s.part0, nullptr, s.v0, md.M, md.Mp);
  const float* tau = c.tb.tau + (size_t)nd.text * md.Mp;
  for (int ch = threadIdx.x; ch < md.M; ch += blockDim.x) s.v1[ch] = tau[ch] * s.v0[ch];
  __syncthreads();
  normalize_and_score(c, nd, s, s.v1, OS_DESCRIBE);
}

__device__ __forceinline__ void eval_same_property(const NodeCtx& c, const NodeRec& nd,
                                                   const SmemPtrs& s, const Coop& co) {
  // SamePropertyModule (models_clevr/nmn3_modules.py:402-452)
  const DevModel& md = c.md;
  load_att(s.a0, c.arena, nd.in0, md.HW);
  load_att(s.a1, c.arena, nd.in1, md.HW);
  __syncthreads();
  const size_t map_floats = (size_t)md.HW * md.Mp;
  pooled_fc_partial(md, co, c.mbuf + nd.aux * map_floats, s.a0, s.part0, s);
  pooled_fc_partial(md, co, c.mbuf + nd.aux2 * map_floats, s.a1, s.part1, s);
  co.sync();
  if (co.rank != 0) return;
  sum_partials(co, s.part0, nullptr, s.v0, md.M, md.Mp);
  sum_partials(co, s.part1, nullptr, s.v1, md.M, md.Mp);
  const float* tau = c.tb.tau + (size_t)nd.text * md.Mp;
  for (int ch = threadIdx.x; ch < md.M; ch += blockDim.x)
    s.v2[ch] = s.v0[ch] * tau[ch] * s.v1[ch];
  __syncthreads();
  normalize_and_score(c, nd, s, s.v2, OS_SAMEPROP);
}

__device__ __forceinline__ void eval_small_answer(const NodeCtx& c, const NodeRec& nd,
                                                  const SmemPtrs& s) {
  // Exist / Count / EqualNum / MoreNum / LessNum (models_clevr/nmn3_modules.py:258-400)
  const DevModel& md = c.md;
  const int HW = md.HW;
  float mn, mx, sum;
  int L, set;
  if (nd.op == OP_EXIST) {
    load_att(s.a0, c.arena, nd.in0, HW);
    __syncthreads();
    minmax(s.a0, HW, s.red, mn, mx, sum);
    if (threadIdx.x == 0) { s.z[0] = mn; s.z[1] = sum / (float)HW; s.z[2] = mx; }
    L = 3; set = SS_EXIST;
  } else {
    const int two = (nd.op != OP_COUNT);
    load_att(s.z, c.arena, nd.in0, HW);
    if (two) load_att(s.z + HW + 2, c.arena, nd.in1, HW);
    __syncthreads();
    minmax(s.z, HW, s.red, mn, mx, sum);
    if (threadIdx.x == 0) { s.z[HW] = mn; s.z[HW + 1] = mx; }
    if (two) {
      minmax(s.z + HW + 2, HW, s.red, mn, mx, sum);
      if (threadIdx.x == 0) { s.z[2 * HW + 2] = mn; s.z[2 * HW + 3] = mx; }
    }
    L = two ? 2 * (HW + 2) : HW + 2;
    set = (nd.op == OP_COUNT) ? SS_COUNT : (nd.op == OP_EQUAL_NUM) ? SS_EQUAL
        : (nd.op == OP_MORE_NUM) ? SS_MORE : SS_LESS;
  }
  __syncthreads();
  small_fc(s.z, L, s.head_w ? s.head_w : md.sc_w[set], md.sc_b[set], md.C,
           score_row(c, nd.out), s.scratch);
}

// Evaluates one node with the CTAs of `co`. Every CTA of the cluster must call it (the heavy
// modules contain cluster barriers); the caller synchronises the cluster afterwards.
template <int KS>
__device__ __forceinline__ void eval_node(const NodeCtx& c, const NodeRec& nd, const SmemPtrs& s,
                                          const Coop& co) {
  const int HW = c.md.HW;
  const int gtid = co.rank * blockDim.x + threadIdx.x, gthreads = co.size * blockDim.x;
  switch (nd.op) {
    case OP_SCENE: {   // models_clevr/nmn3_modules.py:60-72; aux carries pos_val's bits
      float* dst = c.arena + (size_t)nd.out * HW;
      const float v = __int_as_float(nd.aux);
      for (int p = gtid; p < HW; p += gthreads) dst[p] = v;
      break;
    }
    case OP_FIND:      // already written by the projection kernel's epilogue
      break;
    case OP_FILTER: {  // min(input_0, Find(t,b)) (nmn3_modules.py:129-130); find part is in `out`
      float* dst = c.arena + (size_t)nd.out * HW;
      const float* a = c.arena + (size_t)nd.in0 * HW;
      for (int p = gtid; p < HW; p += gthreads) dst[p] = fminf(a[p], dst[p]);
      break;
    }
    case OP_AND:       // tf.minimum / tf.maximum (nmn3_modules.py:233,253)
    case OP_OR: {
      float* dst = c.arena + (size_t)nd.out * HW;
      const float* a = c.arena + (size_t)nd.in0 * HW;
      const float* b = c.arena + (size_t)nd.in1 * HW;
      for (int p = gtid; p < HW; p += gthreads)
        dst[p] = (nd.op == OP_AND) ? fminf(a[p], b[p]) : fmaxf(a[p], b[p]);
      break;
    }
    case OP_TRANSFORM: eval_transform<KS>(c, nd, s, co); break;
    case OP_FIND_SAME_PROPERTY: eval_find_same_property(c, nd, s, co); break;
    case OP_DESCRIBE: cp_async_commit_wait_all(); eval_describe(c, nd, s, co); break;
    case OP_SAME_PROPERTY: cp_async_commit_wait_all(); eval_same_property(c, nd, s, co); break;
    default:
      if (co.rank == 0) { cp_async_commit_wait_all(); eval_small_answer(c, nd, s); }
      break;
  }
}

// One CTA per node of one wave.
template <int KS>
__global__ void __launch_bounds__(kNodeThreads)
wave_kernel(const NodeCtx c, const NodeRec* __restrict__ nodes,
            const int32_t* __restrict__ wave_nodes, int first) {
  extern __shared__ __align__(16) float node_smem[];
  const SmemPtrs s = carve(node_smem, c.md);   // nothing pre-staged: parameters come from L2
  pdl_wait();
  const NodeRec nd = nodes[wave_nodes[first + blockIdx.x]];
  Coop co;
  co.rank = 0; co.size = 1;
  eval_node<KS>(c, nd, s, co);
}

}  // namespace n2nmn
