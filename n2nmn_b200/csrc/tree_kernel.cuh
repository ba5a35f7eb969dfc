// K3 (default executor): one thread-block cluster per question walks the question's nodes in
// Reverse-Polish order, keeping every live attention map of the question in SHARED memory.
//
// Why it looks like this: a question is a chain of 2-6 tiny dependent steps; what bounds it is
// latency (L2 round trips, barriers), not bandwidth or arithmetic. So
//   * the attention "stack" lives in smem, replicated in every CTA of the cluster — the cheap
//     modules (Scene / Filter / And / Or / Transform) are recomputed redundantly by every CTA and
//     need no cluster barrier and no global memory at all;
//   * TransformModule is evaluated as a per-node quadratic form over the 5x5 window (common.cuh):
//     its coefficients come from the text kernel, a pixel costs 377 FMAs, there is no filter bank
//     in shared memory;
//   * launch-table records, the Find maps produced by the projection kernel and the text vectors
//     are fetched with cp.async in the prologue, behind PDL;
//   * only FindSameProperty is split over the cluster (pooled fc_att by rows of the stored map,
//     then pixels), pieces exchanged through double-buffered distributed shared memory with ONE
//     cluster barrier per exchange;
//   * evaluation (kDirect): the kernel produces ATTENTION ONLY. The inputs of every answer root go
//     to the pooled-attention buffer and the batched head kernel (head_kernel.cuh) computes all
//     seven answer modules for many questions at once; the training / compiled-schedule form
//     (kDirect = false) finishes the answer modules here, from stored fc_att maps.
// With many batches in flight the pool launches ONE CTA per question (no cluster barriers at
// all): less latency hiding per question, more questions per second (DESIGN.md §9).
// Results agree with wave_kernel / eval_node (node_eval.cuh) up to fp32 summation order.
#pragma once
#include "node_eval.cuh"

namespace n2nmn {

constexpr int kTreeWriteArena = 1;     // launch flags
constexpr int kTreeFp32Stencil = 2;    // (kept for ABI stability: Transform is always fp32 now)
constexpr int kTreeFindSlots = 10;   // Find / Filter maps prefetched per question
constexpr int kTreeNodeCap = 48;     // node records of one question kept in smem
constexpr int kTreeTextCap = 4;      // text vectors (tau, tau∘w2) of one question prefetched
constexpr int kTreeQuadCap = 4;      // Transform coefficient rows of one question prefetched

struct TreeSmem {
  int HWp, stack, ftmp, outbuf, pad, v, part, z, head, nodes, tvec, quad, total;
};
// `direct`: the evaluation form (no answer heads here: no head weights, no z vector)
__host__ __device__ inline TreeSmem tree_smem_layout(int H, int W, int Mp, int ksize, int M, int C,
                                                     int stack_slots, bool direct = false) {
  TreeSmem s;
  const int HW = H * W;
  s.HWp = (HW + 3) & ~3;
  s.stack = stack_slots * s.HWp;
  s.ftmp = kTreeFindSlots * s.HWp;
  s.outbuf = 2 * s.HWp;
  s.pad = ((H + ksize - 1) * (W + ksize - 1) + 3) & ~3;   // zero-padded map of a Transform input
  s.v = 3 * Mp;
  s.part = 4 * Mp;
  s.z = direct ? 0 : ((2 * (HW + 2) + 3) & ~3);
  const int rows = (2 * (HW + 2) > M) ? 2 * (HW + 2) : M;
  s.head = (!direct && rows * C <= kHeadCapFloats) ? ((rows * C + 3) & ~3) : 0;
  s.nodes = kTreeNodeCap * (int)(sizeof(NodeRec) / sizeof(float));
  s.tvec = (Mp <= 512) ? kTreeTextCap * 2 * Mp : 0;
  s.quad = (ksize > 1) ? kTreeQuadCap * quad_pitch(ksize) : 0;
  s.total = s.stack + s.ftmp + s.outbuf + 2 * s.HWp + s.pad + kNodeScratch + s.v + s.part + 64 +
            s.z + s.head + s.nodes + s.tvec + s.quad;
  return s;
}

struct TreePtrs {
  float *stack, *ftmp, *outbuf, *a0, *a1, *pad, *scratch, *v0, *v1, *v2, *part, *red, *z, *head;
  int HWp, Mp;
};

// softmax of one map by a single warp (HW is a few hundred at most), in place.
__device__ __forceinline__ void warp_softmax(float* a, int HW) {
  const int lane = threadIdx.x & 31;
  float mx = -INFINITY;
  for (int p = lane; p < HW; p += 32) mx = fmaxf(mx, a[p]);
  mx = warp_max(mx);
  float sum = 0.f;
  for (int p = lane; p < HW; p += 32) {
    const float e = expf(a[p] - mx);
    a[p] = e;
    sum += e;
  }
  sum = warp_sum(sum);
  for (int p = lane; p < HW; p += 32) a[p] = a[p] / sum;
}

// min / max / sum of one map by a single warp.
__device__ __forceinline__ void warp_minmax(const float* a, int HW, float& mn, float& mx,
                                            float& sum) {
  const int lane = threadIdx.x & 31;
  float lmn = INFINITY, lmx = -INFINITY, ls = 0.f;
  for (int p = lane; p < HW; p += 32) {
    const float v = a[p];
    lmn = fminf(lmn, v); lmx = fmaxf(lmx, v); ls += v;
  }
  mn = warp_min(lmn); mx = warp_max(lmx); sum = warp_sum(ls);
}

// After a pixel-split phase and its cluster barrier: assemble the full map in the local stack.
// Work unit u (a pixel, or a horizontal run of `run` pixels) was done by global warp u % gwarps.
__device__ __forceinline__ void gather_pixels(const Coop& co, const float* outbuf, float* dst,
                                              int HW, int W, int run) {
  const int nwarps = blockDim.x >> 5, gwarps = co.size * nwarps;
  const int runs_x = (W + run - 1) / run;
  for (int p = threadIdx.x; p < HW; p += blockDim.x) {
    const int y = p / W, x = p - y * W;
    const int unit = (run == 1) ? p : y * runs_x + x / run;
    dst[p] = co.peer(outbuf, (unit % gwarps) / nwarps)[p];
  }
}

// ---- Transform as a quadratic form (common.cuh) ----------------------------------------------------
// pad: zero-padded input map [(H+KS-1)][(W+KS-1)]; q: the node's coefficients from the text kernel
// (u[n] then the upper triangle of Q row by row); out[p] = num·rsqrt(max(den, eps)) + b2
// (l2_normalize + conv_eltwise of models_clevr/nmn3_modules.py:211-214). One thread per pixel,
// n + n(n+1)/2 FMAs each, all operands in registers / broadcast shared-memory reads.
template <int KS>
__device__ __forceinline__ void transform_quad(const float* pad, const float* q, float b2,
                                               float* out, int Hh, int Ww) {
  constexpr int N = KS * KS + 1;
  const int PW = Ww + KS - 1, HW = Hh * Ww;
  for (int p = threadIdx.x; p < HW; p += blockDim.x) {
    const int y = p / Ww, x = p - y * Ww;
    float w[N];
#pragma unroll
    for (int dy = 0; dy < KS; ++dy)
#pragma unroll
      for (int dx = 0; dx < KS; ++dx) w[dy * KS + dx] = pad[(y + dy) * PW + x + dx];
    w[N - 1] = 1.f;
    float num = 0.f, den = 0.f;
#pragma unroll
    for (int i = 0; i < N; ++i) num = fmaf(w[i], q[i], num);
    int idx = (N + 3) & ~3;   // quad_u_pitch
#pragma unroll
    for (int i = 0; i < N; ++i) {
      float row = 0.f;
#pragma unroll
      for (int j = i; j < N; ++j) row = fmaf(w[j], q[idx++], row);
      den = fmaf(w[i], row, den);
    }
    out[p] = num * rsqrtf(fmaxf(den, kEps)) + b2;
  }
}

// kDirect: evaluation schedules with pooled_direct — answer roots only hand their (softmaxed, for
// the pooled modules) input maps to the head kernel (head_kernel.cuh).
template <int KS, bool kDirect>
__global__ void __launch_bounds__(kNodeThreads, kDirect ? 3 : 2)
tree_kernel(const NodeCtx c, const NodeRec* __restrict__ nodes, const int32_t* __restrict__ q_ptr,
            int csize, int stack_slots, int flags) {
  const bool write_arena = (flags & kTreeWriteArena) != 0;
  extern __shared__ __align__(16) float tree_smem[];
  const DevModel& md = c.md;
  const int HW = md.HW, Mp = md.Mp, M = md.M;
  const TreeSmem L = tree_smem_layout(md.H, md.W, Mp, md.ksize, M, md.C, stack_slots, kDirect);
  TreePtrs s;
  s.HWp = L.HWp; s.Mp = Mp;
  s.stack = tree_smem;
  s.ftmp = s.stack + L.stack;
  s.outbuf = s.ftmp + L.ftmp;
  s.a0 = s.outbuf + L.outbuf;
  s.a1 = s.a0 + L.HWp;
  s.pad = s.a1 + L.HWp;
  s.scratch = s.pad + L.pad;
  s.v0 = s.scratch + kNodeScratch;
  s.v1 = s.v0 + Mp;
  s.v2 = s.v1 + Mp;
  s.part = s.v2 + Mp;
  s.red = s.part + L.part;
  s.z = s.red + 64;
  s.head = L.head ? s.z + L.z : nullptr;
  NodeRec* s_nodes = reinterpret_cast<NodeRec*>(s.z + L.z + L.head);
  float* s_tvec = reinterpret_cast<float*>(s_nodes) + L.nodes;    // [kTreeTextCap][2][Mp]
  float* s_quad = s_tvec + L.tvec;                                  // [kTreeQuadCap][quad_pitch]
  const int qp = quad_pitch(KS);

  Coop co;
  co.size = csize;
  co.rank = (csize > 1) ? (int)cg::this_cluster().block_rank() : 0;
  const int q = blockIdx.x / csize;
  const int beg = q_ptr[q], end = q_ptr[q + 1];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int gwarp = co.rank * nwarps + warp, gwarps = co.size * nwarps;

  // ---- prologue part 1: launch tables and weights only (overlaps the predecessors)
  const float* head_w = nullptr;
  const bool nodes_in_smem = (end - beg) <= kTreeNodeCap;
  if (beg < end) {
    if (nodes_in_smem) {   // node records: the loop below must not wait on L2 after pdl_wait
      const int nwords = (end - beg) * (int)(sizeof(NodeRec) / 4);
      const int32_t* src = reinterpret_cast<const int32_t*>(nodes + beg);
      int32_t* dst = reinterpret_cast<int32_t*>(s_nodes);
      for (int j = threadIdx.x; j < nwords; j += blockDim.x) dst[j] = src[j];
    }
    if (!kDirect && co.rank == 0 && s.head != nullptr) {
      const int rop = nodes[end - 1].op;
      const float* w = nullptr;
      int rows = 0;
      switch (rop) {
        case OP_EXIST: w = md.sc_w[SS_EXIST]; rows = 3; break;
        case OP_COUNT: w = md.sc_w[SS_COUNT]; rows = HW + 2; break;
        case OP_EQUAL_NUM: w = md.sc_w[SS_EQUAL]; rows = 2 * (HW + 2); break;
        case OP_MORE_NUM: w = md.sc_w[SS_MORE]; rows = 2 * (HW + 2); break;
        case OP_LESS_NUM: w = md.sc_w[SS_LESS]; rows = 2 * (HW + 2); break;
        case OP_SAME_PROPERTY: w = md.out_w[OS_SAMEPROP]; rows = M; break;
        case OP_DESCRIBE: w = md.out_w[OS_DESCRIBE]; rows = M; break;
        default: break;
      }
      if (w) { stage_async(s.head, w, rows * md.C); head_w = s.head; }
    }
  }
  // ---- the attention arena, stored maps and text projections come from the preceding kernels
  pdl_wait();
  // the node records staged above are read by every thread below. (A CTA of the first wave sits in
  // pdl_wait long enough for the writes to land; a CTA that starts after the predecessor has
  // finished does not — without this barrier the questions of the second wave read stale records:
  // tools/dbg_group.py, r2.)
  __syncthreads();
  if (beg == end) {   // invalid layout: zeros(num_choices) (models_clevr/nmn3_model.py:144-155)
    if (co.rank == 0)
      for (int i = threadIdx.x; i < md.C; i += blockDim.x) score_row(c, q)[i] = 0.f;
    return;
  }
  // ---- prologue part 2: the question's Find maps (written by the projection kernel's epilogue),
  //      the text vectors of its FindSameProperty / pooled nodes and the quadratic-form
  //      coefficients of its Transform nodes (written by the text kernel)
  const NodeRec* qnodes = nodes_in_smem ? s_nodes : nodes + beg;
  {
    int nf = 0, nt = 0, nq = 0;
    for (int i = beg; i < end; ++i) {
      const int op = qnodes[i - beg].op;
      const bool wants_tau = op == OP_FIND_SAME_PROPERTY ||
                             (!kDirect && (op == OP_DESCRIBE || op == OP_SAME_PROPERTY));
      if (L.tvec && nt < kTreeTextCap && wants_tau) {
        const size_t row = (size_t)qnodes[i - beg].text * Mp;
        stage_async(s_tvec + (nt * 2) * Mp, c.tb.tau + row, Mp);
        stage_async(s_tvec + (nt * 2 + 1) * Mp, c.tb.tauw + row, Mp);
        ++nt;
      }
      if (op == OP_TRANSFORM && KS > 1 && nq < kTreeQuadCap) {
        stage_async(s_quad + nq * qp, c.tb.tq + (size_t)qnodes[i - beg].text * qp, qp);
        ++nq;
      }
      if (op == OP_FIND || op == OP_FILTER) {   // staged apart: stack slots are reused over time
        if (nf < kTreeFindSlots)
          stage_async(s.ftmp + nf * L.HWp, c.arena + (size_t)nodes[i].out * HW, HW);
        ++nf;
      }
    }
    cp_async_commit_wait_all();
    __syncthreads();
  }

  int exch = 0;        // cluster exchanges so far: selects the double-buffered outbuf / part half
  int nfilter = 0, ntext = 0, nquad = 0;
  for (int i = beg; i < end; ++i) {
    const NodeRec nd = qnodes[i - beg];
    // text vectors of this node: prefetched copy if it got a slot, else straight from L2
    const float* tau = nullptr;
    const float* tauw = nullptr;
    if (nd.op == OP_FIND_SAME_PROPERTY ||
        (!kDirect && (nd.op == OP_DESCRIBE || nd.op == OP_SAME_PROPERTY))) {
      if (L.tvec && ntext < kTreeTextCap) {
        tau = s_tvec + (ntext * 2) * Mp;
        tauw = tau + Mp;
      } else {
        tau = c.tb.tau + (size_t)nd.text * Mp;
        tauw = c.tb.tauw + (size_t)nd.text * Mp;
      }
      ++ntext;
    }
    float* out = (nd.so >= 0) ? s.stack + nd.so * L.HWp : nullptr;
    const float* in0 = (nd.s0 >= 0) ? s.stack + nd.s0 * L.HWp : nullptr;
    const float* in1 = (nd.s1 >= 0) ? s.stack + nd.s1 * L.HWp : nullptr;
    if (kDirect && nd.op >= OP_EXIST) {
      // answer root: its input maps go to the head kernel. Describe / SameProperty pool the image
      // features with softmax(att) (models_clevr/nmn3_modules.py:432-440, 482-487): the softmax is
      // done here, the weighted feature sum by the pool kernel.
      const bool two = nd.aux2 >= 0;
      const bool soft = (nd.op == OP_DESCRIBE || nd.op == OP_SAME_PROPERTY);
      if (co.rank == 0) {
        const float* src0 = in0;
        const float* src1 = in1;
        if (soft) {
          for (int p = threadIdx.x; p < HW; p += blockDim.x) {
            s.a0[p] = in0[p];
            if (two) s.a1[p] = in1[p];
          }
          __syncthreads();
          if (warp == 0) warp_softmax(s.a0, HW);
          if (two && warp == 1) warp_softmax(s.a1, HW);
          __syncthreads();
          src0 = s.a0; src1 = s.a1;
        }
        float* w0 = c.pool_att + (size_t)nd.aux * L.HWp;
        for (int p = threadIdx.x; p < HW; p += blockDim.x) w0[p] = src0[p];
        if (two) {
          float* w1 = c.pool_att + (size_t)nd.aux2 * L.HWp;
          for (int p = threadIdx.x; p < HW; p += blockDim.x) w1[p] = src1[p];
        }
      }
      continue;   // (answer roots are last; nothing of the stack is written)
    }
    switch (nd.op) {
      case OP_FIND: {        // computed by the projection kernel's epilogue; prefetched above
        const float* f = (nfilter < kTreeFindSlots) ? s.ftmp + nfilter * L.HWp
                                                    : c.arena + (size_t)nd.out * HW;
        ++nfilter;
        for (int p = threadIdx.x; p < HW; p += blockDim.x) out[p] = f[p];
        break;
      }
      case OP_SCENE: {       // models_clevr/nmn3_modules.py:60-72
        const float v = __int_as_float(nd.aux);
        for (int p = threadIdx.x; p < HW; p += blockDim.x) out[p] = v;
        break;
      }
      case OP_FILTER: {      // min(input_0, Find(t,b)) (nmn3_modules.py:129-130)
        const float* f = (nfilter < kTreeFindSlots) ? s.ftmp + nfilter * L.HWp
                                                    : c.arena + (size_t)nd.out * HW;
        ++nfilter;
        for (int p = threadIdx.x; p < HW; p += blockDim.x) out[p] = fminf(in0[p], f[p]);
        break;
      }
      case OP_AND:           // tf.minimum / tf.maximum (nmn3_modules.py:233,253)
      case OP_OR:
        for (int p = threadIdx.x; p < HW; p += blockDim.x)
          out[p] = (nd.op == OP_AND) ? fminf(in0[p], in1[p]) : fmaxf(in0[p], in1[p]);
        break;
      case OP_TRANSFORM: {
        // TransformModule, conv variant (models_clevr/nmn3_modules.py:185-216, SHAPES :71-101),
        // as the quadratic form of common.cuh; every CTA of a cluster computes the whole map
        if (KS > 1) {
          const int Hh = md.H, Ww = md.W;
          const int PW = Ww + KS - 1, PH = Hh + KS - 1, R = (KS - 1) / 2;
          for (int j = threadIdx.x; j < PH * PW; j += blockDim.x) s.pad[j] = 0.f;
          const float* qc;
          if (nquad < kTreeQuadCap) {
            qc = s_quad + nquad * qp;
          } else {   // more Transform nodes than prefetch slots: stage this one now
            float* dst = s.v0;   // 3*Mp floats >= quad_pitch for every supported shape
            for (int j = threadIdx.x; j < qp; j += blockDim.x)
              dst[j] = c.tb.tq[(size_t)nd.text * qp + j];
            qc = dst;
          }
          ++nquad;
          __syncthreads();
          for (int p = threadIdx.x; p < HW; p += blockDim.x) {
            const int y = p / Ww, x = p - y * Ww;
            s.pad[(y + R) * PW + x + R] = in0[p];
          }
          __syncthreads();
          transform_quad<KS>(s.pad, qc, md.elt_b[ES_TRANSFORM][0], out, Hh, Ww);
        }
        break;
      }
      case OP_FIND_SAME_PROPERTY: {
        // FindSamePropertyModule (models_clevr/nmn3_modules.py:134-183) / VQA TransformModule
        // (models_vqa/nmn3_modules.py:123-171): l2norm_c(m ∘ τ ∘ φ)·w2 + b2, φ = Σ_p s_p·G[p,:]
        for (int p = threadIdx.x; p < HW; p += blockDim.x) s.a0[p] = in0[p];
        __syncthreads();
        if (warp == 0) warp_softmax(s.a0, HW);
        __syncthreads();
        float* part = s.part + (exch & 1) * 2 * Mp;
        int p0, p1;
        coop_range(co, HW, p0, p1);
        gemv_partial(s.a0 + p0, p0, p1, c.mbuf + (size_t)nd.aux2 * HW * Mp, Mp, part, s.scratch);
        co.sync();
        ++exch;
        sum_partials(co, part, nullptr, s.v0, M, Mp);
        for (int ch = threadIdx.x; ch < Mp; ch += blockDim.x) {
          const float phi = s.v0[ch];
          const float tp = tau[ch] * phi;
          s.v1[ch] = tauw[ch] * phi;
          s.v2[ch] = tp * tp;
        }
        __syncthreads();
        const float b2 = md.elt_b[ES_FSP][0];
        const float* mimg = c.mbuf + (size_t)nd.aux * HW * Mp;
        float* ob = s.outbuf + (exch & 1) * L.HWp;
        // four pixels per step: their map rows are independent L2 reads, issued together (one pixel
        // at a time the warp pays an L2 round trip per pixel: ~19 of them with one CTA per question)
        constexpr int PX = 4;
        for (int pb = gwarp; pb < HW; pb += gwarps * PX) {
          float num[PX], den[PX];
#pragma unroll
          for (int u = 0; u < PX; ++u) { num[u] = 0.f; den[u] = 0.f; }
          for (int qd = lane; qd < (Mp >> 2); qd += 32) {
            float4 m[PX];
#pragma unroll
            for (int u = 0; u < PX; ++u) {
              const int p = min(pb + u * gwarps, HW - 1);
              m[u] = __ldg(reinterpret_cast<const float4*>(mimg + (size_t)p * Mp) + qd);
            }
            const float4 a = reinterpret_cast<const float4*>(s.v1)[qd];
            const float4 d = reinterpret_cast<const float4*>(s.v2)[qd];
#pragma unroll
            for (int u = 0; u < PX; ++u) {
              num[u] = fmaf(m[u].x, a.x, num[u]); num[u] = fmaf(m[u].y, a.y, num[u]);
              num[u] = fmaf(m[u].z, a.z, num[u]); num[u] = fmaf(m[u].w, a.w, num[u]);
              den[u] = fmaf(m[u].x * m[u].x, d.x, den[u]); den[u] = fmaf(m[u].y * m[u].y, d.y, den[u]);
              den[u] = fmaf(m[u].z * m[u].z, d.z, den[u]); den[u] = fmaf(m[u].w * m[u].w, d.w, den[u]);
            }
          }
#pragma unroll
          for (int u = 0; u < PX; ++u) {
            const float n = warp_sum(num[u]), dd = warp_sum(den[u]);
            const int p = pb + u * gwarps;
            if (lane == 0 && p < HW) ob[p] = n * rsqrtf(fmaxf(dd, kEps)) + b2;
          }
        }
        co.sync();
        gather_pixels(co, ob, out, HW, md.W, 1);
        ++exch;
        break;
      }
      case OP_DESCRIBE:
      case OP_SAME_PROPERTY: {
        // (kDirect = false only) DescribeModule (nmn3_modules.py:454-495) / SamePropertyModule
        // (:402-452) from the stored fc_att maps
        const bool two = (nd.op == OP_SAME_PROPERTY);
        for (int p = threadIdx.x; p < HW; p += blockDim.x) {
          s.a0[p] = in0[p];
          if (two) s.a1[p] = in1[p];
        }
        __syncthreads();
        if (warp == 0) warp_softmax(s.a0, HW);
        if (two && warp == 1) warp_softmax(s.a1, HW);
        __syncthreads();
        float* part = s.part + (exch & 1) * 2 * Mp;
        int p0, p1;
        coop_range(co, HW, p0, p1);
        const size_t map_floats = (size_t)HW * Mp;
        gemv_partial(s.a0 + p0, p0, p1, c.mbuf + nd.aux * map_floats, Mp, part, s.scratch);
        if (two)
          gemv_partial(s.a1 + p0, p0, p1, c.mbuf + nd.aux2 * map_floats, Mp, part + Mp, s.scratch);
        co.sync();
        ++exch;
        if (co.rank == 0) {   // the tail is tiny: one CTA finishes it
          sum_partials(co, part, nullptr, s.v0, M, Mp);
          if (two) sum_partials(co, part + Mp, nullptr, s.v1, M, Mp);
          if (c.phi_out != nullptr) {
            __syncthreads();
            float* ph = c.phi_out + (size_t)nd.out * 2 * Mp;
            for (int ch = threadIdx.x; ch < Mp; ch += blockDim.x) {
              ph[ch] = ch < M ? s.v0[ch] : 0.f;
              ph[Mp + ch] = (two && ch < M) ? s.v1[ch] : 0.f;
            }
          }
          float ss = 0.f;
          for (int ch = threadIdx.x; ch < M; ch += blockDim.x) {
            const float e = two ? s.v0[ch] * tau[ch] * s.v1[ch] : tau[ch] * s.v0[ch];
            s.v2[ch] = e;
            ss = fmaf(e, e, ss);
          }
          ss = block_reduce<0>(ss, s.red);
          const float inv = rsqrtf(fmaxf(ss, kEps));   // tf.nn.l2_normalize(e, 1)
          for (int ch = threadIdx.x; ch < M; ch += blockDim.x) s.v2[ch] *= inv;
          cp_async_commit_wait_all();
          __syncthreads();
          const int os = two ? OS_SAMEPROP : OS_DESCRIBE;
          small_fc(s.v2, M, head_w ? head_w : md.out_w[os], md.out_b[os], md.C,
                   score_row(c, nd.out), s.scratch);
        }
        break;
      }
      default: {
        // (kDirect = false only) Exist / Count / EqualNum / MoreNum / LessNum
        // (nmn3_modules.py:258-400): rank 0 only, everything it needs is in its local stack
        if (co.rank != 0) break;
        int Lz, set;
        if (nd.op == OP_EXIST) {
          if (warp == 0) {
            float mn, mx, sum;
            warp_minmax(in0, HW, mn, mx, sum);
            if (lane == 0) { s.z[0] = mn; s.z[1] = sum / (float)HW; s.z[2] = mx; }
          }
          Lz = 3; set = SS_EXIST;
        } else {
          const bool two = (nd.op != OP_COUNT);
          for (int p = threadIdx.x; p < HW; p += blockDim.x) {
            s.z[p] = in0[p];
            if (two) s.z[HW + 2 + p] = in1[p];
          }
          if (warp == 0) {
            float mn, mx, sum;
            warp_minmax(in0, HW, mn, mx, sum);
            if (lane == 0) { s.z[HW] = mn; s.z[HW + 1] = mx; }
          } else if (two && warp == 1) {
            float mn, mx, sum;
            warp_minmax(in1, HW, mn, mx, sum);
            if (lane == 0) { s.z[2 * HW + 2] = mn; s.z[2 * HW + 3] = mx; }
          }
          Lz = two ? 2 * (HW + 2) : HW + 2;
          set = (nd.op == OP_COUNT) ? SS_COUNT : (nd.op == OP_EQUAL_NUM) ? SS_EQUAL
              : (nd.op == OP_MORE_NUM) ? SS_MORE : SS_LESS;
        }
        cp_async_commit_wait_all();
        __syncthreads();
        small_fc(s.z, Lz, head_w ? head_w : md.sc_w[set], md.sc_b[set], md.C,
                 score_row(c, nd.out), s.scratch);
        break;
      }
    }
    __syncthreads();   // this node's stack writes are visible to the CTA's next node
    if (write_arena && co.rank == 0 && out != nullptr && nd.op != OP_FIND) {
      float* g = c.arena + (size_t)nd.out * HW;
      for (int p = threadIdx.x; p < HW; p += blockDim.x) g[p] = out[p];
    }
  }
  // peers may still be reading this CTA's outbuf / part through distributed shared memory
  if (csize > 1) cg::this_cluster().sync();
}

}  // namespace n2nmn
