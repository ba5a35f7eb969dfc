// Backward pass of the module network (SURVEY.md §8 a20, App. E): gradients of
// avg_sample_loss (exp_clevr/train_clevr_rl_gt_layout.py:108-119) w.r.t. every module variable and
// w.r.t. word_vecs, following TF 1.0's registered gradients (ties of tf.minimum/maximum go to
// input_0; reduce_min/max split ties equally; l2_normalize takes the constant branch below eps).
//
// Structure (DESIGN.md §4b has the measured history):
//   loss_kernel      : softmax cross-entropy (+ optional question-prior logits), validity select
//                      (VQA: cross-entropy on every row), d(loss)/d(scores)
//   tail_prep_kernel + head_tail_wgmma_kernel + xtb_mma_kernel<TailGradSrc> : answer heads with
//                      many classes, batched over all roots before the walk: dê = dS·W_outᵀ,
//                      d(W_out) = Êᵀ·dS, d(b_out)
//   tree_bwd_kernel  : reverse walk, ONE CTA PER NODE and one launch per depth level from the
//                      roots down; gradient maps travel through a global [nodes][HW] buffer (a map
//                      has one consumer, so one writer); recomputes each module's forward
//                      intermediates from the saved attention maps / stored tensor-core maps and
//                      emits (a) small weight gradients by atomics, (b) d(tau) per text row,
//                      (c) one [HW, Mp] "B map" per feature-side layer use (dm for conv_image,
//                      s_p*dphi for the fc_att layers). Nodes with independent per-pixel work are
//                      split over several CTAs by pixel ranges.
//   xtb_mma_kernel   : C[k,c] += Σ_p X[p,k]·B[p,c] on mma.sync TF32 fragments: the weight gradient
//                      of every "X·W + b" layer — d(W_set) = Σ_entries X_b^T · B_entry for the
//                      feature-side layers, d(fc_text W) = Σ t^T dtau for the text layers
//   text_xgrad_mma_kernel : d(word_vecs) = dtau · W^T
//   feat_grad_kernel / text_wgrad_kernel / text_xgrad_kernel : the same three products in exact
//                      fp32 on the CUDA cores (verification path, N2NMN_FLAG_PROJ_FP32_SIMT)
//   (weight decay, per-tensor clip_by_norm and Adam, train_clevr_rl_gt_layout.py:126-139, are in
//   optim.cuh, shared with the layout generator)
#pragma once
#include "node_eval.cuh"
#include "optim.cuh"

namespace n2nmn {

// Offsets (in floats) of every variable's gradient inside the flat gradient buffer, TF layout.
struct GradOffsets {
  int proj_w[NUM_PROJ_SETS], proj_b[NUM_PROJ_SETS];   // conv_image / fc_att layers
  int txt_w[NUM_TEXT_SETS], txt_b[NUM_TEXT_SETS];
  int elt_w[NUM_ELT_SETS], elt_b[NUM_ELT_SETS];
  int conv_k, conv_b;
  int out_w[NUM_OUT_SETS], out_b[NUM_OUT_SETS];
  int sc_w[NUM_SCORE_SETS], sc_b[NUM_SCORE_SETS];
};

struct BwdEntry { int32_t set, b; };   // one B map: which layer, which image

struct BwdCtx {
  DevModel md;
  TextBufs tb;
  const float* arena;     // forward attention maps, [nodes][HW] (tree kernel ran with write_arena)
  const float* scores;    // [NQ][C]
  const float* dscores;   // [NQ][C]
  const float* mbuf;      // stored maps; PS_FIND maps are stored too in training schedules
  float* gflat;           // flat gradient buffer (zero-initialised)
  float* dtau;            // [text rows][Mp]
  float* dmap;            // [entries][HW][Mp]
  float* dstencil;        // [nodes][HW][Mp] scratch: d(conv_maps output) of a Transform node
  float* gmap;            // [nodes][HWp] d loss / d(attention map of the node), zero-initialised
  const float* phi;       // [score rows][2][Mp] attended features of the Describe-type roots (forward)
  // many-class heads (C > 32): d loss / d ê of the Describe-type roots, [score rows][Mp], computed
  // for all roots at once before the walk (tail_prep_kernel + head_tail_wgmma_kernel), with the
  // fc_eltwise weight gradient (xtb_mma_kernel<TailGradSrc>); nullptr: the walk does both per root
  const float* dehat;
  GradOffsets go;
};

// ---- loss ------------------------------------------------------------------------------------
// One warp per question. loss_acc[0] += per-sample loss, dscores = (softmax - onehot) / NQ for
// valid questions, 0 otherwise (invalid rows cost the constant invalid_expr_loss).
// prior (optional, [NQ][C]): logits added to the module scores before the loss and written back
// into `scores` (the VQA question-prior net, exp_vqa/train_vqa_gt_layout.py:101-121).
// ce_all: softmax cross-entropy on every row, invalid layouts included (VQA: an invalid layout
// scores zeros, so its row is CE(prior, label)). dscores_out (optional): out_scale * dscores.
__global__ void loss_kernel(float* __restrict__ scores, const float* __restrict__ prior,
                            const int32_t* __restrict__ labels, const int32_t* __restrict__ q_ptr,
                            int NQ, int C, float invalid_loss, int ce_all,
                            float* __restrict__ dscores, float* __restrict__ dscores_out,
                            float out_scale, float* __restrict__ per_sample,
                            float* __restrict__ loss_acc) {
  const int q = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (q >= NQ) return;
  const bool valid = q_ptr[q + 1] > q_ptr[q];
  float* s = scores + (size_t)q * C;
  float* d = dscores + (size_t)q * C;
  float* dout = dscores_out ? dscores_out + (size_t)q * C : nullptr;
  if (prior != nullptr)   // each lane adds and later reads only its own columns
    for (int c = lane; c < C; c += 32) s[c] += prior[(size_t)q * C + c];
  if (!valid && !ce_all) {
    for (int c = lane; c < C; c += 32) { d[c] = 0.f; if (dout) dout[c] = 0.f; }
    if (lane == 0) { per_sample[q] = invalid_loss; atomicAdd(loss_acc, invalid_loss); }
    return;
  }
  float mx = -INFINITY;
  for (int c = lane; c < C; c += 32) mx = fmaxf(mx, s[c]);
  mx = warp_max(mx);
  float sum = 0.f;
  for (int c = lane; c < C; c += 32) sum += expf(s[c] - mx);
  sum = warp_sum(sum);
  const int y = labels[q];
  const float inv = 1.f / sum, invn = 1.f / (float)NQ;
  for (int c = lane; c < C; c += 32) {
    const float p = expf(s[c] - mx) * inv;
    d[c] = (p - (c == y ? 1.f : 0.f)) * invn;
    if (dout) dout[c] = d[c] * out_scale;
  }
  if (lane == 0) {
    const float l = logf(sum) + mx - s[y];
    per_sample[q] = l;
    atomicAdd(loss_acc, l);
  }
}

// ---- many-class answer heads: operands of the batched tail backward ----------------------------
// dÊ = dS·W_outᵀ runs on head_tail_wgmma_kernel (3xTF32, the forward's fp32-parity scheme: dÊ
// feeds the l2norm backward, whose projection term cancels), d(W_out) = Êᵀ·dS on xtb_mma_kernel.
// One CTA per question q: root_set[q] = the fc_eltwise set of its Describe-type root (-1: other
// root or invalid layout); ê[q] = l2norm(τ∘φ0 (∘φ1)) from the forward's φ, zero for the others;
// dS[q] as hi / lo planes (value, value - trunc_tf32(value)) with row pitch Cp, zero padded;
// dst[set][q] = the dê row of q for the set of its root, nullptr otherwise.
__global__ void __launch_bounds__(256)
tail_prep_kernel(const BwdCtx c, const NodeRec* __restrict__ nodes, const int32_t* __restrict__ q_ptr,
                 int Cp, int nb, int32_t* __restrict__ root_set, float* __restrict__ ehat,
                 float* __restrict__ ds_hi, float* __restrict__ ds_lo, float* __restrict__ dehat,
                 float** __restrict__ dst) {
  __shared__ float red[32];
  const int q = blockIdx.x, Mp = c.md.Mp, M = c.md.M, C = c.md.C;
  int os = -1, text = 0;
  if (q_ptr[q + 1] > q_ptr[q]) {
    const NodeRec nd = nodes[q_ptr[q + 1] - 1];
    os = nd.op == OP_DESCRIBE ? OS_DESCRIBE : nd.op == OP_SAME_PROPERTY ? OS_SAMEPROP : -1;
    text = nd.text;
  }
  if (threadIdx.x == 0) {
    root_set[q] = os;
    for (int s = 0; s < NUM_OUT_SETS; ++s) dst[s * nb + q] = (s == os) ? dehat + (size_t)q * Mp : nullptr;
  }
  for (int cc = threadIdx.x; cc < Cp; cc += blockDim.x) {
    const float v = cc < C ? c.dscores[(size_t)q * C + cc] : 0.f;
    ds_hi[(size_t)q * Cp + cc] = v;
    ds_lo[(size_t)q * Cp + cc] = v - __uint_as_float(__float_as_uint(v) & 0xffffe000u);
  }
  float* eh = ehat + (size_t)q * Mp;
  if (os < 0) {
    for (int ch = threadIdx.x; ch < Mp; ch += blockDim.x) eh[ch] = 0.f;
    return;
  }
  const float* ph = c.phi + (size_t)q * 2 * Mp;
  const float* tau = c.tb.tau + (size_t)text * Mp;
  float ss = 0.f;
  for (int ch = threadIdx.x; ch < M; ch += blockDim.x) {
    const float e = os == OS_SAMEPROP ? ph[ch] * tau[ch] * ph[Mp + ch] : tau[ch] * ph[ch];
    ss = fmaf(e, e, ss);
  }
  ss = block_reduce<0>(ss, red);
  const float inv = rsqrtf(fmaxf(ss, kEps));
  for (int ch = threadIdx.x; ch < Mp; ch += blockDim.x) {
    float e = 0.f;
    if (ch < M) e = (os == OS_SAMEPROP ? ph[ch] * tau[ch] * ph[Mp + ch] : tau[ch] * ph[ch]) * inv;
    eh[ch] = e;
  }
}

// lo[i] = w[i] - trunc_tf32(w[i]): the remainder plane of a matrix for the 3xTF32 products.
__global__ void tf32_lo_kernel(const float* __restrict__ w, float* __restrict__ lo, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float v = w[i];
    lo[i] = v - __uint_as_float(__float_as_uint(v) & 0xffffe000u);
  }
}

// ---- helpers for the reverse tree walk ---------------------------------------------------------
// Backward of the answer heads' input vector z = [a.flat, min, max] (or [min, mean, max]).
__device__ __forceinline__ void minmax_count(const float* a, int HW, float* red, float& mn,
                                             float& mx, float& cmn, float& cmx) {
  float lmn = INFINITY, lmx = -INFINITY;
  for (int p = threadIdx.x; p < HW; p += blockDim.x) { lmn = fminf(lmn, a[p]); lmx = fmaxf(lmx, a[p]); }
  mn = block_reduce<2>(lmn, red);
  mx = block_reduce<1>(lmx, red);
  float c0 = 0.f, c1 = 0.f;
  for (int p = threadIdx.x; p < HW; p += blockDim.x) { c0 += (a[p] == mn); c1 += (a[p] == mx); }
  cmn = block_reduce<0>(c0, red);
  cmx = block_reduce<0>(c1, red);
}

// dz[k] = Σ_c W[k*C+c]·g[c]  and  dW[k*C+c] += z[k]·g[c], db[c] += g[c]
__device__ __forceinline__ void head_backward(const float* z, int L, const float* __restrict__ W,
                                              const float* g, int C, float* dz, float* gW,
                                              float* gb) {
  for (int k = threadIdx.x; k < L; k += blockDim.x) {
    float acc = 0.f;
    const float zk = z[k];
    for (int c = 0; c < C; ++c) {
      acc = fmaf(W[(size_t)k * C + c], g[c], acc);
      atomicAdd(gW + (size_t)k * C + c, zk * g[c]);
    }
    dz[k] = acc;
  }
  for (int c = threadIdx.x; c < C; c += blockDim.x) atomicAdd(gb + c, g[c]);
  __syncthreads();
}

// Backward of  out = l2norm_c(e)·w2 + b2  for ONE pixel handled by one warp, e_c = base_c*coef_c.
// Given lane-strided e values it returns de (in place of e) and accumulates dw2 / db2.
//   ê = e*inv ; dê = g*w2 ; de = (dê - ê(ê·dê))*inv   (no projection term when ss <= eps)

// Shared-memory layout of tree_bwd_kernel (floats).
struct BwdSmem {
  int HWp, g, pad, k, vec, z, total;
};
__host__ __device__ inline BwdSmem bwd_smem_layout(int H, int W, int Mp, int ksize, int C) {
  BwdSmem s;
  const int HW = H * W;
  s.HWp = (HW + 3) & ~3;
  s.g = 0;
  s.pad = ((H + ksize - 1) * (W + ksize - 1) + 3) & ~3;
  s.k = 2 * ksize * ksize * Mp;          // filter bank + its gradient
  s.vec = 10 * Mp;
  s.z = 2 * ((2 * (HW + 2) + 3) & ~3) + ((C + 3) & ~3);
  s.total = s.g + 4 * s.HWp + 2 * s.pad + s.k + s.vec + s.z + 64;
  return s;
}

constexpr int kBwdSlicesMax = 8;   // CTAs per splittable node (>= 19 of the 150 CLEVR pixels each)

// One CTA per NODE, one launch per depth level from the roots down (bwd_nodes lists the nodes by
// depth): the gradient maps travel between the levels through c.gmap (a node's map feeds exactly
// one parent, so its gradient row has one writer, and that writer ran in an earlier launch).
// Round 1 walked a question's nodes inside one CTA: 64 CTAs on all the SMs and the longest question
// (~10 dependent modules, each bound by its own reductions) set the time: 360 us.
// Two instantiations: kTransform = true handles every op (the stencil backward of Transform keeps
// ~170 registers busy: one CTA per SM) and runs the levels that contain Transform nodes; false
// leaves the Transform body out (128 registers, two CTAs per SM) and runs the other levels.
// kWide: Mp > 512 (the VQA family, KS = 1, no conv Transform): the Find-type case takes two passes
// over the channels.
template <int KS, bool kTransform, bool kWide = false>
__global__ void __launch_bounds__(kNodeThreads, kTransform ? 1 : 2)
tree_bwd_kernel(const BwdCtx c, const NodeRec* __restrict__ nodes,
                const int32_t* __restrict__ bwd_nodes, int first,
                const int32_t* __restrict__ node_entry) {
  pdl_trigger();
  extern __shared__ __align__(16) float bsm[];
  const DevModel& md = c.md;
  const int HW = md.HW, Mp = md.Mp, M = md.M, C = md.C, Hh = md.H, Ww = md.W;
  const BwdSmem L = bwd_smem_layout(Hh, Ww, Mp, md.ksize, C);
  float* a0 = bsm;                        // forward inputs / scratch maps
  float* a1 = a0 + L.HWp;
  float* da = a1 + L.HWp;
  float* db_ = da + L.HWp;
  float* pad = db_ + L.HWp;               // zero-padded forward input of Transform
  float* dpad = pad + L.pad;              // gradient w.r.t. the padded input
  float* ks = dpad + L.pad;               // conv filter bank [KS*KS][Mp]
  float* dks = ks + KS * KS * Mp;         // its gradient
  float* v = dks + KS * KS * Mp;          // 10 vectors of Mp
  float* zb = v + 10 * Mp;                // z, dz, g(C)
  float* red = zb + L.z;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int zlen = (2 * (HW + 2) + 3) & ~3;
  float* z = zb;
  float* dz = zb + zlen;
  float* gsc = dz + zlen;
  {
    const int i = bwd_nodes[first + blockIdx.x];
    const NodeRec nd = nodes[i];
    // gridDim.y CTAs share the pixels of a node whose per-pixel work is independent (Find, Filter,
    // Transform: what they accumulate over pixels goes out through atomics; Describe and
    // SameProperty: slice 0 emits the per-node results); the others run in slice 0 alone
    const bool split = (nd.op == OP_FIND || nd.op == OP_FILTER || nd.op == OP_TRANSFORM ||
                        nd.op == OP_DESCRIBE || nd.op == OP_SAME_PROPERTY);
    const int slice = blockIdx.y, ns = split ? (int)gridDim.y : 1;
    if (slice >= ns) return;
    // The levels are chained with programmatic dependent launch: what does not depend on the level
    // above (the node record, the Transform filter bank — 25 KB per CTA, the top stall of the
    // Transform levels when it was staged after the wait) is fetched before griddepcontrol.wait.
    if constexpr (kTransform) {
      if (nd.op == OP_TRANSFORM)
        for (int j = threadIdx.x; j < KS * KS * Mp; j += blockDim.x) ks[j] = md.conv_k[j];
    }
    pdl_wait();
    const int p_lo = (HW * slice) / ns, p_hi = (HW * (slice + 1)) / ns;
    float* g = c.gmap + (size_t)i * L.HWp;                    // d loss / d this node's map
    float* gin0 = (nd.in0 >= 0) ? c.gmap + (size_t)nd.in0 * L.HWp : nullptr;
    float* gin1 = (nd.in1 >= 0) ? c.gmap + (size_t)nd.in1 * L.HWp : nullptr;
    const float* fin0 = (nd.in0 >= 0) ? c.arena + (size_t)nd.in0 * HW : nullptr;
    const float* fin1 = (nd.in1 >= 0) ? c.arena + (size_t)nd.in1 * HW : nullptr;
    const float* fout = c.arena + (size_t)i * HW;             // this node's forward map
    switch (nd.op) {
      case OP_SCENE: break;
      case OP_AND: case OP_OR:   // ties -> input_0 (App. E)
        for (int p = threadIdx.x; p < HW; p += blockDim.x) {
          const bool to0 = (nd.op == OP_AND) ? (fin0[p] <= fin1[p]) : (fin0[p] >= fin1[p]);
          if (to0) gin0[p] += g[p]; else gin1[p] += g[p];
        }
        break;
      case OP_EXIST: case OP_COUNT: case OP_EQUAL_NUM: case OP_MORE_NUM: case OP_LESS_NUM: {
        for (int cc = threadIdx.x; cc < C; cc += blockDim.x) gsc[cc] = c.dscores[(size_t)nd.out * C + cc];
        const bool two = (nd.op == OP_EQUAL_NUM || nd.op == OP_MORE_NUM || nd.op == OP_LESS_NUM);
        const int set = (nd.op == OP_EXIST) ? SS_EXIST : (nd.op == OP_COUNT) ? SS_COUNT
                      : (nd.op == OP_EQUAL_NUM) ? SS_EQUAL : (nd.op == OP_MORE_NUM) ? SS_MORE : SS_LESS;
        float mn0, mx0, cmn0, cmx0, mn1 = 0, mx1 = 0, cmn1 = 1, cmx1 = 1, sum0 = 0.f;
        for (int p = threadIdx.x; p < HW; p += blockDim.x) { a0[p] = fin0[p]; if (two) a1[p] = fin1[p]; }
        __syncthreads();
        minmax_count(a0, HW, red, mn0, mx0, cmn0, cmx0);
        if (two) minmax_count(a1, HW, red, mn1, mx1, cmn1, cmx1);
        int Lz;
        if (nd.op == OP_EXIST) {
          float ls = 0.f;
          for (int p = threadIdx.x; p < HW; p += blockDim.x) ls += a0[p];
          sum0 = block_reduce<0>(ls, red);
          if (threadIdx.x == 0) { z[0] = mn0; z[1] = sum0 / (float)HW; z[2] = mx0; }
          Lz = 3;
        } else {
          for (int p = threadIdx.x; p < HW; p += blockDim.x) { z[p] = a0[p]; if (two) z[HW + 2 + p] = a1[p]; }
          if (threadIdx.x == 0) {
            z[HW] = mn0; z[HW + 1] = mx0;
            if (two) { z[2 * HW + 2] = mn1; z[2 * HW + 3] = mx1; }
          }
          Lz = two ? 2 * (HW + 2) : HW + 2;
        }
        __syncthreads();
        head_backward(z, Lz, md.sc_w[set], gsc, C, dz, c.gflat + c.go.sc_w[set],
                      c.gflat + c.go.sc_b[set]);
        for (int p = threadIdx.x; p < HW; p += blockDim.x) {
          if (nd.op == OP_EXIST) {
            gin0[p] += dz[0] * (a0[p] == mn0) / cmn0 + dz[1] / (float)HW + dz[2] * (a0[p] == mx0) / cmx0;
          } else {
            gin0[p] += dz[p] + dz[HW] * (a0[p] == mn0) / cmn0 + dz[HW + 1] * (a0[p] == mx0) / cmx0;
            if (two)
              gin1[p] += dz[HW + 2 + p] + dz[2 * HW + 2] * (a1[p] == mn1) / cmn1 +
                         dz[2 * HW + 3] * (a1[p] == mx1) / cmx1;
          }
        }
        break;
      }
      case OP_DESCRIBE: case OP_SAME_PROPERTY: {
        // forward: s = softmax(a); phi = Σ_p s_p G[p]; e = tau∘phi (∘phi1); ê = e/n; scores = ê·Wout+b
        // phi comes from the forward pass (c.phi); every slice redoes the channel-vector part
        // (a few thousand FMAs) and takes its share of the pixels for the B maps and the softmax
        // backward, whose Σ_p s_p ds_p term is dphi·phi in closed form.
        const bool two = (nd.op == OP_SAME_PROPERTY);
        const int os = two ? OS_SAMEPROP : OS_DESCRIBE;
        float* phi0 = v; float* phi1 = v + Mp; float* e = v + 2 * Mp; float* de = v + 3 * Mp;
        float* dphi0 = v + 4 * Mp; float* dphi1 = v + 5 * Mp;
        if (c.dehat == nullptr)
          for (int cc = threadIdx.x; cc < C; cc += blockDim.x) gsc[cc] = c.dscores[(size_t)nd.out * C + cc];
        for (int p = threadIdx.x; p < HW; p += blockDim.x) { a0[p] = fin0[p]; if (two) a1[p] = fin1[p]; }
        __syncthreads();
        softmax_inplace(a0, HW, red);
        if (two) softmax_inplace(a1, HW, red);
        const float* G0 = c.mbuf + (size_t)nd.aux * HW * Mp;
        const float* G1 = two ? c.mbuf + (size_t)nd.aux2 * HW * Mp : nullptr;
        const float* tau = c.tb.tau + (size_t)nd.text * Mp;
        const float* ph = c.phi + (size_t)nd.out * 2 * Mp;
        for (int ch = threadIdx.x; ch < Mp; ch += blockDim.x) {
          const float p0 = ch < M ? ph[ch] : 0.f, p1 = (two && ch < M) ? ph[Mp + ch] : 0.f;
          phi0[ch] = p0; phi1[ch] = p1;
          e[ch] = (ch < M) ? (two ? p0 * tau[ch] * p1 : tau[ch] * p0) : 0.f;
        }
        __syncthreads();
        float ss = 0.f;
        for (int ch = threadIdx.x; ch < M; ch += blockDim.x) ss = fmaf(e[ch], e[ch], ss);
        ss = block_reduce<0>(ss, red);
        const float inv = rsqrtf(fmaxf(ss, kEps));
        // dê = Wout·g ; head weight grads with ê (slice 0)
        float dot = 0.f;
        if (c.dehat != nullptr) {   // dê and the head weight grads were computed before the walk
          const float* dr = c.dehat + (size_t)nd.out * Mp;
          for (int ch = threadIdx.x; ch < M; ch += blockDim.x) {
            const float acc = dr[ch];
            de[ch] = acc;
            dot = fmaf(e[ch] * inv, acc, dot);
          }
        } else {
          for (int ch = threadIdx.x; ch < M; ch += blockDim.x) {
            const float eh = e[ch] * inv;
            float acc = 0.f;
            for (int cc = 0; cc < C; ++cc) {
              acc = fmaf(md.out_w[os][(size_t)ch * C + cc], gsc[cc], acc);
              if (slice == 0) atomicAdd(c.gflat + c.go.out_w[os] + (size_t)ch * C + cc, eh * gsc[cc]);
            }
            de[ch] = acc;            // holds dê for now
            dot = fmaf(eh, acc, dot);
          }
          if (slice == 0)
            for (int cc = threadIdx.x; cc < C; cc += blockDim.x) atomicAdd(c.gflat + c.go.out_b[os] + cc, gsc[cc]);
        }
        dot = block_reduce<0>(dot, red);
        if (!(ss > kEps)) dot = 0.f;
        float* dtau = c.dtau + (size_t)nd.text * Mp;
        float sd0 = 0.f, sd1 = 0.f;   // Σ_ch dphi·phi = Σ_p s_p ds_p
        for (int ch = threadIdx.x; ch < Mp; ch += blockDim.x) {
          float d = 0.f, dt = 0.f, d0 = 0.f, d1 = 0.f;
          if (ch < M) {
            d = (de[ch] - e[ch] * inv * dot) * inv;            // de
            if (two) { dt = d * phi0[ch] * phi1[ch]; d0 = d * tau[ch] * phi1[ch]; d1 = d * tau[ch] * phi0[ch]; }
            else { dt = d * phi0[ch]; d0 = d * tau[ch]; }
          }
          if (slice == 0) dtau[ch] = dt;
          dphi0[ch] = d0; dphi1[ch] = d1;
          sd0 = fmaf(d0, phi0[ch], sd0); sd1 = fmaf(d1, phi1[ch], sd1);
        }
        sd0 = block_reduce<0>(sd0, red);
        sd1 = block_reduce<0>(sd1, red);
        __syncthreads();
        // B maps: dG[p,:] = s_p * dphi ; input gradients through the softmax
        const int ent = node_entry[i];
        for (int which = 0; which < (two ? 2 : 1); ++which) {
          const float* G = which ? G1 : G0;
          const float* sft = which ? a1 : a0;
          const float* dphi = which ? dphi1 : dphi0;
          const float sd = which ? sd1 : sd0;
          float* B = c.dmap + (size_t)(ent + which) * HW * Mp;
          float* gi = which ? gin1 : gin0;
          for (int p = p_lo + warp; p < p_hi; p += nwarps) {
            float acc = 0.f;
            const float sp = sft[p];
            for (int ch = lane; ch < Mp; ch += 32) {
              const float dp = dphi[ch];
              acc = fmaf(G[(size_t)p * Mp + ch], dp, acc);
              B[(size_t)p * Mp + ch] = sp * dp;
            }
            acc = warp_sum(acc);
            if (lane == 0) gi[p] += sp * (acc - sd);
          }
        }
        break;
      }
      case OP_FIND: case OP_FILTER: case OP_FIND_SAME_PROPERTY: {
        // out = l2norm_c(m∘coef)·w2 + b2 with coef = tau (Find/Filter) or tau∘phi (FSP)
        const bool fsp = (nd.op == OP_FIND_SAME_PROPERTY);
        const int es = fsp ? ES_FSP : ES_FIND;
        float* coef = v; float* phi = v + Mp; float* dcoef = v + 2 * Mp; float* dw2 = v + 3 * Mp;
        float* gm = a1;   // gradient that reaches the l2norm/conv_eltwise output
        const float* tau = c.tb.tau + (size_t)nd.text * Mp;
        const float* w2 = md.elt_w[es];
        const float* mimg;
        if (nd.op == OP_FILTER) {
          // out = min(a, find): gradient to `a` where out == a (ties included), else to find
          for (int p = threadIdx.x; p < HW; p += blockDim.x) {
            const bool to_a = (fout[p] == fin0[p]);
            if (to_a) { if (slice == 0) gin0[p] += g[p]; gm[p] = 0.f; } else { gm[p] = g[p]; }
          }
        } else {
          for (int p = threadIdx.x; p < HW; p += blockDim.x) gm[p] = g[p];
        }
        if (fsp) {
          for (int p = threadIdx.x; p < HW; p += blockDim.x) a0[p] = fin0[p];
          __syncthreads();
          softmax_inplace(a0, HW, red);
          const float* G = c.mbuf + (size_t)nd.aux2 * HW * Mp;
          for (int ch = threadIdx.x; ch < Mp; ch += blockDim.x) {
            float p0 = 0.f;
            if (ch < M) {
#pragma unroll 8
              for (int p = 0; p < HW; ++p) p0 = fmaf(a0[p], G[(size_t)p * Mp + ch], p0);
            }
            phi[ch] = p0;
            coef[ch] = (ch < M) ? tau[ch] * p0 : 0.f;
          }
          mimg = c.mbuf + (size_t)nd.aux * HW * Mp;
        } else {
          for (int ch = threadIdx.x; ch < Mp; ch += blockDim.x) coef[ch] = (ch < M) ? tau[ch] : 0.f;
          mimg = c.mbuf + (size_t)nd.aux * HW * Mp;   // training schedules store the Find maps too
        }
        float* w2s = v + 5 * Mp;   // conv_eltwise weights of this layer, zero beyond M
        for (int ch = threadIdx.x; ch < Mp; ch += blockDim.x) {
          dcoef[ch] = 0.f; dw2[ch] = 0.f;
          w2s[ch] = (ch < M) ? w2[ch] : 0.f;
        }
        __syncthreads();
        const int ent = node_entry[i];
        float* B = c.dmap + (size_t)ent * HW * Mp;       // dm rows
        float db2 = 0.f;
        // lane owns channels lane + 32k: the map row is read once into registers, and the
        // per-channel sums over this warp's pixels stay in registers until the end (they used to
        // be one shared-memory atomic per (pixel, channel) with all 8 warps on the same addresses)
        constexpr int kCh = 16;                 // registers per lane: Mp <= 512 in one pass
        const int nk = Mp >> 5;
        if constexpr (kWide) {
          // Mp > 512 (VQA: 1024): a lane's channels do not fit in registers at once. Pass 1 keeps
          // each pixel's l2norm statistics (1/|e|, ê·w2) in shared memory (da, db_); pass 2 walks
          // the channels 16 per lane at a time and re-reads the map rows for every group.
          for (int p = p_lo + warp; p < p_hi; p += nwarps) {
            const float* mrow = mimg + (size_t)p * Mp;
            float ss = 0.f, num = 0.f;
            for (int k0 = 0; k0 < nk; k0 += kCh) {
              float mv[kCh];
#pragma unroll
              for (int k = 0; k < kCh; ++k) mv[k] = (k0 + k < nk) ? __ldg(mrow + (k0 + k) * 32 + lane) : 0.f;
#pragma unroll
              for (int k = 0; k < kCh; ++k) {
                if (k0 + k < nk) {
                  const int ch = (k0 + k) * 32 + lane;
                  const float ev = mv[k] * coef[ch];
                  ss = fmaf(ev, ev, ss);
                  num = fmaf(ev, w2s[ch], num);
                }
              }
            }
            ss = warp_sum(ss); num = warp_sum(num);
            if (lane == 0) {
              const float inv = rsqrtf(fmaxf(ss, kEps));
              da[p] = inv;
              db_[p] = (ss > kEps) ? num * inv : 0.f;
              db2 += gm[p];
            }
          }
          __syncwarp();   // pass 2 visits the same pixels with the same warp
          for (int k0 = 0; k0 < nk; k0 += kCh) {
            float dcoef_r[kCh], dw2_r[kCh];
#pragma unroll
            for (int k = 0; k < kCh; ++k) { dcoef_r[k] = 0.f; dw2_r[k] = 0.f; }
            for (int p = p_lo + warp; p < p_hi; p += nwarps) {
              const float gp = gm[p], inv = da[p], proj = db_[p];
              const float* mrow = mimg + (size_t)p * Mp;
              float mv[kCh];
#pragma unroll
              for (int k = 0; k < kCh; ++k) mv[k] = (k0 + k < nk) ? __ldg(mrow + (k0 + k) * 32 + lane) : 0.f;
#pragma unroll
              for (int k = 0; k < kCh; ++k) {
                if (k0 + k < nk) {
                  const int ch = (k0 + k) * 32 + lane;
                  float dm = 0.f;
                  if (ch < M) {
                    const float eh = mv[k] * coef[ch] * inv;
                    const float dev = gp * (w2s[ch] - eh * proj) * inv;
                    dm = dev * coef[ch];
                    dcoef_r[k] = fmaf(dev, mv[k], dcoef_r[k]);
                    dw2_r[k] = fmaf(gp, eh, dw2_r[k]);
                  }
                  B[(size_t)p * Mp + ch] = dm;
                }
              }
            }
#pragma unroll
            for (int k = 0; k < kCh; ++k) {
              if (k0 + k < nk) {
                atomicAdd(&dcoef[(k0 + k) * 32 + lane], dcoef_r[k]);
                atomicAdd(&dw2[(k0 + k) * 32 + lane], dw2_r[k]);
              }
            }
          }
        } else {   // Mp <= 512: one pass, the lane's channels stay in registers
        float dcoef_r[kCh], dw2_r[kCh];
#pragma unroll
        for (int k = 0; k < kCh; ++k) { dcoef_r[k] = 0.f; dw2_r[k] = 0.f; }
        for (int p = p_lo + warp; p < p_hi; p += nwarps) {
          const float gp = gm[p];
          const float* mrow = mimg + (size_t)p * Mp;
          float mv[kCh];
          // all loads of the row first (columns beyond M are exact zeros in the stored map), then
          // the math: interleaved, every chunk waited for its own L2 round trip
#pragma unroll
          for (int k = 0; k < kCh; ++k) mv[k] = (k < nk) ? __ldg(mrow + k * 32 + lane) : 0.f;
          float ss = 0.f, num = 0.f;
#pragma unroll
          for (int k = 0; k < kCh; ++k) {
            if (k < nk) {
              const int ch = k * 32 + lane;
              const float ev = mv[k] * coef[ch];
              ss = fmaf(ev, ev, ss);
              num = fmaf(ev, w2s[ch], num);
            }
          }
          ss = warp_sum(ss); num = warp_sum(num);
          const float inv = rsqrtf(fmaxf(ss, kEps));
          const float proj = (ss > kEps) ? num * inv : 0.f;   // ê·w2
#pragma unroll
          for (int k = 0; k < kCh; ++k) {
            if (k < nk) {
              const int ch = k * 32 + lane;
              float dm = 0.f;
              if (ch < M) {
                const float eh = mv[k] * coef[ch] * inv;
                const float dev = gp * (w2s[ch] - eh * proj) * inv;
                dm = dev * coef[ch];
                dcoef_r[k] = fmaf(dev, mv[k], dcoef_r[k]);
                dw2_r[k] = fmaf(gp, eh, dw2_r[k]);
              }
              B[(size_t)p * Mp + ch] = dm;
            }
          }
          if (lane == 0) db2 += gp;
        }
#pragma unroll
        for (int k = 0; k < kCh; ++k) {
          if (k < nk) {
            atomicAdd(&dcoef[k * 32 + lane], dcoef_r[k]);
            atomicAdd(&dw2[k * 32 + lane], dw2_r[k]);
          }
        }
        }   // kWide
        if (lane == 0) atomicAdd(c.gflat + c.go.elt_b[es], db2);
        __syncthreads();
        float* dtau = c.dtau + (size_t)nd.text * Mp;
        for (int ch = threadIdx.x; ch < Mp; ch += blockDim.x) {
          if (ch < M) atomicAdd(c.gflat + c.go.elt_w[es] + ch, dw2[ch]);
          if (ns > 1) { if (ch < M) atomicAdd(dtau + ch, dcoef[ch]); }   // dtau is zero-initialised
          else dtau[ch] = (ch < M) ? (fsp ? dcoef[ch] * phi[ch] : dcoef[ch]) : 0.f;
        }
        if (fsp) {
          // dphi = dcoef∘tau -> second B map (s_p*dphi) and the softmax backward into input_0
          float* dphi = v + 4 * Mp;
          for (int ch = threadIdx.x; ch < Mp; ch += blockDim.x) dphi[ch] = (ch < M) ? dcoef[ch] * tau[ch] : 0.f;
          __syncthreads();
          const float* G = c.mbuf + (size_t)nd.aux2 * HW * Mp;
          float* B2 = c.dmap + (size_t)(ent + 1) * HW * Mp;
          for (int p = warp; p < HW; p += nwarps) {
            float acc = 0.f;
            const float sp = a0[p];
            for (int ch = lane; ch < Mp; ch += 32) {
              acc = fmaf(G[(size_t)p * Mp + ch], dphi[ch], acc);
              B2[(size_t)p * Mp + ch] = sp * dphi[ch];
            }
            acc = warp_sum(acc);
            if (lane == 0) da[p] = acc;
          }
          __syncthreads();
          float sd = 0.f;
          for (int p = threadIdx.x; p < HW; p += blockDim.x) sd = fmaf(a0[p], da[p], sd);
          sd = block_reduce<0>(sd, red);
          for (int p = threadIdx.x; p < HW; p += blockDim.x) gin0[p] += a0[p] * (da[p] - sd);
        }
        break;
      }
      case OP_TRANSFORM: if constexpr (kTransform) {
        // A = conv(a)+bK ; e = A∘tau ; out = l2norm(e)·w2 + b2
        const int PW = Ww + KS - 1, PH = Hh + KS - 1, R = (KS - 1) / 2;
        float* tauv = v; float* w2v = v + Mp; float* bkv = v + 2 * Mp; float* dtauv = v + 3 * Mp;
        float* dw2v = v + 4 * Mp; float* dbkv = v + 5 * Mp;
        const float* tau = c.tb.tau + (size_t)nd.text * Mp;
        for (int j = threadIdx.x; j < PH * PW; j += blockDim.x) { pad[j] = 0.f; dpad[j] = 0.f; }
        // (ks, the filter bank, was staged before the dependency wait)
        for (int ch = threadIdx.x; ch < Mp; ch += blockDim.x) {
          const bool live = ch < M;
          tauv[ch] = live ? tau[ch] : 0.f;
          w2v[ch] = live ? md.elt_w[ES_TRANSFORM][ch] : 0.f;
          bkv[ch] = live ? md.conv_b[ch] : 0.f;
          dtauv[ch] = 0.f; dw2v[ch] = 0.f; dbkv[ch] = 0.f;
        }
        __syncthreads();
        for (int p = threadIdx.x; p < HW; p += blockDim.x) {
          const int y = p / Ww, x = p - y * Ww;
          pad[(y + R) * PW + x + R] = fin0[p];
        }
        __syncthreads();
        float db2 = 0.f;
        constexpr int kMaxCh = 16;   // conv Transform exists for Mp <= 512 (CLEVR 256, SHAPES 512)
        const int nj = Mp >> 5;
        float* dA_all = c.dstencil + (size_t)(first + blockIdx.x) * HW * Mp;
        float dtau_r[kMaxCh], dw2_r[kMaxCh], dbk_r[kMaxCh];
#pragma unroll
        for (int j = 0; j < kMaxCh; ++j) { dtau_r[j] = 0.f; dw2_r[j] = 0.f; dbk_r[j] = 0.f; }
        for (int p = p_lo + warp; p < p_hi; p += nwarps) {
          const int y = p / Ww, x = p - y * Ww;
          const float gp = g[p];
          float A[kMaxCh];
          float ss = 0.f, num = 0.f;
#pragma unroll
          for (int j = 0; j < kMaxCh; ++j) {
            A[j] = 0.f;
            if (j < nj) {
              const int ch = j * 32 + lane;
              float acc = bkv[ch];
              for (int dy = 0; dy < KS; ++dy)
                for (int dx = 0; dx < KS; ++dx)
                  acc = fmaf(pad[(y + dy) * PW + x + dx], ks[(dy * KS + dx) * Mp + ch], acc);
              A[j] = acc;
              const float ev = acc * tauv[ch];
              ss = fmaf(ev, ev, ss);
              num = fmaf(ev, w2v[ch], num);
            }
          }
          ss = warp_sum(ss); num = warp_sum(num);
          const float inv = rsqrtf(fmaxf(ss, kEps));
          const float proj = (ss > kEps) ? num * inv : 0.f;
#pragma unroll
          for (int j = 0; j < kMaxCh; ++j) {
            if (j < nj) {
              const int ch = j * 32 + lane;
              const float eh = A[j] * tauv[ch] * inv;
              const float dev = gp * (w2v[ch] - eh * proj) * inv;
              const float dA = dev * tauv[ch];
              dtau_r[j] = fmaf(dev, A[j], dtau_r[j]);
              dw2_r[j] = fmaf(gp, eh, dw2_r[j]);
              dbk_r[j] += dA;
              A[j] = dA;   // keep dA for the input gradient below
              dA_all[(size_t)p * Mp + ch] = dA;   // and for the filter gradient (second pass)
            }
          }
          // d(input)[p + tap] += Σ_ch K[tap, ch]·dA[ch]: per-lane partial sums of all KS² taps, then
          // ONE butterfly that leaves the total of tap L on lane L (31 shuffles with full ILP; a
          // warp_sum per tap was 5 dependent shuffle+add pairs x KS² and dominated the kernel)
          float cv[32];
#pragma unroll
          for (int t = 0; t < 32; ++t) {
            cv[t] = 0.f;
            if (t < KS * KS) {
#pragma unroll
              for (int j = 0; j < kMaxCh; ++j)
                if (j < nj) cv[t] = fmaf(ks[t * Mp + j * 32 + lane], A[j], cv[t]);
            }
          }
#pragma unroll
          for (int off = 16; off >= 1; off >>= 1) {
            const bool up = (lane & off) != 0;
#pragma unroll
            for (int i2 = 0; i2 < off; ++i2) {
              const float send = up ? cv[i2] : cv[i2 + off];
              const float recv = __shfl_xor_sync(0xffffffffu, send, off);
              cv[i2] = (up ? cv[i2 + off] : cv[i2]) + recv;
            }
          }
          if (lane < KS * KS)
            atomicAdd(&dpad[(y + lane / KS) * PW + x + lane % KS], cv[0]);
          if (lane == 0) db2 += gp;
        }
#pragma unroll
        for (int j = 0; j < kMaxCh; ++j) {
          if (j < nj) {
            atomicAdd(&dtauv[j * 32 + lane], dtau_r[j]);
            atomicAdd(&dw2v[j * 32 + lane], dw2_r[j]);
            atomicAdd(&dbkv[j * 32 + lane], dbk_r[j]);
          }
        }
        __syncthreads();   // dA_all (global, written by this CTA) is complete
        // d(conv_maps weights)[tap, ch] = Σ_p window(p)[tap]·dA[p, ch]: one thread per channel with
        // the KS² taps in registers (this was one shared-memory atomic per (pixel, tap, channel))
        for (int ch = threadIdx.x; ch < Mp; ch += blockDim.x) {
          float acc[KS * KS];
#pragma unroll
          for (int t = 0; t < KS * KS; ++t) acc[t] = 0.f;
          int y = p_lo / Ww, x = p_lo - y * Ww;
#pragma unroll 2
          for (int p = p_lo; p < p_hi; ++p, ++x) {
            if (x == Ww) { x = 0; ++y; }
            const float d = dA_all[(size_t)p * Mp + ch];
#pragma unroll
            for (int dy = 0; dy < KS; ++dy)
#pragma unroll
              for (int dx = 0; dx < KS; ++dx)
                acc[dy * KS + dx] = fmaf(pad[(y + dy) * PW + x + dx], d, acc[dy * KS + dx]);
          }
#pragma unroll
          for (int t = 0; t < KS * KS; ++t) dks[t * Mp + ch] = acc[t];
        }
        if (lane == 0) atomicAdd(c.gflat + c.go.elt_b[ES_TRANSFORM], db2);
        __syncthreads();
        float* dtau = c.dtau + (size_t)nd.text * Mp;
        for (int ch = threadIdx.x; ch < Mp; ch += blockDim.x) {
          if (ns > 1) { if (ch < M) atomicAdd(dtau + ch, dtauv[ch]); } else dtau[ch] = dtauv[ch];
          if (ch < M) {
            atomicAdd(c.gflat + c.go.elt_w[ES_TRANSFORM] + ch, dw2v[ch]);
            atomicAdd(c.gflat + c.go.conv_b + ch, dbkv[ch]);
          }
        }
        for (int j = threadIdx.x; j < KS * KS * M; j += blockDim.x) {
          const int tap = j / M, ch = j - tap * M;
          atomicAdd(c.gflat + c.go.conv_k + j, dks[tap * Mp + ch]);
        }
        for (int p = threadIdx.x; p < HW; p += blockDim.x) {
          const int y = p / Ww, x = p - y * Ww;
          const float dv = dpad[(y + R) * PW + x + R];
          if (ns > 1) { if (dv != 0.f) atomicAdd(gin0 + p, dv); } else gin0[p] += dv;
        }
        break;
      } else break;
      default: break;
    }
    __syncthreads();
  }
}

// ---- text layers ---------------------------------------------------------------------------------
// grid = (ceil(Dt/8), NUM_TEXT_SETS): d(fc_text W)[k, :] for 8 rows k of one set, summed over the
// set's text rows; block (0, set) also reduces the bias gradient.
__global__ void __launch_bounds__(256)
text_wgrad_kernel(DevModel md, const float* __restrict__ dtau, const int32_t* __restrict__ text_t,
                  const int32_t* __restrict__ text_b, const int32_t* __restrict__ set_start,
                  float* __restrict__ gflat, GradOffsets go) {
  const int set = blockIdx.y, k0 = blockIdx.x * 8;
  const int r0 = set_start[set], r1 = set_start[set + 1];
  if (r0 == r1) return;
  const int Dt = md.Dt, M = md.M, Mp = md.Mp;
  for (int cbase = 0; cbase < M; cbase += blockDim.x) {
    const int ch = cbase + threadIdx.x;
    float acc[8], bsum = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    if (ch < M) {
      for (int r = r0; r < r1; ++r) {
        const float d = dtau[(size_t)r * Mp + ch];
        const float* t = md.word_vecs + ((size_t)text_t[r] * md.N + text_b[r]) * Dt;
#pragma unroll
        for (int j = 0; j < 8; ++j) if (k0 + j < Dt) acc[j] = fmaf(t[k0 + j], d, acc[j]);
        bsum += d;
      }
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (k0 + j < Dt) gflat[go.txt_w[set] + (size_t)(k0 + j) * M + ch] = acc[j];
      if (blockIdx.x == 0) gflat[go.txt_b[set] + ch] = bsum;
    }
  }
}

// d(word_vecs)[t, b, k] = Σ_c W[k, c]·dtau[row, c]; one CTA per text row (each (t,b) belongs to
// exactly one node, so plain stores; rows never touched stay zero from the memset).
__global__ void __launch_bounds__(256)
text_xgrad_kernel(DevModel md, const float* __restrict__ dtau, const int32_t* __restrict__ text_t,
                  const int32_t* __restrict__ text_b, const int32_t* __restrict__ set_start,
                  float* __restrict__ dword, float scale) {
  extern __shared__ float sdt[];
  const int r = blockIdx.x;
  int set = 0;
  while (set + 1 < NUM_TEXT_SETS && r >= set_start[set + 1]) ++set;
  const int Dt = md.Dt, M = md.M, Mp = md.Mp;
  for (int ch = threadIdx.x; ch < Mp; ch += blockDim.x) sdt[ch] = dtau[(size_t)r * Mp + ch];
  __syncthreads();
  float* dst = dword + ((size_t)text_t[r] * md.N + text_b[r]) * Dt;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  for (int k = warp; k < Dt; k += nwarps) {
    const float* w = md.txt_w[set] + (size_t)k * Mp;
    float acc = 0.f;
    for (int ch = lane; ch < M; ch += 32) acc = fmaf(w[ch], sdt[ch], acc);
    acc = warp_sum(acc);
    if (lane == 0) dst[k] = acc * scale;
  }
}

// ---- feature-side weight gradients: dW_set[k, c] += Σ_entries Σ_p X_b[p, k]·B_entry[p, c] --------
// grid = (Dk tiles of 64, M tiles of 64, entry chunks); 256 threads, 4x4 outputs each; the entry
// chunks are combined with atomics into the zero-initialised gradient buffer.
constexpr int kFgTile = 64, kFgRows = 32;
__global__ void __launch_bounds__(256)
feat_grad_kernel(DevModel md, const float* __restrict__ dmap, const BwdEntry* __restrict__ entries,
                 int num_entries, int entries_per_cta, float* __restrict__ gflat, GradOffsets go) {
  __shared__ __align__(16) float xs[kFgRows][kFgTile];
  __shared__ __align__(16) float bs[kFgRows][kFgTile];
  const int k0 = blockIdx.x * kFgTile, c0 = blockIdx.y * kFgTile;
  const int e0 = blockIdx.z * entries_per_cta, e1 = min(num_entries, e0 + entries_per_cta);
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;   // 16 x 16 threads, 4x4 outputs each
  const int HW = md.HW, Mp = md.Mp, M = md.M, Dk = md.Dk;
  int cur_set = -1;
  float acc[4][4], bsum[4];
  auto flush = [&](int set) {
    if (set < 0) return;
    for (int i = 0; i < 4; ++i)
      for (int j = 0; j < 4; ++j) {
        const int k = k0 + ty * 4 + i, ch = c0 + tx * 4 + j;
        if (k < Dk && ch < M && acc[i][j] != 0.f)
          atomicAdd(gflat + go.proj_w[set] + (size_t)k * M + ch, acc[i][j]);
      }
    if (blockIdx.x == 0 && ty == 0)
      for (int j = 0; j < 4; ++j) {
        const int ch = c0 + tx * 4 + j;
        if (ch < M && bsum[j] != 0.f) atomicAdd(gflat + go.proj_b[set] + ch, bsum[j]);
      }
  };
  // The (entry, 32-row chunk) pairs form one sequence of steps; the global loads of step s+1 are
  // issued into registers before the FMAs of step s (the kernel was a load -> barrier -> compute ->
  // barrier chain that exposed the DRAM latency of every chunk).
  constexpr int kPer = kFgRows * kFgTile / 256;   // 8 elements of each operand per thread
  const int chunks_per_entry = (HW + kFgRows - 1) / kFgRows;
  const int n_steps = (e1 - e0) * chunks_per_entry;
  float xr[kPer], br[kPer];
  auto fetch = [&](int step) {
    const int e = e0 + step / chunks_per_entry, p0 = (step % chunks_per_entry) * kFgRows;
    const float* X = md.feat + (size_t)entries[e].b * HW * md.feat_pitch;
    const float* B = dmap + (size_t)e * HW * Mp;
#pragma unroll
    for (int u = 0; u < kPer; ++u) {
      const int idx = threadIdx.x + u * 256;
      const int r = idx / kFgTile, cc = idx - r * kFgTile, p = p0 + r;
      xr[u] = (p < HW && k0 + cc < Dk) ? X[(size_t)p * md.feat_pitch + k0 + cc] : 0.f;
      br[u] = (p < HW && c0 + cc < Mp) ? B[(size_t)p * Mp + c0 + cc] : 0.f;
    }
  };
  if (n_steps > 0) fetch(0);
  for (int step = 0; step < n_steps; ++step) {
    const int e = e0 + step / chunks_per_entry;
    if (step % chunks_per_entry == 0) {
      const int set = entries[e].set;
      if (set != cur_set) {
        flush(cur_set);
        cur_set = set;
        for (int i = 0; i < 4; ++i) { bsum[i] = 0.f; for (int j = 0; j < 4; ++j) acc[i][j] = 0.f; }
      }
    }
    __syncthreads();   // the previous step's readers are done with xs / bs
#pragma unroll
    for (int u = 0; u < kPer; ++u) {
      const int idx = threadIdx.x + u * 256;
      (&xs[0][0])[idx] = xr[u];
      (&bs[0][0])[idx] = br[u];
    }
    __syncthreads();
    if (step + 1 < n_steps) fetch(step + 1);
#pragma unroll 8
    for (int r = 0; r < kFgRows; ++r) {
      const float4 x4 = *reinterpret_cast<const float4*>(&xs[r][ty * 4]);
      const float4 b4 = *reinterpret_cast<const float4*>(&bs[r][tx * 4]);
      const float xv[4] = {x4.x, x4.y, x4.z, x4.w}, bv[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(xv[i], bv[j], acc[i][j]);
      if (ty == 0)
#pragma unroll
        for (int j = 0; j < 4; ++j) bsum[j] += bv[j];
    }
  }
  flush(cur_set);
}

// ---- C[k][c] += Σ_p X[p][k]·B[p][c]: the weight-gradient contraction of every "X·W + b" layer ----
// (feature-side layers: p = the pixels of one B map, X = that image's feature grid; text layers:
// p = the text rows of one weight set, X = the gathered word vectors). Default path; the CUDA-core
// kernels above stay as the exact-fp32 verification path (N2NMN_FLAG_PROJ_FP32_SIMT).
//   CTA tile 128 (k) x 64 (c), 8 warps of 32 x 32 on mma.sync m16n8k8 TF32 (fp32 accumulate), the
//   contraction index streamed 32 rows at a time through a 4-stage cp.async ring: both operands
//   are stored exactly as they lie in memory ([p][k] and [p][c], padded pitches 136 / 72 make the
//   transposed fragment reads conflict-free), so no register staging and no transposition pass.
//   Operands are rounded to TF32 at fragment-load time by adding half an ulp (the tensor core
//   ignores the low 13 bits): one integer add per element where cvt.rna is an instruction sequence.
//   Round 1's kernel staged 64 x 64 tiles through registers with two barriers per 32 rows and 16
//   MMAs per warp between them: 178 us for 3.6 GFLOP (2.4 % of the TF32 peak).
// Segments [blockIdx.z * segs_per_cta, ...) are walked by one CTA and flushed with atomics when the
// weight set changes; CTAs with blockIdx.x == 0 also sum the columns of B (the bias gradient).
constexpr int kXtbM = 128, kXtbN = 64, kXtbP = 32, kXtbStages = 4, kXtbThreads = 256;
constexpr int kXtbXPitch = kXtbM + 8, kXtbBPitch = kXtbN + 8;
constexpr int kXtbStageFloats = kXtbP * (kXtbXPitch + kXtbBPitch);
constexpr size_t kXtbSmemBytes = (size_t)kXtbStages * kXtbStageFloats * sizeof(float);

__device__ __forceinline__ uint32_t tf32_round_bits(float x) { return __float_as_uint(x) + 0x1000u; }

struct FeatGradSrc {   // segment = one B map (entry)
  DevModel md; const float* dmap; const BwdEntry* entries; int n; float* gflat; GradOffsets go;
  __device__ int num_segs() const { return n; }
  __device__ int rows(int) const { return md.HW; }
  __device__ int set(int sg) const { return entries[sg].set; }
  __device__ const float* x_row(int sg, int p) const {
    return md.feat + ((size_t)entries[sg].b * md.HW + p) * md.feat_pitch;
  }
  __device__ const float* b_row(int sg, int p) const { return dmap + ((size_t)sg * md.HW + p) * md.Mp; }
  __device__ int kdim() const { return md.Dk; }
  __device__ int ncols() const { return md.M; }
  __device__ int ncols_pad() const { return md.Mp; }
  __device__ float* w_out(int st) const { return gflat + go.proj_w[st]; }
  __device__ float* b_out(int st) const { return gflat + go.proj_b[st]; }
};
struct TextGradSrc {   // segment = one text weight set
  DevModel md; const float* dtau; const int32_t* text_t; const int32_t* text_b;
  const int32_t* set_start; float* gflat; GradOffsets go;
  __device__ int num_segs() const { return NUM_TEXT_SETS; }
  __device__ int rows(int sg) const { return set_start[sg + 1] - set_start[sg]; }
  __device__ int set(int sg) const { return sg; }
  __device__ const float* x_row(int sg, int p) const {
    const int r = set_start[sg] + p;
    return word_vec_row(md, text_t[r], text_b[r]);
  }
  __device__ const float* b_row(int sg, int p) const { return dtau + (size_t)(set_start[sg] + p) * md.Mp; }
  __device__ int kdim() const { return md.Dt; }
  __device__ int ncols() const { return md.M; }
  __device__ int ncols_pad() const { return md.Mp; }
  __device__ float* w_out(int st) const { return gflat + go.txt_w[st]; }
  __device__ float* b_out(int st) const { return gflat + go.txt_b[st]; }
};
// segment = one answer-head weight set (fc_eltwise of Describe / SameProperty, many classes):
// d(W_out)[m, c] = Σ_q ê[q, m]·dS[q, c] over the questions whose root uses that set; the rows of
// the other questions read a zero row.
struct TailGradSrc {
  DevModel md; const float* ehat; const float* ds; const int32_t* root_set; const float* zero_row;
  int nq, Cp; float* gflat; GradOffsets go; int has_set[NUM_OUT_SETS];
  __device__ int num_segs() const { return NUM_OUT_SETS; }
  __device__ int rows(int sg) const { return has_set[sg] ? nq : 0; }
  __device__ int set(int sg) const { return sg; }
  __device__ const float* x_row(int, int p) const { return ehat + (size_t)p * md.Mp; }
  __device__ const float* b_row(int sg, int p) const {
    return root_set[p] == sg ? ds + (size_t)p * Cp : zero_row;
  }
  __device__ int kdim() const { return md.M; }
  __device__ int ncols() const { return md.C; }
  __device__ int ncols_pad() const { return Cp; }
  __device__ float* w_out(int st) const { return gflat + go.out_w[st]; }
  __device__ float* b_out(int st) const { return gflat + go.out_b[st]; }
};

template <class Src>
__global__ void __launch_bounds__(kXtbThreads) xtb_mma_kernel(const Src src, int segs_per_cta) {
  extern __shared__ __align__(16) float xsm[];
  const int k0 = blockIdx.x * kXtbM, c0 = blockIdx.y * kXtbN;
  const int s0 = blockIdx.z * segs_per_cta, s1 = min(src.num_segs(), s0 + segs_per_cta);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3, wm = warp & 3, wn = warp >> 2;
  const int Kd = src.kdim(), M = src.ncols(), Mp = src.ncols_pad();
  const bool bias_cta = blockIdx.x == 0;
  struct It { int seg, p0; };
  auto settle = [&](It& it) { while (it.seg < s1 && it.p0 >= src.rows(it.seg)) { ++it.seg; it.p0 = 0; } };
  auto load = [&](const It& it, int stage) {
    float* xs = xsm + stage * kXtbStageFloats;
    float* bs = xs + kXtbP * kXtbXPitch;
    const int rows = src.rows(it.seg);
    for (int i = tid; i < kXtbP * (kXtbM / 4); i += kXtbThreads) {
      const int r = i >> 5, q = i & 31, p = it.p0 + r, k = k0 + 4 * q;
      float* dst = xs + r * kXtbXPitch + 4 * q;
      if (p < rows && k < Kd) tp_cp16(dst, src.x_row(it.seg, p) + k);
      else *reinterpret_cast<float4*>(dst) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    for (int i = tid; i < kXtbP * (kXtbN / 4); i += kXtbThreads) {
      const int r = i >> 4, q = i & 15, p = it.p0 + r, cc = c0 + 4 * q;
      float* dst = bs + r * kXtbBPitch + 4 * q;
      if (p < rows && cc < Mp) tp_cp16(dst, src.b_row(it.seg, p) + cc);
      else *reinterpret_cast<float4*>(dst) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  float acc[2][4][4], bsum = 0.f;
  auto zero = [&] {
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int ni = 0; ni < 4; ++ni)
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[mi][ni][i] = 0.f;
    bsum = 0.f;
  };
  auto flush = [&](int st) {
    float* W = src.w_out(st);
    const bool pair_ok = (M & 1) == 0 && (reinterpret_cast<uintptr_t>(W) & 7) == 0;
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int ni = 0; ni < 4; ++ni)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int k = k0 + wm * 32 + mi * 16 + g + 8 * hh;
          const int ch = c0 + wn * 32 + ni * 8 + 2 * t;
          const float v0 = acc[mi][ni][2 * hh], v1 = acc[mi][ni][2 * hh + 1];
          if (k >= Kd || ch >= M) continue;
          float* dst = W + (size_t)k * M + ch;
          if (pair_ok && ch + 1 < M) {   // one 8-byte reduction for the two adjacent channels
            if (v0 != 0.f || v1 != 0.f) atomicAdd(reinterpret_cast<float2*>(dst), make_float2(v0, v1));
          } else {
            if (v0 != 0.f) atomicAdd(dst, v0);
            if (ch + 1 < M && v1 != 0.f) atomicAdd(dst + 1, v1);
          }
        }
    const int ch = c0 + (tid & (kXtbN - 1));
    if (bias_cta && ch < M && bsum != 0.f) atomicAdd(src.b_out(st) + ch, bsum);
  };
  It ld{s0, 0}, cp{s0, 0};
  settle(ld); settle(cp);
  for (int s = 0; s < kXtbStages - 1; ++s) {
    if (ld.seg < s1) { load(ld, s); ld.p0 += kXtbP; settle(ld); }
    tp_commit();
  }
  int cur_set = -1, step = 0;
  zero();
  while (cp.seg < s1) {
    const int st = src.set(cp.seg);
    if (st != cur_set) {
      if (cur_set >= 0) flush(cur_set);
      zero();
      cur_set = st;
    }
    tp_wait<kXtbStages - 2>();
    __syncthreads();
    if (ld.seg < s1) { load(ld, (step + kXtbStages - 1) % kXtbStages); ld.p0 += kXtbP; settle(ld); }
    tp_commit();
    const float* xs = xsm + (step % kXtbStages) * kXtbStageFloats;
    const float* bs = xs + kXtbP * kXtbXPitch;
#pragma unroll
    for (int ks = 0; ks < kXtbP / 8; ++ks) {
      uint32_t a[2][4], b[4][2];
#pragma unroll
      for (int mi = 0; mi < 2; ++mi) {
        const float* xa = xs + (8 * ks + t) * kXtbXPitch + wm * 32 + mi * 16 + g;
        a[mi][0] = tf32_round_bits(xa[0]);
        a[mi][1] = tf32_round_bits(xa[8]);
        a[mi][2] = tf32_round_bits(xa[4 * kXtbXPitch]);
        a[mi][3] = tf32_round_bits(xa[4 * kXtbXPitch + 8]);
      }
#pragma unroll
      for (int ni = 0; ni < 4; ++ni) {
        const float* ba = bs + (8 * ks + t) * kXtbBPitch + wn * 32 + ni * 8 + g;
        b[ni][0] = tf32_round_bits(ba[0]);
        b[ni][1] = tf32_round_bits(ba[4 * kXtbBPitch]);
      }
#pragma unroll
      for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int ni = 0; ni < 4; ++ni)
          asm volatile(
              "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, "
              "{%8,%9}, {%0,%1,%2,%3};"
              : "+f"(acc[mi][ni][0]), "+f"(acc[mi][ni][1]), "+f"(acc[mi][ni][2]), "+f"(acc[mi][ni][3])
              : "r"(a[mi][0]), "r"(a[mi][1]), "r"(a[mi][2]), "r"(a[mi][3]), "r"(b[ni][0]), "r"(b[ni][1]));
    }
    if (bias_cta) {   // column sums of B from the unrounded values: 4 row groups of 8 per column
      const float* bc = bs + (tid >> 6) * 8 * kXtbBPitch + (tid & (kXtbN - 1));
#pragma unroll
      for (int r = 0; r < 8; ++r) bsum += bc[r * kXtbBPitch];
    }
    cp.p0 += kXtbP; settle(cp);
    ++step;
  }
  if (cur_set >= 0) flush(cur_set);
}

// d(word_vecs)[t, b, :] = scale · dtau[row, :] · W_set^T on the same fragments: A = 64 text rows of
// one weight set (groups as in text_proj_kernel), B = 64 rows k of W_set [Dt][Mp], both K-major
// (channel contiguous) exactly as stored. grid = (ceil(Dt/64), groups).
constexpr int kXgThreads = 256, kXgKC = 256;
constexpr int kXgPitch = kXgKC + 4;
constexpr size_t kXgSmemBytes = (size_t)2 * 64 * kXgPitch * sizeof(float);
__global__ void __launch_bounds__(kXgThreads)
text_xgrad_mma_kernel(DevModel md, const float* __restrict__ dtau, const int32_t* __restrict__ text_t,
                      const int32_t* __restrict__ text_b, TextSetRows rows, float* __restrict__ dword,
                      float scale) {
  extern __shared__ __align__(16) float gsm[];
  float* As = gsm;                    // [64 rows][kXgPitch]
  float* Ws = gsm + 64 * kXgPitch;    // [64 k][kXgPitch]
  int set = 0, gi = blockIdx.y, r0, cnt;
  for (; set < NUM_TEXT_SETS; ++set) {
    const int ng = (rows.start[set + 1] - rows.start[set] + 63) / 64;
    if (gi < ng) break;
    gi -= ng;
  }
  r0 = rows.start[set] + gi * 64;
  cnt = min(64, rows.start[set + 1] - r0);
  const int k0 = blockIdx.x * 64, Dt = md.Dt, Mp = md.Mp;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3, wm = warp & 3, wn = warp >> 2;
  float acc[4][4];
#pragma unroll
  for (int ni = 0; ni < 4; ++ni)
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[ni][i] = 0.f;
  const float* W = md.txt_w[set];
  for (int cb = 0; cb < Mp; cb += kXgKC) {
    const int kc = min(kXgKC, Mp - cb), q4 = kc >> 2;
    __syncthreads();
    for (int i = tid; i < 64 * q4; i += kXgThreads) {
      const int r = i / q4, q = i - r * q4;
      float* da = As + r * kXgPitch + 4 * q;
      float* dw = Ws + r * kXgPitch + 4 * q;
      if (r < cnt) tp_cp16(da, dtau + (size_t)(r0 + r) * Mp + cb + 4 * q);
      else *reinterpret_cast<float4*>(da) = make_float4(0.f, 0.f, 0.f, 0.f);
      if (k0 + r < Dt) tp_cp16(dw, W + (size_t)(k0 + r) * Mp + cb + 4 * q);
      else *reinterpret_cast<float4*>(dw) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    tp_commit();
    tp_wait<0>();
    __syncthreads();
    for (int ks = 0; ks < kc / 8; ++ks) {
      const float* aa = As + (wm * 16 + g) * kXgPitch + 8 * ks + t;
      uint32_t a[4] = {tf32_round_bits(aa[0]), tf32_round_bits(aa[8 * kXgPitch]),
                       tf32_round_bits(aa[4]), tf32_round_bits(aa[8 * kXgPitch + 4])};
#pragma unroll
      for (int ni = 0; ni < 4; ++ni) {
        const float* wa = Ws + (wn * 32 + ni * 8 + g) * kXgPitch + 8 * ks + t;
        const uint32_t b0 = tf32_round_bits(wa[0]), b1 = tf32_round_bits(wa[4]);
        asm volatile(
            "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, "
            "{%8,%9}, {%0,%1,%2,%3};"
            : "+f"(acc[ni][0]), "+f"(acc[ni][1]), "+f"(acc[ni][2]), "+f"(acc[ni][3])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
      }
    }
  }
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int r = wm * 16 + g + 8 * hh;
    if (r >= cnt) continue;
    float* dst = dword + ((size_t)text_t[r0 + r] * md.N + text_b[r0 + r]) * Dt;
#pragma unroll
    for (int ni = 0; ni < 4; ++ni)
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int k = k0 + wn * 32 + ni * 8 + 2 * t + j;
        if (k < Dt) dst[k] = acc[ni][hh * 2 + j] * scale;
      }
  }
}

// The scalar part of the policy-search step (exp_clevr/train_clevr_rl_gt_layout.py:119-124) on
// the device, one block: avg = Σ loss / (N·world); coeff_i = (loss_i - baseline) / (N·world) (the
// stop_gradient factor of the policy-gradient loss); pg = Σ coeff_i·log_seq_prob_i; baseline EMA.
// state_out = {new baseline, avg_sample_loss, policy_gradient_loss, l2_reg (zeroed here, summed by
// grad_norm_kernel)}.
__global__ void train_scalars_kernel(const float* __restrict__ loss_sum,
                                     const float* __restrict__ per_sample,
                                     const float* __restrict__ log_seq_prob, int N, int world,
                                     float baseline_decay, const float* __restrict__ state_in,
                                     float* __restrict__ state_out, float* __restrict__ coeff) {
  __shared__ float red[32];
  const float inv = 1.f / ((float)N * (float)world);
  const float avg = loss_sum[0] * inv, base = state_in[0];
  float pg = 0.f;
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    const float cf = (per_sample[i] - base) * inv;
    if (coeff != nullptr) coeff[i] = cf;
    if (log_seq_prob != nullptr) pg = fmaf(cf, log_seq_prob[i], pg);
  }
  pg = warp_sum(pg);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = pg;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += red[i];
    state_out[0] = base + (1.f - baseline_decay) * (avg - base);
    state_out[1] = avg;
    state_out[2] = t;
    state_out[3] = 0.f;
  }
}

}  // namespace n2nmn
