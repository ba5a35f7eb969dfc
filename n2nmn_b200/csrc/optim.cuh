// Per-tensor clip + Adam over a flat variable buffer, shared by the module network (capi.cu) and
// the layout generator (seq2seq.cu). Every variable starts on a 16-byte boundary of the flat
// buffers (offsets are multiples of 4 floats).
#pragma once
#include "common.cuh"

namespace n2nmn {

struct VarSeg { int offset, count, decay; };   // decay = 1 for ".../weights" variables
// Where a variable's new value goes besides the flat buffer (the module network's packed weight
// buffer): kind 0 = plain copy of `count` floats at dst_off; kind 1 = [rows][cols] -> [rows][pitch]
// zero padded. Also the table of prep.cuh's repack_all_kernel.
struct RepackSeg { int src_off, count, cols, kind; long long dst_off; };

// The kernels are static: capi.cu and seq2seq.cu both include this header and launch them, and
// each translation unit keeps its own copy.
// g = g*gscale + wd*w for weights variables (gscale = 1/world after the all-reduce), then Σ g² per
// variable; l2 (optional) += Σ tf.nn.l2_loss(w) over the weights variables (nmn3_model.py:163-166).
static __global__ void grad_norm_kernel(const float* __restrict__ w, float* __restrict__ g,
                                        const VarSeg* __restrict__ segs, float weight_decay,
                                        float gscale,
                                        float* __restrict__ sumsq, float* __restrict__ l2) {
  __shared__ float red[2][8];
  const VarSeg s = segs[blockIdx.y];
  float acc = 0.f, wsq = 0.f;
  const bool touch = s.decay || gscale != 1.f;
  const int n4 = s.count >> 2;
  float4* g4 = reinterpret_cast<float4*>(g + s.offset);
  const float4* w4 = reinterpret_cast<const float4*>(w + s.offset);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += gridDim.x * blockDim.x) {
    float4 gv = g4[i];
    gv.x *= gscale; gv.y *= gscale; gv.z *= gscale; gv.w *= gscale;
    if (s.decay) {
      const float4 wv = w4[i];
      gv.x = fmaf(weight_decay, wv.x, gv.x); gv.y = fmaf(weight_decay, wv.y, gv.y);
      gv.z = fmaf(weight_decay, wv.z, gv.z); gv.w = fmaf(weight_decay, wv.w, gv.w);
      wsq += wv.x * wv.x + wv.y * wv.y + wv.z * wv.z + wv.w * wv.w;
    }
    if (touch) g4[i] = gv;
    acc += gv.x * gv.x + gv.y * gv.y + gv.z * gv.z + gv.w * gv.w;
  }
  if (blockIdx.x == 0 && (int)threadIdx.x < (s.count & 3)) {   // tail of a count not divisible by 4
    const int i = s.offset + 4 * n4 + threadIdx.x;
    float gv = g[i] * gscale;
    if (s.decay) { const float wv = w[i]; gv = fmaf(weight_decay, wv, gv); wsq = fmaf(wv, wv, wsq); }
    if (touch) g[i] = gv;
    acc = fmaf(gv, gv, acc);
  }
  acc = warp_sum(acc);
  wsq = warp_sum(wsq);
  if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = acc; red[1][threadIdx.x >> 5] = wsq; }
  __syncthreads();
  if (threadIdx.x == 0) {   // one reduction per CTA (44 addresses take them all)
    float a = 0.f, q = 0.f;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) { a += red[0][i]; q += red[1][i]; }
    if (a != 0.f) atomicAdd(sumsq + blockIdx.y, a);
    if (l2 != nullptr && s.decay && q != 0.f) atomicAdd(l2, 0.5f * q);
  }
}

// tf.clip_by_norm per tensor, then Adam (TF: lr_t = lr*sqrt(1-b2^t)/(1-b1^t)). kRepack: the new
// value also goes straight to the variable's place in the context's weight buffer (plain or
// row-pitched copy, RepackSeg): the module network's re-pack pass after the step only has the
// K-major wgmma copies and the Transform quadratic form left to do. Without it (the layout
// generator) only the flat buffer is updated; rp / wbuf / pitch are unused.
template <bool kRepack>
static __global__ void adam_clip_kernel(float* __restrict__ w, const float* __restrict__ g,
                                        float* __restrict__ m, float* __restrict__ v,
                                        const VarSeg* __restrict__ segs,
                                        const float* __restrict__ sumsq, float lr_t, float b1,
                                        float b2, float eps, float max_norm,
                                        const RepackSeg* __restrict__ rp, float* __restrict__ wbuf,
                                        int pitch) {
  const VarSeg s = segs[blockIdx.y];
  RepackSeg r{};
  float* dst = nullptr;
  if constexpr (kRepack) { r = rp[blockIdx.y]; dst = wbuf + r.dst_off; }
  const float nrm = sqrtf(sumsq[blockIdx.y]);
  const float scale = (nrm > max_norm) ? max_norm / nrm : 1.f;
  auto step = [&](float wv, float gv, float& mv, float& vv) {
    gv *= scale;
    mv = b1 * mv + (1.f - b1) * gv;
    vv = b2 * vv + (1.f - b2) * gv * gv;
    return wv - lr_t * mv / (sqrtf(vv) + eps);
  };
  auto put = [&](int i, float wn) {   // the packed copy: plain or row-pitched
    if constexpr (kRepack) {
      if (r.kind == 0) dst[i] = wn;
      else { const int row = i / r.cols; dst[(size_t)row * pitch + (i - row * r.cols)] = wn; }
    }
  };
  const int n4 = s.count >> 2;
  float4* w4 = reinterpret_cast<float4*>(w + s.offset);
  float4* m4 = reinterpret_cast<float4*>(m + s.offset);
  float4* v4 = reinterpret_cast<float4*>(v + s.offset);
  const float4* g4 = reinterpret_cast<const float4*>(g + s.offset);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += gridDim.x * blockDim.x) {
    float4 wv = w4[i], mv = m4[i], vv = v4[i];
    const float4 gv = g4[i];
    wv.x = step(wv.x, gv.x, mv.x, vv.x); wv.y = step(wv.y, gv.y, mv.y, vv.y);
    wv.z = step(wv.z, gv.z, mv.z, vv.z); wv.w = step(wv.w, gv.w, mv.w, vv.w);
    w4[i] = wv; m4[i] = mv; v4[i] = vv;
    if constexpr (kRepack) {
      if (r.kind == 0) reinterpret_cast<float4*>(dst)[i] = wv;   // (dst_off: 16-byte aligned slots)
      else { put(4 * i, wv.x); put(4 * i + 1, wv.y); put(4 * i + 2, wv.z); put(4 * i + 3, wv.w); }
    }
  }
  if (blockIdx.x == 0 && (int)threadIdx.x < (s.count & 3)) {
    const int i = 4 * n4 + threadIdx.x, o = s.offset + i;
    float mv = m[o], vv = v[o];
    const float wn = step(w[o], g[o], mv, vv);
    m[o] = mv; v[o] = vv; w[o] = wn;
    put(i, wn);
  }
}

}  // namespace n2nmn
