// C ABI of the N2NMN module-network hot path (include/n2nmn_b200.h): context, weight packing,
// input binding, schedule upload and kernel launches. sm_90a only; no CPU fallback.
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cmath>
#include <cstring>
#include <ctime>
#include <memory>
#include <string>
#include <vector>

#include "../../include/n2nmn_b200.h"
#include "common.cuh"
#include "launch.cuh"
#include "node_eval.cuh"
#include "prep.cuh"
#include "proj_simt.cuh"
#include "proj_wgmma.cuh"
#include "schedule.hpp"
#include "text_proj.cuh"
#include "tree_kernel.cuh"
#include "head_kernel.cuh"
#include "backward.cuh"
#include "head_tail_wgmma.cuh"
#include "wgrad_wgmma.cuh"

using namespace n2nmn;

namespace {

thread_local std::string g_err;

int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}

// Lazy workspaces allocate through this, so that a retry after a failed setup allocates only what
// is still missing.
template <class T>
cudaError_t alloc_once(T** p, size_t bytes) {
  return *p ? cudaSuccess : cudaMalloc(p, bytes);
}

inline int round_up(int x, int m) { return (x + m - 1) / m * m; }

// VQA features gain two coordinate channels and its Transform has no filter bank
SchedShape sched_shape(const n2nmn_config& g) {
  const bool vqa = g.family == N2NMN_VQA;
  return SchedShape{g.family, g.H, g.W, g.D + (vqa ? 2 : 0), g.text_dim, g.map_dim,
                    round_up(g.map_dim, 256), g.num_choices, vqa ? 1 : g.kernel_size, g.max_T};
}

enum VarKind { VK_PLAIN = 0, VK_PROJ_W, VK_PROJ_B, VK_PITCHED };

struct Variable {
  std::string name;
  std::vector<int64_t> shape;
  VarKind kind;
  int set;           // projection set for VK_PROJ_*
  size_t offset;     // float offset of the plain copy inside wbuf
  size_t count;
  const float** slot;   // DevModel pointer to fill (plain copy)
  bool loaded;
};

constexpr int kTableSlots = 4;

struct TableSlot {
  uint8_t* host = nullptr;   // pinned staging
  uint8_t* dev = nullptr;
  uint64_t uid = 0;          // schedule resident here (0 = none)
  cudaEvent_t last_use = nullptr;
};

struct TableOffsets {
  size_t nodes, q_ptr, text_t, text_b, groups, work, img_ptr, node_text, node_out, mslot,
      wave_nodes, bwd_nodes, entry_order, node_entry, entries, text_set_start, labels, head_work, head_list, pool_img,
      total;
};

// Calls f(offset field, host bytes, byte count) for every schedule table, in device order. The
// labels of a training schedule come from the caller (`labels`, may be null), not from S.
template <class O, class F>
void for_each_table(const HostSchedule& S, const int32_t* labels, O& o, F&& f) {
  auto v = [&](auto& off, const auto& vec) { f(off, vec.data(), vec.size() * sizeof(vec[0])); };
  v(o.nodes, S.nodes); v(o.q_ptr, S.q_ptr); v(o.text_t, S.text_t); v(o.text_b, S.text_b);
  v(o.groups, S.groups); v(o.work, S.work); v(o.img_ptr, S.img_ptr); v(o.node_text, S.node_text);
  v(o.node_out, S.node_out); v(o.mslot, S.mslot); v(o.wave_nodes, S.wave_nodes);
  v(o.bwd_nodes, S.bwd_nodes); v(o.entry_order, S.entry_order); v(o.node_entry, S.node_entry);
  v(o.entries, S.entries); v(o.text_set_start, S.text_set_start);
  f(o.labels, labels, S.train ? (S.q_ptr.size() - 1) * 4 : 0);
  v(o.head_work, S.head_work); v(o.head_list, S.head_list); v(o.pool_img, S.pool_img);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

}  // namespace

struct n2nmn_sched {
  HostSchedule hs;
  uint64_t uid;
  SchedShape shp;
};

struct n2nmn_ctx {
  n2nmn_config cfg;
  int device = 0, num_sms = 0;
  int HW = 0, Dk = 0, Kp = 0, Mp = 0;
  int G = 1;                   // segments (batches) one set of launches may cover
  int QB = 0;                  // question capacity of one launch: G * max_batch
  SchedShape shp;
  DevModel md;
  std::vector<Variable> vars;
  float* wbuf = nullptr;
  size_t wbuf_floats = 0;
  float* proj_wt[NUM_PROJ_SETS] = {};      // [Mp][Kp], allocated for the sets the family owns
  float* proj_bias[NUM_PROJ_SETS] = {};    // [Mp]
  bool proj_used[NUM_PROJ_SETS] = {};
  int num_store_sets = 0;
  // inputs
  bool bound = false;
  int N = 0, T = 0;
  float* feat_aug = nullptr;   // ctx-owned re-pitched / coordinate-augmented copy
  // workspaces
  TextBufs tb = {nullptr, nullptr, nullptr, nullptr};
  int text_rows_cap = 0;
  float* arena = nullptr;
  int arena_slots = 0;
  float* mbuf = nullptr;
  int mbuf_slots = 0;
  float* pooled = nullptr;     // [2*QB][Kp] pooled feature vectors of Describe / SameProperty roots
  float* pool_att = nullptr;   // [2*QB][HWp] input maps of the answer roots (softmaxed for those)
  float* conv_quad = nullptr;  // [quad_rows][Mp] Transform quadratic-form matrix (common.cuh)
  int head_nn = 16;            // root nodes per head-kernel CTA
  int head_smem_bytes = 0;
  float* scores_tmp = nullptr;
  TableSlot slots[kTableSlots];
  size_t table_cap = 0;
  int next_slot = 0;
  ProjTensorMaps tmaps;
  EncodeTiledFn encode = nullptr;
  int node_smem_bytes = 0;
  int tree_smem_bytes = 0;
  int stack_cap = 0;           // attention-stack slots the tree kernel may use
  int tree_cluster = 0;        // 0 = choose from the batch size (n2nmn_set_tree_cluster)
  int proj_max_ctas = 0;       // 0 = one CTA per SM; else cap of the persistent projection grid
  n2nmn_sched module_sched;    // scratch schedule of n2nmn_module_fwd
  n2nmn_sched step_sched;      // scratch schedule of n2nmn_forward_tokens
  // training workspaces (allocated on first use; ready once every allocation and attribute is set)
  bool train_ready = false;
  const int32_t* train_labels = nullptr;   // host labels of the step being compiled
  const uint8_t* last_tables = nullptr;    // device tables of the last run_tables
  TableOffsets last_offsets;
  float* dscores = nullptr;
  float* per_sample = nullptr;
  float* dtau = nullptr;
  float* dmap = nullptr;
  float* dstencil = nullptr;
  float* gmap = nullptr;
  float* phi_buf = nullptr;
  bool wg_ok = false;   // shapes fit wgrad_wgmma_kernel (Mp % 256 == 0, Dk >= 128)
  // batched answer-tail backward of the many-class heads (C > 32, backward.cuh tail_prep_kernel)
  float* dehat = nullptr;        // [NB][Mp] d loss / d ê
  float* ds_hi = nullptr;        // [NB][Cp] d loss / d scores, and its TF32 remainder
  float* ds_lo = nullptr;
  float* tail_zero = nullptr;    // max(Cp, Mp) zeros
  int32_t* root_set = nullptr;   // [NB]
  float** tail_dst = nullptr;    // [NUM_OUT_SETS][NB] dê row addresses
  float* out_wp_lo[NUM_OUT_SETS] = {};   // remainder planes of out_wp
  HeadTailMaps tail_maps[NUM_OUT_SETS];
  // many-class answer heads (C > 32): ê rows + score-row addresses of the roots of a launch, and
  // the fc_eltwise matrices with rows pitched to a multiple of 4 floats (cp.async alignment)
  float* ehat = nullptr;
  float** ehat_dst = nullptr;
  float* out_wp[NUM_OUT_SETS] = {};
  int Cp = 0;
  // ... and its wgmma form (head_tail_wgmma.cuh): remainder plane of ê, W_outᵀ planes, maps
  float* ehat_lo = nullptr;
  float* out_wt_hi[NUM_OUT_SETS] = {};
  float* out_wt_lo[NUM_OUT_SETS] = {};
  HeadTailMaps ht_maps[NUM_OUT_SETS];
  int Cpad = 0;   // [max_batch][HW][Mp] scratch of the Transform backward
  int dmap_entries = 0;
  VarSeg* d_segs = nullptr;                // Adam segment table, ready with d_sumsq
  float* d_sumsq = nullptr;
  bool segs_ready = false;
  RepackSeg* d_repack = nullptr;           // fused re-pack tables (n2nmn_load_flat_weights)
  bool repack_ready = false;
  ProjRepack proj_repack;
  int proj_repack_sets = 0;
  float dword_scale = 1.f;                 // n2nmn_set_grad_scale
  GradOffsets go;
  std::vector<int64_t> flat_offset;
  int64_t flat_size = 0;
  // e2e staging
  float* e2e_feat = nullptr;
  float* e2e_wv = nullptr;
  float* e2e_scores = nullptr;
  uint16_t* e2e_feat_f16 = nullptr;   // fp16 staging of host features (host_f16 path)
  // profiling
  bool profiling = false;
  std::vector<cudaEvent_t> ev;
  std::vector<const char*> ev_names;
  int ev_used = 0;
  int64_t launches = 0;
};

namespace {

std::atomic<uint64_t> g_uid{1};

void add_var(n2nmn_ctx* c, const std::string& name, std::vector<int64_t> shape, VarKind kind,
             int set, const float** slot) {
  Variable v;
  v.name = name; v.shape = shape; v.kind = kind; v.set = set; v.slot = slot; v.loaded = false;
  v.count = 1;
  for (int64_t d : shape) v.count *= (size_t)d;
  v.offset = c->wbuf_floats;
  const size_t stored = (kind == VK_PITCHED) ? v.count / (size_t)shape.back() * c->Mp : v.count;
  c->wbuf_floats += (stored + 3) & ~(size_t)3;
  c->vars.push_back(v);
}

// proj_set >= 0: conv_image (repacked for the tensor cores); proj_set == -2: a [rows][M] matrix
// stored with row pitch Mp (fc_text / fc_att) for aligned float4 loads.
void add_layer(n2nmn_ctx* c, const std::string& scope, std::vector<int64_t> wshape,
               const float** wslot, const float** bslot, int proj_set = -1) {
  add_var(c, scope + "/weights", wshape,
          proj_set >= 0 ? VK_PROJ_W : (proj_set == -2 ? VK_PITCHED : VK_PLAIN), proj_set, wslot);
  add_var(c, scope + "/biases", {wshape.back()}, proj_set >= 0 ? VK_PROJ_B : VK_PLAIN, proj_set,
          bslot);
}

// Variable table; order and names match n2nmn_b200/weights.py::variable_shapes.
void build_variables(n2nmn_ctx* c) {
  const n2nmn_config& g = c->cfg;
  DevModel& md = c->md;
  const int64_t D = c->Dk, M = g.map_dim, Dt = g.text_dim, C = g.num_choices, k = g.kernel_size;
  const int64_t HW = c->HW;
  add_layer(c, "FindModule/conv_image", {D, M}, &md.proj_w[PS_FIND], nullptr, PS_FIND);
  add_layer(c, "FindModule/fc_text", {Dt, M}, &md.txt_w[TS_FIND], &md.txt_b[TS_FIND], -2);
  add_layer(c, "FindModule/conv_eltwise", {M, 1}, &md.elt_w[ES_FIND], &md.elt_b[ES_FIND]);
  if (g.family == N2NMN_VQA) {
    add_layer(c, "TransformModule/conv_image", {D, M}, &md.proj_w[PS_FSP_IMG], nullptr, PS_FSP_IMG);
    add_layer(c, "TransformModule/fc_text", {Dt, M}, &md.txt_w[TS_FSP], &md.txt_b[TS_FSP], -2);
    add_layer(c, "TransformModule/fc_att", {D, M}, &md.proj_w[PS_FSP_ATT], nullptr, PS_FSP_ATT);
    add_layer(c, "TransformModule/conv_eltwise", {M, 1}, &md.elt_w[ES_FSP], &md.elt_b[ES_FSP]);
  } else {
    add_layer(c, "TransformModule/conv_maps", {k, k, 1, M}, &md.conv_k, &md.conv_b, -2);
    add_layer(c, "TransformModule/text_fc", {Dt, M}, &md.txt_w[TS_TRANSFORM],
              &md.txt_b[TS_TRANSFORM], -2);
    add_layer(c, "TransformModule/conv_eltwise", {M, 1}, &md.elt_w[ES_TRANSFORM],
              &md.elt_b[ES_TRANSFORM]);
  }
  if (g.family == N2NMN_SHAPES) {
    add_layer(c, "AnswerModule/fc_scores", {3, C}, &md.sc_w[SS_EXIST], &md.sc_b[SS_EXIST]);
    return;
  }
  if (g.family == N2NMN_CLEVR) {
    add_layer(c, "FindSamePropertyModule/conv_image", {D, M}, &md.proj_w[PS_FSP_IMG], nullptr,
              PS_FSP_IMG);
    add_layer(c, "FindSamePropertyModule/fc_text", {Dt, M}, &md.txt_w[TS_FSP], &md.txt_b[TS_FSP], -2);
    add_layer(c, "FindSamePropertyModule/fc_att", {D, M}, &md.proj_w[PS_FSP_ATT], nullptr,
              PS_FSP_ATT);
    add_layer(c, "FindSamePropertyModule/conv_eltwise", {M, 1}, &md.elt_w[ES_FSP],
              &md.elt_b[ES_FSP]);
    add_layer(c, "ExistModule/fc_scores", {3, C}, &md.sc_w[SS_EXIST], &md.sc_b[SS_EXIST]);
    add_layer(c, "CountModule/fc_scores", {HW + 2, C}, &md.sc_w[SS_COUNT], &md.sc_b[SS_COUNT]);
    add_layer(c, "EqualNumModule/fc_scores", {2 * (HW + 2), C}, &md.sc_w[SS_EQUAL],
              &md.sc_b[SS_EQUAL]);
    add_layer(c, "MoreNumModule/fc_scores", {2 * (HW + 2), C}, &md.sc_w[SS_MORE],
              &md.sc_b[SS_MORE]);
    add_layer(c, "LessNumModule/fc_scores", {2 * (HW + 2), C}, &md.sc_w[SS_LESS],
              &md.sc_b[SS_LESS]);
    add_layer(c, "SamePropertyModule/fc_text", {Dt, M}, &md.txt_w[TS_SAMEPROP],
              &md.txt_b[TS_SAMEPROP], -2);
    add_layer(c, "SamePropertyModule/fc_att_0", {D, M}, &md.proj_w[PS_SP_ATT0], nullptr,
              PS_SP_ATT0);
    add_layer(c, "SamePropertyModule/fc_att_1", {D, M}, &md.proj_w[PS_SP_ATT1], nullptr,
              PS_SP_ATT1);
    add_layer(c, "SamePropertyModule/fc_eltwise", {M, C}, &md.out_w[OS_SAMEPROP],
              &md.out_b[OS_SAMEPROP]);
  }
  add_layer(c, "DescribeModule/fc_text", {Dt, M}, &md.txt_w[TS_DESCRIBE], &md.txt_b[TS_DESCRIBE], -2);
  add_layer(c, "DescribeModule/fc_att", {D, M}, &md.proj_w[PS_DESC_ATT], nullptr, PS_DESC_ATT);
  add_layer(c, "DescribeModule/fc_eltwise", {M, C}, &md.out_w[OS_DESCRIBE],
            &md.out_b[OS_DESCRIBE]);
}

int encode_2d(n2nmn_ctx* c, CUtensorMap* map, const float* base, uint64_t inner, uint64_t outer,
              uint64_t pitch_elems, uint32_t box_inner, uint32_t box_outer) {
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {pitch_elems * sizeof(float)};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = c->encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims,
                         strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return fail(N2NMN_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult " + std::to_string(r));
  return 0;
}

TableOffsets table_offsets(const HostSchedule& S) {
  TableOffsets o;
  size_t off = 0;
  for_each_table(S, nullptr, o, [&](size_t& at, const void*, size_t bytes) {
    at = off;
    off += (bytes + 15) & ~(size_t)15;
  });
  o.total = off;
  return o;
}

// The device copy of a schedule's tables.
struct DevTables {
  const uint8_t* d;
  TableOffsets o;
  template <class T = int32_t>
  const T* at(size_t off) const { return reinterpret_cast<const T*>(d + off); }
};

void prof_mark(n2nmn_ctx* c, const char* name, cudaStream_t st) {
  if (!c->profiling) return;
  if (c->ev_used >= (int)c->ev.size()) {
    cudaEvent_t e;
    cudaEventCreate(&e);
    c->ev.push_back(e);
    c->ev_names.push_back(name);
  }
  c->ev_names[c->ev_used] = name;
  cudaEventRecord(c->ev[c->ev_used++], st);
}

// Every kernel launch of the context goes through here and is counted once.
template <class... KArgs, class... Args>
int ctx_launch(n2nmn_ctx* c, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
               cudaStream_t st, LaunchAttrs a, Args... args) {
  return launch(c->launches, kernel, grid, block, smem, st, a, args...);
}

// Kernel variants, chosen in one place for the attribute setup and the launch.
auto tree_variant(int ks, bool direct) {
  if (direct) return ks == 5 ? &tree_kernel<5, true> : &tree_kernel<3, true>;
  return ks == 5 ? &tree_kernel<5, false> : &tree_kernel<3, false>;
}
auto wave_variant(int ks) { return ks == 5 ? &wave_kernel<5> : &wave_kernel<3>; }
auto head_variant(int nn) {
  return nn == 16 ? &head_kernel<16> : nn == 8 ? &head_kernel<8> : &head_kernel<4>;
}
// VQA walks Find-type nodes only (in two channel passes when wide); the conv families run the
// Transform instantiation on a level with Transform nodes (tr) and the lighter one otherwise
auto bwd_variant(bool vqa, bool tr, int ks, bool wide) {
  if (vqa) return wide ? &tree_bwd_kernel<1, false, true> : &tree_bwd_kernel<1, false, false>;
  if (tr) return ks == 5 ? &tree_bwd_kernel<5, true> : &tree_bwd_kernel<3, true>;
  return ks == 5 ? &tree_bwd_kernel<5, false> : &tree_bwd_kernel<3, false>;
}

// Makes the schedule's tables resident in a table slot, uploading them unless a slot holds them.
int upload_tables(n2nmn_ctx* c, const n2nmn_sched* sc, const TableOffsets& o, cudaStream_t st,
                  TableSlot** out) {
  for (int i = 0; i < kTableSlots; ++i)
    if (c->slots[i].uid == sc->uid) *out = &c->slots[i];
  if (*out) return 0;
  TableSlot* slot = *out = &c->slots[c->next_slot];
  c->next_slot = (c->next_slot + 1) % kTableSlots;
  CUDA_TRY(cudaEventSynchronize(slot->last_use));   // previous tenant no longer in flight
  for_each_table(sc->hs, c->train_labels, o, [&](size_t at, const void* src, size_t bytes) {
    if (src && bytes) std::memcpy(slot->host + at, src, bytes);
  });
  CUDA_TRY(cudaMemcpyAsync(slot->dev, slot->host, o.total, cudaMemcpyHostToDevice, st));
  slot->uid = sc->uid;
  return 0;
}

// K1: text projections (+ the quadratic-form coefficients of the Transform nodes)
int text_stage(n2nmn_ctx* c, const HostSchedule& S, const DevTables& t, cudaStream_t st) {
  if (S.groups.empty()) return 0;
  TextSetRows tsr;
  for (int i = 0; i <= NUM_TEXT_SETS; ++i) tsr.start[i] = S.text_set_start[i];
  TRY(ctx_launch(c, text_proj_kernel, dim3((unsigned)(c->Mp / kMmaCols), (unsigned)S.groups.size()),
                 kMmaThreads, mma_smem_bytes(4, kTextStages), st, {}, c->md, c->tb, tsr,
                 t.at(t.o.text_t), t.at(t.o.text_b)));
  prof_mark(c, "text_proj_kernel", st);
  const int tr0 = S.text_set_start[TS_TRANSFORM];
  const int trn = S.text_set_start[TS_TRANSFORM + 1] - tr0;
  if (trn > 0 && c->conv_quad) {
    const int qcols = quad_pitch(c->cfg.kernel_size) - quad_u_pitch(c->cfg.kernel_size);
    TRY(ctx_launch(c, quad_kernel,
                   dim3((unsigned)(1 + (qcols + kMmaCols - 1) / kMmaCols), (unsigned)((trn + 63) / 64)),
                   kMmaThreads, mma_smem_bytes(4, kTextStages), st, {true}, c->md, c->tb,
                   tr0, trn));
    prof_mark(c, "quad_kernel", st);
  }
  return 0;
}

// K2: conv_image contraction with fused Find / stored FindSameProperty maps
int contraction_stage(n2nmn_ctx* c, const HostSchedule& S, const DevTables& t, float* arena,
                      cudaStream_t st) {
  if (S.work.empty()) return 0;
  ProjParams p;
  p.work = t.at<ProjWork>(t.o.work);
  p.num_tiles = (int)S.work.size();
  p.total_rows = c->md.N * c->HW;
  p.num_seg = c->md.num_seg;
  p.seg_images = c->md.N;
  p.n_tiles = c->Mp / 256;
  p.k_blocks = (c->Dk + kBK - 1) / kBK;
  p.HW = c->HW; p.M = c->cfg.map_dim; p.Mp = c->Mp; p.Dk = c->Dk;
  p.feat_pitch = c->md.feat_pitch;
  for (int s = 0; s < kMaxSeg; ++s) p.feat_seg[s] = c->md.feat_seg[s];
  for (int s = 0; s < NUM_PROJ_SETS; ++s) {
    p.bias[s] = c->proj_bias[s];
    p.w_orig[s] = c->md.proj_w[s];
  }
  p.img_ptr = t.at(t.o.img_ptr);
  p.node_text = t.at(t.o.node_text);
  p.node_out = t.at(t.o.node_out);
  p.tauw = c->tb.tauw; p.tau2 = c->tb.tau2;
  p.elt_b = c->md.elt_b[ES_FIND];
  p.arena = arena;
  p.mslot = t.at(t.o.mslot);
  p.num_images = (int)(S.mslot.size() / NUM_PROJ_SETS);
  p.mbuf = c->mbuf;
  // persistent grid: CTA i walks the tiles i, i + CTAs, ...
  const int max_ctas = c->proj_max_ctas > 0 ? std::min(c->proj_max_ctas, c->num_sms) : c->num_sms;
  const int ctas = std::max(1, std::min(p.num_tiles, max_ctas));
  if (c->cfg.flags & N2NMN_FLAG_PROJ_FP32_SIMT) {
    const size_t smem = (size_t)(kSimtRows * kSimtKChunk + kSimtRows * c->Mp) * sizeof(float);
    TRY(ctx_launch(c, proj_simt_kernel, p.num_tiles, 256, smem, st, {}, p));
    prof_mark(c, "proj_simt_kernel", st);
  } else {
    TRY(ctx_launch(c, proj_wgmma_kernel, ctas, kProjThreads, proj_smem_bytes(), st, {true},
                   c->tmaps, p));
    prof_mark(c, "proj_wgmma_kernel", st);
  }
  return 0;
}

// K3: node evaluation, by depth waves or one tree walk per question
int node_stage(n2nmn_ctx* c, const HostSchedule& S, const DevTables& t, const NodeCtx& nc,
               float* const* scores_seg, bool use_wave, bool write_arena, cudaStream_t st) {
  const int NQ = (int)S.q_ptr.size() - 1;
  const int nseg = std::max(1, S.num_seg);
  const int ks = c->cfg.kernel_size;
  const NodeRec* d_nodes = t.at<NodeRec>(t.o.nodes);
  if (use_wave) {
    for (int s = 0; s < nseg; ++s)
      CUDA_TRY(cudaMemsetAsync(scores_seg[s], 0,
                               (size_t)(nseg > 1 ? S.N : NQ) * c->cfg.num_choices * sizeof(float),
                               st));
    for (int dep = 1; dep <= S.max_depth; ++dep) {
      const int first = S.wave_ptr[dep], cnt = S.wave_ptr[dep + 1] - first;
      if (cnt == 0) continue;
      TRY(ctx_launch(c, wave_variant(ks), cnt, kNodeThreads, c->node_smem_bytes, st, {}, nc,
                     d_nodes, t.at(t.o.wave_nodes), first));
      prof_mark(c, "wave_kernel", st);
    }
    return 0;
  }
  if (NQ <= 0) return 0;
  // cluster size: spread one question over several SMs while the batch is small
  int cs = c->tree_cluster;
  if (cs <= 0) cs = (NQ * 4 <= 2 * c->num_sms) ? 4 : (NQ * 2 <= 2 * c->num_sms) ? 2 : 1;
  const int slots = std::max(1, S.max_stack);
  const size_t smem = sizeof(float) * (size_t)tree_smem_layout(
      c->cfg.H, c->cfg.W, c->Mp, ks, c->cfg.map_dim, c->cfg.num_choices, slots,
      S.pooled_direct).total;
  const int wa = (write_arena ? kTreeWriteArena : 0) |
                 ((c->cfg.flags & N2NMN_FLAG_PROJ_FP32_SIMT) ? kTreeFp32Stencil : 0);
  TRY(ctx_launch(c, tree_variant(ks, S.pooled_direct), NQ * cs, kNodeThreads, smem, st,
                 {true, (unsigned)cs}, nc, d_nodes, t.at(t.o.q_ptr), cs, slots, wa));
  prof_mark(c, "tree_kernel", st);
  return 0;
}

// K4: batched answer heads of the attention-pooled roots of the tree executor
int head_stage(n2nmn_ctx* c, const HostSchedule& S, const DevTables& t, const NodeCtx& nc,
               cudaStream_t st) {
  if (!S.pooled_direct || S.head_work.empty()) return 0;
  if ((int)S.num_pool_rows > 2 * c->QB)
    return fail(N2NMN_ERR_CAPACITY, "too many pooled root nodes for this context");
  const LaunchAttrs pdl{true};
  if (S.num_feat_rows > 0) {   // pooled features: one CTA per (root row, 128-channel chunk)
    const int HWp = (c->HW + 3) & ~3;
    const int quads = c->md.feat_pitch / 4;
    TRY(ctx_launch(c, pool_kernel,
                   dim3((unsigned)S.num_feat_rows, (unsigned)((quads + kPoolQuads - 1) / kPoolQuads)),
                   kPoolQuads * kPoolSlices, (size_t)(HWp + 4 * kPoolQuads * kPoolSlices) * sizeof(float),
                   st, pdl, nc, t.at(t.o.pool_img), HWp));
    prof_mark(c, "pool_kernel", st);
  }
  TRY(ctx_launch(c, head_variant(c->head_nn), (unsigned)S.head_work.size(), kHeadThreads,
                 (size_t)c->head_smem_bytes, st, pdl, nc, t.at<NodeRec>(t.o.nodes),
                 t.at<HeadWork>(t.o.head_work), t.at(t.o.head_list)));
  prof_mark(c, "head_kernel", st);
  if (!c->ehat) return 0;
  // fc_eltwise of the Describe-type roots as one GEMM per weight set
  for (int op : {OP_DESCRIBE, OP_SAME_PROPERTY}) {
    int r0 = 1 << 30, r1 = 0;
    for (const HeadWork& w : S.head_work)
      if (w.op == op) { r0 = std::min(r0, (int)w.first); r1 = std::max(r1, (int)(w.first + w.count)); }
    if (r1 <= r0) continue;
    const int os = op == OP_DESCRIBE ? OS_DESCRIBE : OS_SAMEPROP;
    if (!c->out_wp[os]) return fail(N2NMN_ERR_STATE, "answer-head weights not packed");
    TRY(ctx_launch(c, head_tail_wgmma_kernel,
                   dim3((unsigned)(c->Cpad / kHtN), (unsigned)((r1 - r0 + kHtM - 1) / kHtM)),
                   kHtThreads, kHtSmemBytes, st, pdl, c->ht_maps[os], c->md.out_b[os],
                   (float* const*)c->ehat_dst, r0, r1 - r0, (int)c->cfg.num_choices,
                   (int)c->cfg.map_dim));
    // named after the retired mma.sync tail kernel: launch-time reports are keyed on this name
    prof_mark(c, "head_tail_gemm_kernel", st);
  }
  return 0;
}

// Uploads (if needed) and launches everything for one compiled batch.
int run_tables(n2nmn_ctx* c, n2nmn_sched* sc, float* const* scores_seg, float* arena,
               cudaStream_t st, bool force_wave = false, bool write_arena = false) {
  const bool use_wave = (c->cfg.flags & N2NMN_FLAG_WAVE_EXECUTOR) || force_wave ||
                        sc->hs.max_stack > c->stack_cap;
  if (use_wave && sc->hs.pooled_direct) {
    // the wave executor evaluates Describe / SameProperty from stored fc_att maps: rebuild the
    // derived tables in that form (layouts deeper than the shared-memory stack end up here)
    sc->hs.pooled_direct = false;
    if (int rc = finalize_schedule(sc->shp, sc->hs.N, &sc->hs, false))
      return fail(rc, "finalize_schedule failed");
    sc->uid = g_uid++;
  }
  if (use_wave) build_waves(&sc->hs);
  const HostSchedule& S = sc->hs;
  const TableOffsets o = table_offsets(S);
  if (o.total > c->table_cap)
    return fail(N2NMN_ERR_CAPACITY, "schedule tables exceed the context capacity");
  if ((int)S.text_t.size() > c->text_rows_cap)
    return fail(N2NMN_ERR_CAPACITY, "too many text nodes for this context");
  if (S.num_mslots > c->mbuf_slots)
    return fail(N2NMN_ERR_CAPACITY, "too many stored feature maps for this context");
  TableSlot* slot = nullptr;
  TRY(upload_tables(c, sc, o, st, &slot));
  const DevTables t{slot->dev, o};
  c->last_tables = slot->dev;
  c->last_offsets = o;

  NodeCtx nc;
  nc.md = c->md; nc.tb = c->tb; nc.arena = arena; nc.scores = scores_seg[0]; nc.mbuf = c->mbuf;
  nc.pooled = c->pooled; nc.pool_pitch = c->Kp; nc.pool_att = c->pool_att;
  nc.phi_out = S.train ? c->phi_buf : nullptr;
  nc.ehat = c->ehat; nc.ehat_lo = c->ehat_lo; nc.ehat_dst = c->ehat_dst;
  // several segments: question q writes row q % N of segment q / N; one segment: row q (the
  // per-module entry point numbers its call rows beyond the bound batch size)
  const int nseg = std::max(1, S.num_seg);
  nc.score_rows = nseg > 1 ? S.N : (1 << 30);
  for (int s = 0; s < kMaxSeg; ++s) nc.scores_seg[s] = scores_seg[s < nseg ? s : 0];

  // every kernel of the step after the first is a programmatic dependent launch of its
  // predecessor (each calls griddepcontrol.wait before it touches the predecessor's output)
  c->ev_used = 0;
  prof_mark(c, "begin", st);
  TRY(text_stage(c, S, t, st));
  TRY(contraction_stage(c, S, t, arena, st));
  TRY(node_stage(c, S, t, nc, scores_seg, use_wave, write_arena, st));
  TRY(head_stage(c, S, t, nc, st));
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaEventRecord(slot->last_use, st));
  return 0;
}

// The many-class answer tail's copies of fc_eltwise set `os` (row-pitched, and split into TF32
// planes for wgmma), from its [map_dim, C] weights at `src`.
int pack_out_weights(n2nmn_ctx* c, int os, const float* src, cudaStream_t st) {
  if (!c->out_wp[os]) return 0;
  TRY(ctx_launch(c, pitch_rows_kernel, c->cfg.map_dim, 256, 0, st, {}, src, c->cfg.map_dim,
                 c->cfg.num_choices, c->out_wp[os], c->Cp));
  if (c->out_wt_hi[os])
    TRY(ctx_launch(c, out_wt_split_kernel, dim3((c->Cpad + 31) / 32, (c->Mp + 31) / 32), dim3(32, 8),
                   0, st, {}, src, c->cfg.map_dim, c->cfg.num_choices, c->out_wt_hi[os],
                   c->out_wt_lo[os], c->Mp, c->Cpad));
  return 0;
}

int update_conv_quad(n2nmn_ctx* c, cudaStream_t st) {
  if (!c->conv_quad) return 0;
  return ctx_launch(c, conv_quad_kernel, quad_pitch(c->cfg.kernel_size), 256, 0, st, {},
                    c->md.conv_k, c->md.conv_b, c->md.elt_w[ES_TRANSFORM], c->cfg.kernel_size,
                    c->cfg.map_dim, c->Mp, c->conv_quad);
}

int check_ready(n2nmn_ctx* c) {
  if (!c->bound) return fail(N2NMN_ERR_STATE, "n2nmn_bind_inputs has not been called");
  for (const Variable& v : c->vars)
    if (!v.loaded) return fail(N2NMN_ERR_STATE, "variable not set: " + v.name);
  return 0;
}

}  // namespace

// ================================================================================== C ABI
namespace n2nmn {
int fail_with(int code, const std::string& msg) { return fail(code, msg); }   // other TUs
}

extern "C" {

const char* n2nmn_last_error(void) { return g_err.c_str(); }

int n2nmn_create(const n2nmn_config* cfg, n2nmn_ctx** out) {
  if (!cfg || !out) return fail(N2NMN_ERR_ARG, "null argument");
  if (cfg->abi_version != N2NMN_ABI_VERSION) return fail(N2NMN_ERR_ARG, "ABI version mismatch");
  if (cfg->family < 0 || cfg->family > 2 || cfg->H <= 0 || cfg->W <= 0 || cfg->D <= 0 ||
      cfg->map_dim <= 0 || cfg->map_dim > 1024 || cfg->num_choices <= 0 || cfg->max_batch <= 0 ||
      cfg->max_T <= 0 || cfg->text_dim <= 0 || cfg->max_group < 0 || cfg->max_group > kMaxSeg)
    return fail(N2NMN_ERR_ARG, "bad configuration");
  if (cfg->family != N2NMN_VQA && cfg->kernel_size != 3 && cfg->kernel_size != 5)
    return fail(N2NMN_ERR_ARG, "kernel_size must be 3 or 5");
  CUDA_TRY(cudaSetDevice(cfg->device));
  cudaDeviceProp prop;
  CUDA_TRY(cudaGetDeviceProperties(&prop, cfg->device));
  if (prop.major != 9)
    return fail(N2NMN_ERR_DEVICE, std::string("n2nmn_b200 needs an sm_90 GPU, found sm_") +
                                      std::to_string(prop.major) + std::to_string(prop.minor));
  // every failure below frees what was built so far (n2nmn_destroy takes a partial context)
  std::unique_ptr<n2nmn_ctx, int (*)(n2nmn_ctx*)> owner(new n2nmn_ctx(), n2nmn_destroy);
  n2nmn_ctx* c = owner.get();
  c->shp = sched_shape(*cfg);
  c->cfg = *cfg;
  c->cfg.kernel_size = c->shp.ksize;
  c->device = cfg->device;
  c->num_sms = prop.multiProcessorCount;
  c->HW = cfg->H * cfg->W;
  c->Dk = c->shp.Dk;
  c->Kp = round_up(c->Dk, kBK);
  c->Mp = c->shp.Mp;
  c->G = std::max(1, std::min(cfg->max_group, kMaxSeg));
  c->QB = c->G * cfg->max_batch;
  std::memset(&c->md, 0, sizeof(c->md));
  DevModel& md = c->md;
  md.H = cfg->H; md.W = cfg->W; md.HW = c->HW; md.Dk = c->Dk; md.Dt = cfg->text_dim;
  md.M = cfg->map_dim; md.Mp = c->Mp; md.C = cfg->num_choices; md.ksize = c->cfg.kernel_size;
  md.family = cfg->family;
  build_variables(c);
  {   // flat TF-layout buffer (weights / gradients / Adam moments) and where each gradient goes
    int64_t off = 0;
    std::memset(&c->go, 0, sizeof(c->go));
    for (const Variable& v : c->vars) {
      c->flat_offset.push_back(off);
      const int o = (int)off;
      if (v.kind == VK_PROJ_W) c->go.proj_w[v.set] = o;
      else if (v.kind == VK_PROJ_B) c->go.proj_b[v.set] = o;
      else {
        for (int i = 0; i < NUM_TEXT_SETS; ++i) {
          if (v.slot == &md.txt_w[i]) c->go.txt_w[i] = o;
          if (v.slot == &md.txt_b[i]) c->go.txt_b[i] = o;
        }
        for (int i = 0; i < NUM_ELT_SETS; ++i) {
          if (v.slot == &md.elt_w[i]) c->go.elt_w[i] = o;
          if (v.slot == &md.elt_b[i]) c->go.elt_b[i] = o;
        }
        for (int i = 0; i < NUM_OUT_SETS; ++i) {
          if (v.slot == &md.out_w[i]) c->go.out_w[i] = o;
          if (v.slot == &md.out_b[i]) c->go.out_b[i] = o;
        }
        for (int i = 0; i < NUM_SCORE_SETS; ++i) {
          if (v.slot == &md.sc_w[i]) c->go.sc_w[i] = o;
          if (v.slot == &md.sc_b[i]) c->go.sc_b[i] = o;
        }
        if (v.slot == &md.conv_k) c->go.conv_k = o;
        if (v.slot == &md.conv_b) c->go.conv_b = o;
      }
      off += (int64_t)((v.count + 3) & ~(size_t)3);
    }
    c->flat_size = off;
  }

  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  CUDA_TRY(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
  if (!fn || qres != cudaDriverEntryPointSuccess)
    return fail(N2NMN_ERR_CUDA, "cuTensorMapEncodeTiled not available from the driver");
  c->encode = reinterpret_cast<EncodeTiledFn>(fn);

  // weights: plain copies + repacked projection operands
  CUDA_TRY(cudaMalloc(&c->wbuf, c->wbuf_floats * sizeof(float)));
  CUDA_TRY(cudaMemset(c->wbuf, 0, c->wbuf_floats * sizeof(float)));
  for (Variable& v : c->vars)
    if (v.slot) *v.slot = c->wbuf + v.offset;
  for (const Variable& v : c->vars)
    if (v.kind == VK_PROJ_W) c->proj_used[v.set] = true;
  for (int s = 0; s < NUM_PROJ_SETS; ++s) {
    if (!c->proj_used[s]) continue;
    if (s != PS_FIND) ++c->num_store_sets;
    CUDA_TRY(cudaMalloc(&c->proj_wt[s], (size_t)c->Mp * c->Kp * sizeof(float)));
    CUDA_TRY(cudaMemset(c->proj_wt[s], 0, (size_t)c->Mp * c->Kp * sizeof(float)));
    CUDA_TRY(cudaMalloc(&c->proj_bias[s], (size_t)c->Mp * sizeof(float)));
    CUDA_TRY(cudaMemset(c->proj_bias[s], 0, (size_t)c->Mp * sizeof(float)));
    md.proj_b[s] = c->proj_bias[s];
    TRY(encode_2d(c, &c->tmaps.b[s], c->proj_wt[s], c->Kp, c->Mp, c->Kp, kBK, kBNHalf));
  }
  for (int s = 0; s < NUM_PROJ_SETS; ++s)      // sets the family lacks alias set 0 (never used)
    if (!c->proj_used[s]) c->tmaps.b[s] = c->tmaps.b[PS_FIND];
  // workspaces (sized for a full group of segments)
  const int NB = c->QB, TT = cfg->max_T;
  c->text_rows_cap = NB * TT;
  const size_t tb_floats = (size_t)c->text_rows_cap * c->Mp;
  CUDA_TRY(cudaMalloc(&c->tb.tau, 3 * tb_floats * sizeof(float)));
  c->tb.tauw = c->tb.tau + tb_floats;
  c->tb.tau2 = c->tb.tauw + tb_floats;
  c->arena_slots = std::max(NB * TT, 3 * NB);
  CUDA_TRY(cudaMalloc(&c->arena, (size_t)c->arena_slots * c->HW * sizeof(float)));
  c->mbuf_slots = (c->num_store_sets + 1) * NB;   // +1: conv_image maps of Find kept for backward
  CUDA_TRY(cudaMalloc(&c->mbuf, (size_t)c->mbuf_slots * c->HW * c->Mp * sizeof(float)));
  CUDA_TRY(cudaMalloc(&c->scores_tmp,
                      (size_t)cfg->max_batch * TT * cfg->num_choices * sizeof(float)));
  CUDA_TRY(cudaMalloc(&c->pooled, (size_t)2 * NB * c->Kp * sizeof(float)));
  CUDA_TRY(cudaMalloc(&c->pool_att, (size_t)2 * NB * ((c->HW + 3) & ~3) * sizeof(float)));
  if (c->cfg.family != N2NMN_VQA) {
    const int ks = c->cfg.kernel_size;
    CUDA_TRY(cudaMalloc(&c->conv_quad, (size_t)quad_pitch(ks) * c->Mp * sizeof(float)));
    CUDA_TRY(cudaMemset(c->conv_quad, 0, (size_t)quad_pitch(ks) * c->Mp * sizeof(float)));
    CUDA_TRY(cudaMalloc(&c->tb.tq, (size_t)c->text_rows_cap * quad_pitch(ks) * sizeof(float)));
    md.conv_quad = c->conv_quad;
    if (quad_pitch(ks) > 3 * c->Mp)
      return fail(N2NMN_ERR_ARG, "kernel_size too large for this map_dim");
  }
  if (2 * (c->HW + 2) * kHeadNodesMax > head_smem_floats(c->head_nn, c->Kp, c->Mp) - 8 * kHeadNodesMax * 32)
    return fail(N2NMN_ERR_ARG, "grid too large for the answer-head kernel");
  if (cfg->num_choices > 32) {
    c->Cp = round_up(cfg->num_choices, 4);
    CUDA_TRY(cudaMalloc(&c->ehat, (size_t)NB * c->Mp * sizeof(float)));
    CUDA_TRY(cudaMalloc(&c->ehat_dst, (size_t)NB * sizeof(float*)));
    c->Cpad = round_up(cfg->num_choices, kHtN);
    CUDA_TRY(cudaMalloc(&c->ehat_lo, (size_t)NB * c->Mp * sizeof(float)));
    for (const Variable& v : c->vars)
      for (int os = 0; os < NUM_OUT_SETS; ++os)
        if (v.slot == &md.out_w[os]) {
          CUDA_TRY(cudaMalloc(&c->out_wp[os], (size_t)cfg->map_dim * c->Cp * sizeof(float)));
          CUDA_TRY(cudaMemset(c->out_wp[os], 0, (size_t)cfg->map_dim * c->Cp * sizeof(float)));
          const size_t wt = (size_t)c->Cpad * c->Mp * sizeof(float);
          CUDA_TRY(cudaMalloc(&c->out_wt_hi[os], wt));
          CUDA_TRY(cudaMalloc(&c->out_wt_lo[os], wt));
          CUDA_TRY(cudaMemset(c->out_wt_hi[os], 0, wt));
          CUDA_TRY(cudaMemset(c->out_wt_lo[os], 0, wt));
          HeadTailMaps& hm = c->ht_maps[os];
          TRY(encode_2d(c, &hm.a_hi, c->ehat, c->Mp, NB, c->Mp, kHtK, kHtM));
          TRY(encode_2d(c, &hm.a_lo, c->ehat_lo, c->Mp, NB, c->Mp, kHtK, kHtM));
          TRY(encode_2d(c, &hm.b_hi, c->out_wt_hi[os], c->Mp, c->Cpad, c->Mp, kHtK, kHtN));
          TRY(encode_2d(c, &hm.b_lo, c->out_wt_lo[os], c->Mp, c->Cpad, c->Mp, kHtK, kHtN));
        }
    TRY(set_smem(head_tail_wgmma_kernel, (int)kHtSmemBytes));
  }
  c->head_nn = head_nodes_per_cta(c->Dk, c->Mp);
  c->head_smem_bytes = head_smem_layout(c->head_nn, c->Kp, c->Mp).total * (int)sizeof(float);
  if (cfg->family == N2NMN_VQA || (cfg->D % 4) != 0) {
    CUDA_TRY(cudaMalloc(&c->feat_aug, (size_t)NB * c->HW * c->Kp * sizeof(float)));
  }
  // schedule tables: generous upper bound on every table for (max_batch, max_T)
  {
    const size_t nodes = (size_t)NB * TT;
    const size_t tiles = (size_t)c->G * (((size_t)cfg->max_batch * c->HW + 127) / 128 + 1);
    c->table_cap = nodes * (sizeof(NodeRec) + 4 * 6) + (nodes / 8 + 8) * sizeof(TextGroup) +
                   tiles * (TT / kMaxProjNodesPerPass + 1 + NUM_PROJ_SETS) * sizeof(ProjWork) +
                   (size_t)NB * (12 + 4 * NUM_PROJ_SETS) + nodes * (16 + 2 * sizeof(BwdEntryHost)) +
                   (size_t)NB * (4 + 8 + sizeof(HeadWork)) + 4096;
    for (int i = 0; i < kTableSlots; ++i) {
      CUDA_TRY(cudaMallocHost(&c->slots[i].host, c->table_cap));
      CUDA_TRY(cudaMalloc(&c->slots[i].dev, c->table_cap));
      CUDA_TRY(cudaEventCreateWithFlags(&c->slots[i].last_use, cudaEventDisableTiming));
    }
  }
  // kernel attributes
  const NodeSmem L = node_smem_layout(cfg->H, cfg->W, c->Mp, c->cfg.kernel_size, cfg->map_dim,
                                      cfg->num_choices);
  c->node_smem_bytes = L.total * (int)sizeof(float);
  c->stack_cap = cfg->max_T / 2 + 2;
  for (;;) {   // largest attention stack that still fits in shared memory
    c->tree_smem_bytes = (int)sizeof(float) * tree_smem_layout(
        cfg->H, cfg->W, c->Mp, c->cfg.kernel_size, cfg->map_dim, cfg->num_choices,
        c->stack_cap).total;
    if (c->tree_smem_bytes <= 200 * 1024 || c->stack_cap <= 2) break;
    --c->stack_cap;
  }
  for (int ks : {3, 5})
    for (bool direct : {false, true}) TRY(set_smem(tree_variant(ks, direct), c->tree_smem_bytes));
  if (cfg->text_dim % 4 != 0)
    return fail(N2NMN_ERR_ARG, "text_dim must be a multiple of 4 (16-byte word-vector rows)");
  TRY(set_smem(text_proj_kernel, (int)mma_smem_bytes(4, kTextStages), 100));
  TRY(set_smem(quad_kernel, (int)mma_smem_bytes(4, kTextStages), 100));
  for (int nn : {16, 8, 4}) {
    const int bytes = head_smem_layout(nn, c->Kp, c->Mp).total * (int)sizeof(float);
    TRY(set_smem(head_variant(nn), bytes <= 200 * 1024 ? bytes : 48 * 1024));
  }
  if (c->head_smem_bytes > 200 * 1024)
    return fail(N2NMN_ERR_ARG, "feature depth too large for the answer-head kernel");
  for (int ks : {3, 5}) TRY(set_smem(wave_variant(ks), c->node_smem_bytes));
  TRY(set_smem(proj_wgmma_kernel, proj_smem_bytes()));
  TRY(set_smem(proj_simt_kernel, (int)((kSimtRows * kSimtKChunk + kSimtRows * c->Mp) * sizeof(float))));
  c->module_sched.uid = g_uid++;
  c->module_sched.shp = c->shp;
  c->step_sched.shp = c->shp;
  *out = owner.release();
  return 0;
}

int n2nmn_destroy(n2nmn_ctx* c) {
  if (!c) return 0;
  cudaSetDevice(c->device);
  cudaDeviceSynchronize();
  cudaFree(c->wbuf);
  for (int s = 0; s < NUM_PROJ_SETS; ++s) { cudaFree(c->proj_wt[s]); cudaFree(c->proj_bias[s]); }
  cudaFree(c->feat_aug); cudaFree(c->tb.tau); cudaFree(c->arena); cudaFree(c->mbuf);
  cudaFree(c->pooled); cudaFree(c->pool_att); cudaFree(c->conv_quad); cudaFree(c->tb.tq);
  cudaFree(c->dscores); cudaFree(c->per_sample); cudaFree(c->dtau); cudaFree(c->dmap); cudaFree(c->dstencil); cudaFree(c->gmap); cudaFree(c->phi_buf);
  cudaFree(c->ehat); cudaFree(c->ehat_dst); cudaFree(c->ehat_lo);
  cudaFree(c->dehat); cudaFree(c->ds_hi); cudaFree(c->ds_lo); cudaFree(c->tail_zero);
  cudaFree(c->root_set); cudaFree(c->tail_dst);
  for (int os = 0; os < NUM_OUT_SETS; ++os) {
    cudaFree(c->out_wp[os]); cudaFree(c->out_wt_hi[os]); cudaFree(c->out_wt_lo[os]);
    cudaFree(c->out_wp_lo[os]);
  }
  cudaFree(c->d_segs); cudaFree(c->d_sumsq); cudaFree(c->d_repack);
  cudaFree(c->scores_tmp); cudaFree(c->e2e_feat); cudaFree(c->e2e_wv); cudaFree(c->e2e_scores);
  cudaFree(c->e2e_feat_f16);
  for (int i = 0; i < kTableSlots; ++i) {
    cudaFreeHost(c->slots[i].host); cudaFree(c->slots[i].dev);
    if (c->slots[i].last_use) cudaEventDestroy(c->slots[i].last_use);
  }
  for (cudaEvent_t e : c->ev) cudaEventDestroy(e);
  delete c;
  return 0;
}

int n2nmn_num_variables(const n2nmn_ctx* c) { return c ? (int)c->vars.size() : 0; }

int n2nmn_variable_info(const n2nmn_ctx* c, int index, const char** name, int64_t shape[4],
                        int* ndim) {
  if (!c || index < 0 || index >= (int)c->vars.size()) return fail(N2NMN_ERR_ARG, "bad index");
  const Variable& v = c->vars[index];
  if (name) *name = v.name.c_str();
  if (ndim) *ndim = (int)v.shape.size();
  if (shape) for (size_t i = 0; i < v.shape.size() && i < 4; ++i) shape[i] = v.shape[i];
  return 0;
}

int n2nmn_set_weight(n2nmn_ctx* c, const char* name, const float* src, const int64_t* shape,
                     int ndim, void* stream) {
  if (!c || !name || !src) return fail(N2NMN_ERR_ARG, "null argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  for (Variable& v : c->vars) {
    if (v.name != name) continue;
    if (ndim != (int)v.shape.size()) return fail(N2NMN_ERR_ARG, std::string("rank mismatch for ") + name);
    for (int i = 0; i < ndim; ++i)
      if (shape[i] != v.shape[i]) return fail(N2NMN_ERR_ARG, std::string("shape mismatch for ") + name);
    if (v.kind == VK_PITCHED) {
      const int rows = (int)(v.count / (size_t)v.shape.back());
      TRY(ctx_launch(c, pitch_rows_kernel, rows, 256, 0, st, {}, src, rows, (int)v.shape.back(),
                     c->wbuf + v.offset, c->Mp));
    } else {
      CUDA_TRY(cudaMemcpyAsync(c->wbuf + v.offset, src, v.count * sizeof(float),
                               cudaMemcpyDeviceToDevice, st));
    }
    if (v.kind == VK_PROJ_W) {
      TRY(ctx_launch(c, transpose_pad_kernel, dim3((c->Kp + 31) / 32, (c->Mp + 31) / 32), dim3(32, 8),
                     0, st, {}, c->wbuf + v.offset, c->Dk, c->cfg.map_dim, c->proj_wt[v.set], c->Kp,
                     c->Mp));
    } else if (v.kind == VK_PROJ_B) {
      TRY(ctx_launch(c, pad_copy_kernel, (c->Mp + 255) / 256, 256, 0, st, {}, c->wbuf + v.offset,
                     c->cfg.map_dim, c->proj_bias[v.set], c->Mp));
    }
    for (int os = 0; os < NUM_OUT_SETS; ++os)
      if (v.slot == &c->md.out_w[os]) TRY(pack_out_weights(c, os, src, st));
    // the Transform quadratic-form matrix depends on these three variables
    if (v.slot == &c->md.conv_k || v.slot == &c->md.conv_b || v.slot == &c->md.elt_w[ES_TRANSFORM])
      TRY(update_conv_quad(c, st));
    v.loaded = true;
    return 0;
  }
  return fail(N2NMN_ERR_ARG, std::string("unknown variable: ") + name);
}

namespace {
// Points the context at `nseg` batches of identical shape (segments): feature grids [N,H,W,D],
// word vectors [T,N,Dt]. One TMA tensor map per segment; VQA / odd channel counts get their
// augmented / re-pitched copy per segment.
int bind_segments(n2nmn_ctx* c, int nseg, const float* const* feat, const float* const* wv, int N,
                  int T, cudaStream_t st) {
  if (nseg <= 0 || nseg > c->G) return fail(N2NMN_ERR_CAPACITY, "too many batches for one group");
  if (N <= 0 || T <= 0) return fail(N2NMN_ERR_ARG, "N and T must be positive");
  if (N > c->cfg.max_batch || T > c->cfg.max_T)
    return fail(N2NMN_ERR_CAPACITY, "N or T exceeds the context capacity");
  const int rows = N * c->HW;
  const int pitch = c->feat_aug ? c->Kp : c->cfg.D;
  for (int sgi = 0; sgi < nseg; ++sgi) {
    if (!feat[sgi] || !wv[sgi]) return fail(N2NMN_ERR_ARG, "null argument");
    const float* eff = feat[sgi];
    if (c->feat_aug) {
      float* dst = c->feat_aug + (size_t)sgi * c->cfg.max_batch * c->HW * c->Kp;
      TRY(ctx_launch(c, augment_features_kernel, rows, 128, 0, st, {}, feat[sgi], rows, c->cfg.D,
                     c->cfg.H, c->cfg.W, c->cfg.family == N2NMN_VQA ? 1 : 0, dst, c->Kp));
      eff = dst;
    }
    if ((reinterpret_cast<uintptr_t>(eff) & 15) != 0)
      return fail(N2NMN_ERR_ARG, "image_feat_grid must be 16-byte aligned");
    c->md.feat_seg[sgi] = eff;
    c->md.wv_seg[sgi] = wv[sgi];
    TRY(encode_2d(c, &c->tmaps.a[sgi], eff, c->Dk, rows, pitch, kBK, kBM));
  }
  for (int sgi = nseg; sgi < kMaxSeg; ++sgi) {
    c->md.feat_seg[sgi] = c->md.feat_seg[0];
    c->md.wv_seg[sgi] = c->md.wv_seg[0];
  }
  c->md.feat = c->md.feat_seg[0]; c->md.feat_pitch = pitch; c->md.word_vecs = c->md.wv_seg[0];
  c->md.N = N; c->md.T = T; c->md.num_seg = nseg;
  c->N = N; c->T = T;
  c->bound = true;
  return 0;
}
}  // namespace

int n2nmn_bind_inputs(n2nmn_ctx* c, const float* feat, const float* wv, int N, int T,
                      void* stream) {
  if (!c || !feat || !wv) return fail(N2NMN_ERR_ARG, "null argument");
  return bind_segments(c, 1, &feat, &wv, N, T, static_cast<cudaStream_t>(stream));
}

int n2nmn_compile_schedule(n2nmn_ctx* c, const int32_t* tokens, int T, int N,
                           const int32_t* vocab_ops, int num_vocab, uint8_t* validity_out,
                           n2nmn_sched** out) {
  if (!c || !tokens || !vocab_ops || !out) return fail(N2NMN_ERR_ARG, "null argument");
  if (N <= 0 || T <= 0) return fail(N2NMN_ERR_ARG, "N and T must be positive");
  if (N > c->cfg.max_batch || T > c->cfg.max_T)
    return fail(N2NMN_ERR_CAPACITY, "N or T exceeds the context capacity");
  n2nmn_sched* sc = new n2nmn_sched();
  sc->uid = g_uid++;
  sc->shp = c->shp;
  const char* err = nullptr;
  const bool direct = !(c->cfg.flags & N2NMN_FLAG_WAVE_EXECUTOR);
  const int rc = compile_schedule_group(c->shp, &tokens, 1, T, N, vocab_ops, num_vocab, &sc->hs,
                                        &err, false, direct);
  if (rc) { delete sc; return fail(rc, err ? err : "compile_schedule failed"); }
  if (validity_out) std::memcpy(validity_out, sc->hs.validity.data(), N);
  *out = sc;
  return 0;
}

int n2nmn_compile_schedule_host(const n2nmn_config* cfg, const int32_t* tokens, int T, int N,
                                const int32_t* vocab_ops, int num_vocab, uint8_t* validity_out,
                                n2nmn_sched** out) {
  if (!cfg || !tokens || !vocab_ops || !out) return fail(N2NMN_ERR_ARG, "null argument");
  if (N <= 0 || T <= 0) return fail(N2NMN_ERR_ARG, "N and T must be positive");
  const SchedShape shp = sched_shape(*cfg);
  n2nmn_sched* sc = new n2nmn_sched();
  sc->uid = g_uid++;
  sc->shp = shp;
  const char* err = nullptr;
  const int rc = compile_schedule(shp, tokens, T, N, vocab_ops, num_vocab, &sc->hs, &err);
  if (rc) { delete sc; return fail(rc, err ? err : "compile_schedule failed"); }
  if (validity_out) std::memcpy(validity_out, sc->hs.validity.data(), N);
  *out = sc;
  return 0;
}

// Diagnostic: nanoseconds per layout compile (host only), reusing one schedule object the way
// n2nmn_forward_tokens does.
double n2nmn_time_compile(const n2nmn_config* cfg, const int32_t* tokens, int T, int N,
                          const int32_t* vocab_ops, int num_vocab, int iters) {
  if (!cfg || !tokens || !vocab_ops || iters <= 0) return -1.0;
  const SchedShape shp = sched_shape(*cfg);
  HostSchedule hs;
  const char* err = nullptr;
  compile_schedule(shp, tokens, T, N, vocab_ops, num_vocab, &hs, &err);
  timespec t0, t1;
  clock_gettime(CLOCK_MONOTONIC, &t0);
  for (int i = 0; i < iters; ++i) compile_schedule(shp, tokens, T, N, vocab_ops, num_vocab, &hs, &err);
  clock_gettime(CLOCK_MONOTONIC, &t1);
  return ((t1.tv_sec - t0.tv_sec) * 1e9 + (t1.tv_nsec - t0.tv_nsec)) / iters;
}

int n2nmn_compile_nodes(n2nmn_ctx* c, const int32_t* op, const int32_t* t_idx,
                        const int32_t* b_idx, const int32_t* in0, const int32_t* in1, int n,
                        const int32_t* q_ptr, int nq, n2nmn_sched** out) {
  if (!c || !q_ptr || !out || (n > 0 && (!op || !t_idx || !b_idx || !in0 || !in1)))
    return fail(N2NMN_ERR_ARG, "null argument");
  if (nq <= 0 || nq > c->cfg.max_batch) return fail(N2NMN_ERR_CAPACITY, "bad question count");
  if (q_ptr[0] != 0 || q_ptr[nq] != n) return fail(N2NMN_ERR_ARG, "q_ptr does not span the nodes");
  n2nmn_sched* sc = new n2nmn_sched();
  sc->uid = g_uid++;
  sc->shp = c->shp;
  HostSchedule& S = sc->hs;
  S.N = c->cfg.max_batch; S.T = c->cfg.max_T;   // batch_idx may name any bound image
  S.pooled_direct = !(c->cfg.flags & N2NMN_FLAG_WAVE_EXECUTOR);
  S.nodes.resize(n); S.depth.assign(n, 1);
  S.q_ptr.assign(q_ptr, q_ptr + nq + 1);
  S.validity.assign(nq, 0);
  const int scene_bits = [] { float v = 3.0f; int b; std::memcpy(&b, &v, 4); return b; }();
  for (int q = 0; q < nq; ++q) {
    if (q_ptr[q + 1] < q_ptr[q]) { delete sc; return fail(N2NMN_ERR_ARG, "q_ptr not monotone"); }
    if (q_ptr[q + 1] > q_ptr[q]) { S.validity[q] = 1; ++S.num_valid; }
    for (int i = q_ptr[q]; i < q_ptr[q + 1]; ++i) {
      NodeRec& r = S.nodes[i];
      const int o = op[i];
      bool ok = o >= 0 && o < NUM_OPS && t_idx[i] >= 0 && t_idx[i] < c->cfg.max_T &&
                b_idx[i] >= 0 && b_idx[i] < c->cfg.max_batch;
      const int kids[2] = {in0[i], in1[i]};
      for (int k = 0; ok && k < 2; ++k) {
        if (k < kArity[o]) {
          ok = kids[k] >= q_ptr[q] && kids[k] < i && !kIsAns[op[kids[k]]];
          if (ok) S.depth[i] = std::max(S.depth[i], S.depth[kids[k]] + 1);
        } else {
          ok = kids[k] < 0;
        }
      }
      if (ok && kIsAns[o] != (i == q_ptr[q + 1] - 1)) ok = false;   // exactly the root answers
      if (!ok) { delete sc; return fail(N2NMN_ERR_ARG, "malformed expression node " + std::to_string(i)); }
      r.op = o; r.t = t_idx[i]; r.b = b_idx[i];
      r.in0 = in0[i]; r.in1 = in1[i];
      r.out = kIsAns[o] ? q : i;
      r.text = -1;
      r.aux = (o == OP_SCENE) ? scene_bits : -1;
      r.aux2 = -1; r.s0 = r.s1 = r.so = -1;
    }
  }
  if (int rc = finalize_schedule(c->shp, c->cfg.max_batch, &S)) {
    delete sc;
    return fail(rc, "finalize_schedule failed");
  }
  *out = sc;
  return 0;
}

int n2nmn_sched_destroy(n2nmn_sched* s) { delete s; return 0; }

int n2nmn_sched_get_info(const n2nmn_sched* s, n2nmn_sched_info* info) {
  if (!s || !info) return fail(N2NMN_ERR_ARG, "null argument");
  account_schedule(s->shp, const_cast<HostSchedule*>(&s->hs));
  const HostSchedule& S = s->hs;
  info->num_questions = (int)S.q_ptr.size() - 1;
  info->num_valid = S.num_valid;
  info->num_nodes = (int)S.nodes.size();
  info->max_depth = S.max_depth;
  info->num_text_nodes = (int)S.text_t.size();
  info->num_find_nodes = S.num_find_nodes;
  info->num_proj_tiles = (int)S.work.size();
  info->num_launches = (S.groups.empty() ? 0 : 1) + (S.work.empty() ? 0 : 1) + 1 +
                       (S.head_work.empty() ? 0 : 1);
  info->algorithmic_bytes = S.per_node_bytes;
  info->algorithmic_flops = S.per_node_flops;
  for (int k = 0; k < 3; ++k) { info->kernel_bytes[k] = S.kbytes[k]; info->kernel_flops[k] = S.kflops[k]; }
  info->bwd_gemm_flops = S.train ? 2ll * (int64_t)S.entries.size() * s->shp.H * s->shp.W *
                                       s->shp.Dk * s->shp.M : 0;
  return 0;
}

int n2nmn_last_step_info(const n2nmn_ctx* c, n2nmn_sched_info* info) {
  if (!c) return fail(N2NMN_ERR_ARG, "null context");
  return n2nmn_sched_get_info(&c->step_sched, info);
}

int n2nmn_sched_get_nodes(const n2nmn_sched* s, int32_t* out6, int cap) {
  if (!s || !out6) return fail(N2NMN_ERR_ARG, "null argument");
  const HostSchedule& S = s->hs;
  if (cap < (int)S.nodes.size()) return fail(N2NMN_ERR_CAPACITY, "node buffer too small");
  for (size_t i = 0; i < S.nodes.size(); ++i) {
    const NodeRec& r = S.nodes[i];
    int32_t* o = out6 + 6 * i;
    o[0] = r.op; o[1] = r.t; o[2] = r.b; o[3] = S.depth[i]; o[4] = r.in0; o[5] = r.in1;
  }
  return (int)S.nodes.size();
}

int n2nmn_run_schedule(n2nmn_ctx* c, n2nmn_sched* s, float* scores, float* att_arena,
                       void* stream) {
  if (!c || !s || !scores) return fail(N2NMN_ERR_ARG, "null argument");
  if (int rc = check_ready(c)) return rc;
  for (const NodeRec& r : s->hs.nodes)
    if (r.b >= c->N || r.t >= c->T)
      return fail(N2NMN_ERR_ARG, "schedule refers to a batch/time index outside the bound inputs");
  if ((int)s->hs.img_ptr.size() - 1 > c->N && s->hs.img_ptr.back() != s->hs.img_ptr[c->N])
    return fail(N2NMN_ERR_ARG, "schedule image range exceeds the bound inputs");
  float* arena = att_arena ? att_arena : c->arena;
  if (!att_arena && (int)s->hs.nodes.size() > c->arena_slots)
    return fail(N2NMN_ERR_CAPACITY, "too many nodes for the context arena");
  if (s->hs.num_seg != 1 || c->md.num_seg != 1)
    return fail(N2NMN_ERR_STATE, "n2nmn_run_schedule works on a single bound batch");
  return run_tables(c, s, &scores, arena, static_cast<cudaStream_t>(stream), false,
                    att_arena != nullptr);
}

namespace {
int module_fwd_impl(n2nmn_ctx* c, int op, const float* in0, const float* in1,
                    const int32_t* t_idx, const int32_t* b_idx, int n, float* out, void* stream,
                    float scene_val);
}

int n2nmn_module_fwd(n2nmn_ctx* c, int op, const float* in0, const float* in1,
                     const int32_t* t_idx, const int32_t* b_idx, int n, float* out,
                     void* stream) {
  return module_fwd_impl(c, op, in0, in1, t_idx, b_idx, n, out, stream, 3.0f);
}

int n2nmn_scene_fwd(n2nmn_ctx* c, int n, float pos_val, float* out, void* stream) {
  return module_fwd_impl(c, OP_SCENE, nullptr, nullptr, nullptr, nullptr, n, out, stream, pos_val);
}

namespace {
int module_fwd_impl(n2nmn_ctx* c, int op, const float* in0, const float* in1,
                    const int32_t* t_idx, const int32_t* b_idx, int n, float* out, void* stream,
                    float scene_val) {
  if (!c) return fail(N2NMN_ERR_ARG, "null context");
  if (op < 0 || op >= NUM_OPS) return fail(N2NMN_ERR_ARG, "bad opcode");
  if (n == 0) return 0;   // TF Fold's zero-size batches: nothing to do
  if (n < 0 || !out) return fail(N2NMN_ERR_ARG, "bad arguments");
  if (int rc = check_ready(c)) return rc;
  static const bool needs_idx[NUM_OPS] = {0, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0, 1, 1};
  if ((kArity[op] >= 1 && !in0) || (kArity[op] >= 2 && !in1))
    return fail(N2NMN_ERR_ARG, "missing attention input");
  if (needs_idx[op] && (!t_idx || !b_idx))
    return fail(N2NMN_ERR_ARG, "time_idx / batch_idx required for this module");
  if (3 * n > c->arena_slots || n > c->cfg.max_batch * c->cfg.max_T)
    return fail(N2NMN_ERR_CAPACITY, "n exceeds the context capacity for a single module call");
  if (c->md.num_seg != 1) return fail(N2NMN_ERR_STATE, "module calls need a single bound batch");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  n2nmn_sched* sc = &c->module_sched;
  sc->uid = g_uid++;   // tables change every call
  HostSchedule& S = sc->hs;
  S.reset();
  S.N = c->N; S.T = c->T;
  S.nodes.resize(n); S.depth.assign(n, 1); S.q_ptr.resize(n + 1);
  int scene_bits;
  std::memcpy(&scene_bits, &scene_val, 4);
  for (int i = 0; i < n; ++i) {
    NodeRec& r = S.nodes[i];
    r.op = op;
    r.t = t_idx ? t_idx[i] : 0;
    r.b = b_idx ? b_idx[i] : 0;
    if (needs_idx[op] && (r.b < 0 || r.b >= c->N || r.t < 0 || r.t >= c->T))
      return fail(N2NMN_ERR_ARG, "time_idx / batch_idx out of range");
    if (!needs_idx[op]) { r.t = 0; r.b = 0; }
    r.in0 = kArity[op] >= 1 ? i : -1;
    r.in1 = kArity[op] >= 2 ? n + i : -1;
    r.out = kIsAns[op] ? i : 2 * n + i;
    r.text = -1;
    r.aux = (op == OP_SCENE) ? scene_bits : -1;
    r.aux2 = -1; r.s0 = r.s1 = r.so = -1;
    S.q_ptr[i] = i;
  }
  S.q_ptr[n] = n;
  if (int rc = finalize_schedule(c->shp, c->N, &S)) return fail(rc, "finalize_schedule failed");
  const size_t map_bytes = (size_t)n * c->HW * sizeof(float);
  if (kArity[op] >= 1)
    CUDA_TRY(cudaMemcpyAsync(c->arena, in0, map_bytes, cudaMemcpyDeviceToDevice, st));
  if (kArity[op] >= 2)
    CUDA_TRY(cudaMemcpyAsync(c->arena + (size_t)n * c->HW, in1, map_bytes,
                             cudaMemcpyDeviceToDevice, st));
  float* scores = kIsAns[op] ? out : c->scores_tmp;
  if (int rc = run_tables(c, sc, &scores, c->arena, st, /*force_wave=*/true)) return rc;
  if (!kIsAns[op])
    CUDA_TRY(cudaMemcpyAsync(out, c->arena + (size_t)2 * n * c->HW, map_bytes,
                             cudaMemcpyDeviceToDevice, st));
  return 0;
}
}  // namespace

int n2nmn_forward_group(n2nmn_ctx* c, int num_batches, const float* const* feat_dev,
                        const float* const* wv_dev, const int32_t* const* tokens, int T, int N,
                        const int32_t* vocab_ops, int num_vocab, float* const* scores_dev,
                        uint8_t* const* validity_out, void* stream) {
  if (!c || !feat_dev || !wv_dev || !tokens || !vocab_ops || !scores_dev || num_batches <= 0)
    return fail(N2NMN_ERR_ARG, "null argument");
  for (int i = 0; i < num_batches; ++i)
    if (!tokens[i] || !scores_dev[i]) return fail(N2NMN_ERR_ARG, "null argument");
  CUDA_TRY(cudaSetDevice(c->device));   // callers may drive one context per host thread
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int rc = bind_segments(c, num_batches, feat_dev, wv_dev, N, T, st)) return rc;
  if (int rc = check_ready(c)) return rc;
  n2nmn_sched* sc = &c->step_sched;
  sc->uid = g_uid++;
  const char* err = nullptr;
  const bool direct = !(c->cfg.flags & N2NMN_FLAG_WAVE_EXECUTOR);
  if (int rc = compile_schedule_group(c->shp, tokens, num_batches, T, N, vocab_ops, num_vocab,
                                      &sc->hs, &err, false, direct))
    return fail(rc, err ? err : "compile_schedule failed");
  if (validity_out)
    for (int i = 0; i < num_batches; ++i)
      if (validity_out[i]) std::memcpy(validity_out[i], sc->hs.validity.data() + (size_t)i * N, N);
  if ((int)sc->hs.nodes.size() > c->arena_slots)
    return fail(N2NMN_ERR_CAPACITY, "too many nodes for the context arena");
  return run_tables(c, sc, scores_dev, c->arena, st);
}

int n2nmn_forward_tokens(n2nmn_ctx* c, const float* feat_dev, const float* wv_dev,
                         const int32_t* tokens, int T, int N, const int32_t* vocab_ops,
                         int num_vocab, float* scores_dev, uint8_t* validity_out, void* stream) {
  if (!c || !tokens || !vocab_ops || !scores_dev) return fail(N2NMN_ERR_ARG, "null argument");
  return n2nmn_forward_group(c, 1, &feat_dev, &wv_dev, &tokens, T, N, vocab_ops, num_vocab,
                             &scores_dev, validity_out ? &validity_out : nullptr, stream);
}

namespace {
// Host-buffer variant of n2nmn_forward_group: H2D of every batch's features and word vectors into
// context-owned staging, the kernels, D2H of every batch's scores — all enqueued on `stream`.
int forward_host_impl(n2nmn_ctx* c, int nb, const void* const* feat_host,
                      const float* const* wv_host, const int32_t* const* tokens, int T, int N,
                      const int32_t* vocab_ops, int num_vocab, float* const* scores_host,
                      uint8_t* const* validity_out, void* stream, bool sync, bool feat_f16 = false) {
  if (!c || !feat_host || !wv_host || !tokens || !scores_host || nb <= 0)
    return fail(N2NMN_ERR_ARG, "null argument");
  if (nb > c->G) return fail(N2NMN_ERR_CAPACITY, "too many batches for one group");
  if (N <= 0 || N > c->cfg.max_batch || T <= 0 || T > c->cfg.max_T)
    return fail(N2NMN_ERR_CAPACITY, "N or T exceeds the context capacity");
  CUDA_TRY(cudaSetDevice(c->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t fcap = (size_t)c->cfg.max_batch * c->HW * c->cfg.D;
  const size_t wcap = (size_t)c->cfg.max_T * c->cfg.max_batch * c->cfg.text_dim;
  const size_t scap = (size_t)c->cfg.max_batch * c->cfg.num_choices;
  const size_t fbytes = (size_t)N * c->HW * c->cfg.D * sizeof(float);
  const size_t wbytes = (size_t)T * N * c->cfg.text_dim * sizeof(float);
  const size_t sbytes = (size_t)N * c->cfg.num_choices * sizeof(float);
  CUDA_TRY(alloc_once(&c->e2e_feat, c->G * fcap * sizeof(float)));
  CUDA_TRY(alloc_once(&c->e2e_wv, c->G * wcap * sizeof(float)));
  CUDA_TRY(alloc_once(&c->e2e_scores, c->G * scap * sizeof(float)));
  if (feat_f16 && (fbytes / sizeof(float)) % 8 != 0)
    return fail(N2NMN_ERR_ARG, "fp16 host features need N*H*W*D to be a multiple of 8");
  const size_t fcap16 = (fcap + 7) & ~(size_t)7;   // fp16 staging slots stay 16-byte aligned
  if (feat_f16) CUDA_TRY(alloc_once(&c->e2e_feat_f16, c->G * fcap16 * sizeof(uint16_t)));
  const float* fd[kMaxSeg];
  const float* wd[kMaxSeg];
  float* sd[kMaxSeg];
  for (int i = 0; i < nb; ++i) {
    if (!feat_host[i] || !wv_host[i] || !scores_host[i]) return fail(N2NMN_ERR_ARG, "null argument");
    fd[i] = c->e2e_feat + i * fcap; wd[i] = c->e2e_wv + i * wcap; sd[i] = c->e2e_scores + i * scap;
    if (feat_f16)
      CUDA_TRY(cudaMemcpyAsync(c->e2e_feat_f16 + i * fcap16, feat_host[i], fbytes / 2,
                               cudaMemcpyHostToDevice, st));
    else
      CUDA_TRY(cudaMemcpyAsync(c->e2e_feat + i * fcap, feat_host[i], fbytes, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(c->e2e_wv + i * wcap, wv_host[i], wbytes, cudaMemcpyHostToDevice, st));
  }
  if (feat_f16) {   // widen every staged grid to the fp32 layout the kernels read
    const size_t cnt = fbytes / sizeof(float);
    for (int i = 0; i < nb; ++i) {
      const size_t n8 = (cnt + 7) / 8;
      TRY(ctx_launch(c, widen_f16_kernel, (unsigned)std::min<size_t>((n8 + 255) / 256, (size_t)c->num_sms * 8),
                     256, 0, st, {}, reinterpret_cast<const uint4*>(c->e2e_feat_f16 + i * fcap16),
                     reinterpret_cast<float4*>(c->e2e_feat + i * fcap), n8));
    }
  }
  int rc = n2nmn_forward_group(c, nb, fd, wd, tokens, T, N, vocab_ops, num_vocab, sd, validity_out,
                               stream);
  if (rc == 0) {
    cudaError_t e = cudaSuccess;
    for (int i = 0; i < nb && e == cudaSuccess; ++i)
      e = cudaMemcpyAsync(scores_host[i], sd[i], sbytes, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess && sync) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) rc = fail(N2NMN_ERR_CUDA, cudaGetErrorString(e));
  } else if (sync) {
    cudaStreamSynchronize(st);
  }
  return rc;
}
}  // namespace

int n2nmn_forward_host(n2nmn_ctx* c, const float* feat_host, const float* wv_host,
                       const int32_t* tokens, int T, int N, const int32_t* vocab_ops,
                       int num_vocab, float* scores_host, uint8_t* validity_out, void* stream) {
  return forward_host_impl(c, 1, reinterpret_cast<const void* const*>(&feat_host), &wv_host, &tokens, T, N, vocab_ops, num_vocab,
                           &scores_host, validity_out ? &validity_out : nullptr, stream, true);
}

int n2nmn_forward_host_async(n2nmn_ctx* c, const float* feat_host, const float* wv_host,
                             const int32_t* tokens, int T, int N, const int32_t* vocab_ops,
                             int num_vocab, float* scores_host, uint8_t* validity_out,
                             void* stream) {
  return forward_host_impl(c, 1, reinterpret_cast<const void* const*>(&feat_host), &wv_host, &tokens, T, N, vocab_ops, num_vocab,
                           &scores_host, validity_out ? &validity_out : nullptr, stream, false);
}

int n2nmn_forward_group_host_async(n2nmn_ctx* c, int num_batches, const float* const* feat_host,
                                   const float* const* wv_host, const int32_t* const* tokens,
                                   int T, int N, const int32_t* vocab_ops, int num_vocab,
                                   float* const* scores_host, uint8_t* const* validity_out,
                                   void* stream) {
  return forward_host_impl(c, num_batches, reinterpret_cast<const void* const*>(feat_host), wv_host,
                           tokens, T, N, vocab_ops, num_vocab, scores_host, validity_out, stream,
                           false);
}

int n2nmn_forward_group_host_f16_async(n2nmn_ctx* c, int num_batches,
                                       const uint16_t* const* feat_host_f16,
                                       const float* const* wv_host, const int32_t* const* tokens,
                                       int T, int N, const int32_t* vocab_ops, int num_vocab,
                                       float* const* scores_host, uint8_t* const* validity_out,
                                       void* stream) {
  return forward_host_impl(c, num_batches, reinterpret_cast<const void* const*>(feat_host_f16),
                           wv_host, tokens, T, N, vocab_ops, num_vocab, scores_host, validity_out,
                           stream, false, true);
}

int n2nmn_max_group(const n2nmn_ctx* c) { return c ? c->G : 0; }


int64_t n2nmn_flat_size(const n2nmn_ctx* c) { return c ? c->flat_size : 0; }

int n2nmn_flat_offset(const n2nmn_ctx* c, int index, int64_t* offset, int64_t* count) {
  if (!c || index < 0 || index >= (int)c->vars.size()) return fail(N2NMN_ERR_ARG, "bad index");
  if (offset) *offset = c->flat_offset[index];
  if (count) *count = (int64_t)c->vars[index].count;
  return 0;
}

namespace {
int ensure_repack_tables(n2nmn_ctx* c) {
  const int nv = (int)c->vars.size();
  if (!c->repack_ready) {   // what n2nmn_set_weight does per variable, as device tables
    std::vector<RepackSeg> segs(nv);
    ProjRepack& pr = c->proj_repack;
    for (int s = 0; s < NUM_PROJ_SETS; ++s) { pr.w_off[s] = pr.b_off[s] = -1; pr.wt[s] = pr.bias[s] = nullptr; }
    c->proj_repack_sets = 0;
    for (int i = 0; i < nv; ++i) {
      const Variable& v = c->vars[i];
      segs[i].src_off = (int)c->flat_offset[i];
      segs[i].count = (int)v.count;
      segs[i].cols = (int)v.shape.back();
      segs[i].kind = v.kind == VK_PITCHED ? 1 : 0;
      segs[i].dst_off = (long long)v.offset;
      if (v.kind == VK_PROJ_W) {
        pr.w_off[v.set] = (int)c->flat_offset[i];
        pr.wt[v.set] = c->proj_wt[v.set];
        pr.bias[v.set] = c->proj_bias[v.set];
        pr.set_of_z[c->proj_repack_sets++] = v.set;
      } else if (v.kind == VK_PROJ_B) {
        pr.b_off[v.set] = (int)c->flat_offset[i];
      }
    }
    CUDA_TRY(alloc_once(&c->d_repack, nv * sizeof(RepackSeg)));
    CUDA_TRY(cudaMemcpy(c->d_repack, segs.data(), nv * sizeof(RepackSeg), cudaMemcpyHostToDevice));
    c->repack_ready = true;
  }
  return 0;
}

// the derived copies: K-major padded projection weights / biases and the Transform quadratic form
int repack_derived(n2nmn_ctx* c, const float* wflat_dev, cudaStream_t st) {
  for (size_t i = 0; i < c->vars.size(); ++i)
    for (int os = 0; os < NUM_OUT_SETS; ++os)
      if (c->vars[i].slot == &c->md.out_w[os]) TRY(pack_out_weights(c, os, wflat_dev + c->flat_offset[i], st));
  if (c->proj_repack_sets > 0)
    TRY(ctx_launch(c, proj_repack_kernel,
                   dim3((c->Kp + 31) / 32, (c->Mp + 31) / 32, c->proj_repack_sets), dim3(32, 8), 0, st,
                   {}, wflat_dev, c->proj_repack, c->Dk, c->cfg.map_dim, c->Kp, c->Mp));
  TRY(update_conv_quad(c, st));
  for (Variable& v : c->vars) v.loaded = true;
  return 0;
}
}  // namespace

int n2nmn_load_flat_weights(n2nmn_ctx* c, const float* wflat_dev, void* stream) {
  if (!c || !wflat_dev) return fail(N2NMN_ERR_ARG, "null argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  TRY(ensure_repack_tables(c));
  TRY(ctx_launch(c, repack_all_kernel, dim3(16, (unsigned)c->vars.size()), 256, 0, st, {}, wflat_dev,
                 c->d_repack, c->wbuf, c->Mp));
  return repack_derived(c, wflat_dev, st);
}

int n2nmn_train_backward(n2nmn_ctx* c, const float* feat_dev, const float* wv_dev,
                         const int32_t* tokens, int T, int N, const int32_t* vocab_ops,
                         int num_vocab, const int32_t* labels_host, float invalid_expr_loss,
                         float* scores_dev, float* gflat_dev, float* dword_dev, float* loss_dev,
                         uint8_t* validity_out, void* stream) {
  return n2nmn_train_backward_ex(c, feat_dev, wv_dev, tokens, T, N, vocab_ops, num_vocab,
                                 labels_host, invalid_expr_loss, scores_dev, gflat_dev, dword_dev,
                                 loss_dev, validity_out, nullptr, nullptr, stream);
}

namespace {
// Training workspaces and kernel attributes, set up on the first backward pass.
int ensure_train_workspace(n2nmn_ctx* c) {
  if (c->train_ready) return 0;
  const bool vqa = c->cfg.family == N2NMN_VQA;
  const int NB = c->cfg.max_batch, C = c->cfg.num_choices;
  CUDA_TRY(alloc_once(&c->dscores, (size_t)NB * C * sizeof(float)));
  CUDA_TRY(alloc_once(&c->per_sample, (size_t)NB * sizeof(float)));
  CUDA_TRY(alloc_once(&c->dtau, (size_t)c->text_rows_cap * c->Mp * sizeof(float)));
  c->dmap_entries = NB * c->cfg.max_T;
  CUDA_TRY(alloc_once(&c->dmap, (size_t)c->dmap_entries * c->HW * c->Mp * sizeof(float)));
  if (!vqa)   // d(conv output) scratch of the conv Transform
    CUDA_TRY(alloc_once(&c->dstencil, (size_t)c->dmap_entries * c->HW * c->Mp * sizeof(float)));
  CUDA_TRY(alloc_once(&c->gmap, (size_t)c->arena_slots * ((c->HW + 3) & ~3) * sizeof(float)));
  CUDA_TRY(alloc_once(&c->phi_buf, (size_t)NB * 2 * c->Mp * sizeof(float)));
  c->wg_ok = c->Mp % kWgN == 0 && c->Dk >= kWgM;
  if (c->wg_ok) TRY(set_smem(wgrad_wgmma_kernel, (int)kWgSmemBytes));
  if (c->ehat) {   // many-class heads: the batched tail backward
    const int zeros = std::max(c->Cp, c->Mp);
    CUDA_TRY(alloc_once(&c->dehat, (size_t)NB * c->Mp * sizeof(float)));
    CUDA_TRY(alloc_once(&c->ds_hi, (size_t)NB * c->Cp * sizeof(float)));
    CUDA_TRY(alloc_once(&c->ds_lo, (size_t)NB * c->Cp * sizeof(float)));
    CUDA_TRY(alloc_once(&c->tail_zero, (size_t)zeros * sizeof(float)));
    CUDA_TRY(cudaMemset(c->tail_zero, 0, (size_t)zeros * sizeof(float)));
    CUDA_TRY(alloc_once(&c->root_set, (size_t)NB * sizeof(int32_t)));
    CUDA_TRY(alloc_once(&c->tail_dst, (size_t)NUM_OUT_SETS * NB * sizeof(float*)));
    for (int os = 0; os < NUM_OUT_SETS; ++os) {
      if (!c->out_wp[os]) continue;
      const int M = c->cfg.map_dim;
      CUDA_TRY(alloc_once(&c->out_wp_lo[os], (size_t)M * c->Cp * sizeof(float)));
      HeadTailMaps& tm = c->tail_maps[os];
      TRY(encode_2d(c, &tm.a_hi, c->ds_hi, c->Cp, NB, c->Cp, kHtK, kHtM));
      TRY(encode_2d(c, &tm.a_lo, c->ds_lo, c->Cp, NB, c->Cp, kHtK, kHtM));
      TRY(encode_2d(c, &tm.b_hi, c->out_wp[os], c->Cp, M, c->Cp, kHtK, kHtN));
      TRY(encode_2d(c, &tm.b_lo, c->out_wp_lo[os], c->Cp, M, c->Cp, kHtK, kHtN));
    }
  }
  const int ks = vqa ? 1 : c->cfg.kernel_size;
  const int bwd_smem = (int)(bwd_smem_layout(c->cfg.H, c->cfg.W, c->Mp, ks, C).total * sizeof(float));
  if (vqa) {
    for (bool wide : {false, true}) TRY(set_smem(bwd_variant(true, false, 1, wide), bwd_smem, 100));
  } else {   // the Transform instantiations keep the default carveout
    for (int k : {3, 5})
      for (bool tr : {false, true}) TRY(set_smem(bwd_variant(false, tr, k, false), bwd_smem, tr ? -1 : 100));
  }
  TRY(set_smem(xtb_mma_kernel<FeatGradSrc>, (int)kXtbSmemBytes));
  TRY(set_smem(xtb_mma_kernel<TextGradSrc>, (int)kXtbSmemBytes));
  TRY(set_smem(xtb_mma_kernel<TailGradSrc>, (int)kXtbSmemBytes));
  TRY(set_smem(text_xgrad_mma_kernel, (int)kXgSmemBytes));
  c->train_ready = true;
  return 0;
}

// Many-class heads: dê of every Describe-type root and the fc_eltwise gradients, batched.
int bwd_answer_tail(n2nmn_ctx* c, const BwdCtx& bc, const DevTables& t, int N, float* gflat,
                    cudaStream_t st) {
  const int NB = c->cfg.max_batch, M = c->cfg.map_dim, C = c->cfg.num_choices;
  TRY(ctx_launch(c, tail_prep_kernel, N, 256, 0, st, {}, bc, t.at<NodeRec>(t.o.nodes), t.at(t.o.q_ptr),
                 c->Cp, NB, c->root_set, c->ehat, c->ds_hi, c->ds_lo, c->dehat, c->tail_dst));
  prof_mark(c, "tail_prep_kernel", st);
  TailGradSrc ts;
  ts.md = c->md; ts.ehat = c->ehat; ts.ds = c->ds_hi; ts.root_set = c->root_set;
  ts.zero_row = c->tail_zero; ts.nq = N; ts.Cp = c->Cp; ts.gflat = gflat; ts.go = c->go;
  for (int os = 0; os < NUM_OUT_SETS; ++os) {
    ts.has_set[os] = c->out_wp[os] != nullptr;
    if (!c->out_wp[os]) continue;
    const size_t n = (size_t)M * c->Cp;
    TRY(ctx_launch(c, tf32_lo_kernel, (unsigned)std::min<size_t>((n + 255) / 256, 4 * (size_t)c->num_sms),
                   256, 0, st, {}, c->out_wp[os], c->out_wp_lo[os], n));
    // dÊ[q, :] = dS[q, :]·W_outᵀ for the questions whose root uses this set (3xTF32)
    TRY(ctx_launch(c, head_tail_wgmma_kernel,
                   dim3((unsigned)((M + kHtN - 1) / kHtN), (unsigned)((N + kHtM - 1) / kHtM)), kHtThreads,
                   kHtSmemBytes, st, {}, c->tail_maps[os], c->tail_zero, c->tail_dst + (size_t)os * NB,
                   0, N, M, C));
  }
  prof_mark(c, "tail_dehat_kernel", st);
  // d(W_out) = Êᵀ·dS and d(b_out) = Σ_q dS, one segment per weight set
  TRY(ctx_launch(c, xtb_mma_kernel<TailGradSrc>,
                 dim3((M + kXtbM - 1) / kXtbM, (C + kXtbN - 1) / kXtbN, NUM_OUT_SETS), kXtbThreads,
                 kXtbSmemBytes, st, {}, ts, 1));
  prof_mark(c, "tail_wgrad_kernel", st);
  return 0;
}

// The reverse tree walk, one launch per level, top down.
int bwd_walk(n2nmn_ctx* c, const BwdCtx& bc, const HostSchedule& S, const DevTables& t,
             cudaStream_t st) {
  const bool vqa = c->cfg.family == N2NMN_VQA;
  const BwdSmem L = bwd_smem_layout(c->cfg.H, c->cfg.W, c->Mp, vqa ? 1 : c->cfg.kernel_size,
                                    c->cfg.num_choices);
  CUDA_TRY(cudaMemsetAsync(c->gmap, 0, S.nodes.size() * (size_t)L.HWp * sizeof(float), st));
  CUDA_TRY(cudaMemsetAsync(c->dtau, 0, S.text_t.size() * (size_t)c->Mp * sizeof(float), st));
  // a level's nodes are listed [Transform nodes | others]; a level with Transform nodes runs the
  // full instantiation over all of them (one CTA per SM), a level without the lighter one
  for (int dd = S.max_depth; dd >= 1; --dd) {
    const int first = S.bwd_ptr[2 * dd], cnt = S.bwd_ptr[2 * dd + 2] - first;
    if (cnt <= 0) continue;
    const int n_tr = S.bwd_ptr[2 * dd + 1] - S.bwd_ptr[2 * dd];
    // CTAs per splittable node: as many as keep the level's heavy CTAs within one wave of the
    // SMs (one CTA per SM with Transform nodes, two without)
    const int slices = n_tr > 0 ? std::max(3, std::min(kBwdSlicesMax, c->num_sms / n_tr))
                                : std::max(2, std::min(6, 2 * c->num_sms / cnt));
    TRY(ctx_launch(c, bwd_variant(vqa, n_tr > 0, c->cfg.kernel_size, c->Mp > 512), dim3(cnt, slices),
                   kNodeThreads, L.total * sizeof(float), st, {true}, bc,
                   t.at<NodeRec>(t.o.nodes), t.at(t.o.bwd_nodes), first, t.at(t.o.node_entry)));
  }
  prof_mark(c, "tree_bwd_kernel", st);
  return 0;
}

// Text layers: weight gradients and, when asked for, d(word vectors).
int bwd_text(n2nmn_ctx* c, const HostSchedule& S, const DevTables& t, float* gflat, float* dword,
             cudaStream_t st) {
  const int rows = (int)S.text_t.size();
  if (rows == 0) return 0;
  const int32_t *d_tt = t.at(t.o.text_t), *d_tb = t.at(t.o.text_b), *d_ss = t.at(t.o.text_set_start);
  const int Dt = c->cfg.text_dim;
  const bool exact = (c->cfg.flags & N2NMN_FLAG_PROJ_FP32_SIMT) != 0;
  if (exact)
    TRY(ctx_launch(c, text_wgrad_kernel, dim3((Dt + 7) / 8, NUM_TEXT_SETS), 256, 0, st, {}, c->md,
                   c->dtau, d_tt, d_tb, d_ss, gflat, c->go));
  else
    TRY(ctx_launch(c, xtb_mma_kernel<TextGradSrc>,
                   dim3((Dt + kXtbM - 1) / kXtbM, (c->cfg.map_dim + kXtbN - 1) / kXtbN, NUM_TEXT_SETS),
                   kXtbThreads, kXtbSmemBytes, st, {},
                   TextGradSrc{c->md, c->dtau, d_tt, d_tb, d_ss, gflat, c->go}, 1));
  if (dword) {
    if (exact) {
      TRY(ctx_launch(c, text_xgrad_kernel, rows, 256, c->Mp * sizeof(float), st, {}, c->md, c->dtau,
                     d_tt, d_tb, d_ss, dword, c->dword_scale));
    } else {
      TextSetRows tsr;
      int groups = 0;
      for (int i = 0; i <= NUM_TEXT_SETS; ++i) tsr.start[i] = S.text_set_start[i];
      for (int i = 0; i < NUM_TEXT_SETS; ++i) groups += (tsr.start[i + 1] - tsr.start[i] + 63) / 64;
      TRY(ctx_launch(c, text_xgrad_mma_kernel, dim3((Dt + 63) / 64, groups), kXgThreads, kXgSmemBytes,
                     st, {}, c->md, c->dtau, d_tt, d_tb, tsr, dword, c->dword_scale));
    }
  }
  prof_mark(c, "text_grad_kernels", st);
  return 0;
}

// Feature-side layers: dW_set = Σ X^T·B, on CUDA cores (exact), wgmma or mma.sync.
int bwd_features(n2nmn_ctx* c, const HostSchedule& S, const DevTables& t, float* gflat,
                 cudaStream_t st) {
  const int ne = (int)S.entries.size();
  if (ne == 0) return 0;
  const BwdEntry* d_ent = t.at<BwdEntry>(t.o.entries);
  const int M = c->cfg.map_dim;
  const bool exact = (c->cfg.flags & N2NMN_FLAG_PROJ_FP32_SIMT) != 0;
  const bool wgmma = !exact && c->wg_ok && !std::getenv("N2NMN_WGRAD_MMA_SYNC");
  if (exact) {
    const int chunks = std::min(ne, 16);
    const int per = (ne + chunks - 1) / chunks;
    TRY(ctx_launch(c, feat_grad_kernel,
                   dim3((c->Dk + kFgTile - 1) / kFgTile, (M + kFgTile - 1) / kFgTile, (ne + per - 1) / per),
                   256, 0, st, {}, c->md, c->dmap, d_ent, ne, per, gflat, c->go));
  } else if (wgmma) {
    // both operands staged transposed (K-major) from the feature grid and the B maps
    const int slabs = (c->Dk + kWgM - 1) / kWgM, ntiles = c->Mp / kWgN, tiles = slabs * ntiles;
    int chunks = std::max(1, std::min(ne, c->num_sms / tiles));
    if (chunks < 4) {   // few entry chunks per tile: pick the count that wastes the least of the waves
      double best = 1e30;
      for (int k = 1; k <= std::min(ne, 8); ++k) {
        const double cost = (double)((tiles * k + c->num_sms - 1) / c->num_sms) / k;
        if (cost < best - 1e-9) { best = cost; chunks = k; }
      }
    }
    WgradParams wp;
    wp.feat = c->md.feat; wp.dmap = c->dmap; wp.entries = d_ent;
    wp.order = t.at(t.o.entry_order);
    wp.num_entries = ne; wp.per_cta = (ne + chunks - 1) / chunks;
    wp.HW = c->HW; wp.Dk = c->Dk; wp.M = M; wp.Mp = c->Mp;
    wp.pitch = c->md.feat_pitch; wp.gflat = gflat; wp.go = c->go;
    TRY(ctx_launch(c, wgrad_wgmma_kernel, dim3(slabs, (ne + wp.per_cta - 1) / wp.per_cta, ntiles),
                   kWgThreads, kWgSmemBytes, st, {}, wp));
  } else {
    // two CTAs per SM (106 KB of ring each): ~2 x SMs CTAs over (Dk/128) x (M/64) tiles
    const int tiles = ((c->Dk + kXtbM - 1) / kXtbM) * ((M + kXtbN - 1) / kXtbN);
    const int chunks = std::max(1, std::min(ne, (2 * c->num_sms + tiles - 1) / tiles));
    const int per = (ne + chunks - 1) / chunks;
    TRY(ctx_launch(c, xtb_mma_kernel<FeatGradSrc>,
                   dim3((c->Dk + kXtbM - 1) / kXtbM, (M + kXtbN - 1) / kXtbN, (ne + per - 1) / per),
                   kXtbThreads, kXtbSmemBytes, st, {},
                   FeatGradSrc{c->md, c->dmap, d_ent, ne, gflat, c->go}, per));
  }
  prof_mark(c, "feat_grad_kernel", st);
  if (wgmma) {   // the wgmma kernel leaves the bias gradients to a column sum of the B maps
    TRY(ctx_launch(c, bmap_colsum_kernel, ne, 1024, 0, st, {}, c->dmap, d_ent, c->HW, M, c->Mp, gflat,
                   c->go));
    prof_mark(c, "bias_grad_kernel", st);
  }
  return 0;
}
}  // namespace

int n2nmn_train_backward_ex(n2nmn_ctx* c, const float* feat_dev, const float* wv_dev,
                            const int32_t* tokens, int T, int N, const int32_t* vocab_ops,
                            int num_vocab, const int32_t* labels_host, float invalid_expr_loss,
                            float* scores_dev, float* gflat_dev, float* dword_dev, float* loss_dev,
                            uint8_t* validity_out, const float* score_prior_dev, float* dscores_dev,
                            void* stream) {
  if (!c || !tokens || !vocab_ops || !labels_host || !scores_dev || !gflat_dev || !loss_dev)
    return fail(N2NMN_ERR_ARG, "null argument");
  if (c->cfg.flags & N2NMN_FLAG_WAVE_EXECUTOR)
    return fail(N2NMN_ERR_ARG, "training uses the tree executor");
  // The conv-Transform backward (3x3 / 5x5 filter bank, channels in registers) covers Mp <= 512;
  // the VQA family has no conv Transform and runs the wide Find-type walk at any map_dim.
  const bool vqa = c->cfg.family == N2NMN_VQA;
  if (!vqa && c->Mp > 512)
    return fail(N2NMN_ERR_ARG,
                "n2nmn_train_backward: map_dim > 512 is not supported for the conv-Transform families");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  TRY(n2nmn_bind_inputs(c, feat_dev, wv_dev, N, T, stream));
  TRY(check_ready(c));
  const int C = c->cfg.num_choices;
  TRY(ensure_train_workspace(c));
  n2nmn_sched* sc = &c->step_sched;
  sc->uid = g_uid++;
  const char* err = nullptr;
  if (int rc = compile_schedule(c->shp, tokens, T, N, vocab_ops, num_vocab, &sc->hs, &err, true))
    return fail(rc, err ? err : "compile_schedule failed");
  build_bwd_order(&sc->hs);
  const HostSchedule& S = sc->hs;
  if (validity_out) std::memcpy(validity_out, S.validity.data(), N);
  if ((int)S.nodes.size() > c->arena_slots || (int)S.entries.size() > c->dmap_entries ||
      (int)S.nodes.size() > c->dmap_entries)
    return fail(N2NMN_ERR_CAPACITY, "too many nodes for the context");
  if (S.max_stack > c->stack_cap)
    return fail(N2NMN_ERR_CAPACITY, "layout too deep for the training path");
  for (int i = 0; i < N; ++i)
    if (labels_host[i] < 0 || labels_host[i] >= C) return fail(N2NMN_ERR_ARG, "label out of range");
  // ---- forward (keeps every attention map in the context arena + the stored maps)
  c->train_labels = labels_host;
  const int rc = run_tables(c, sc, &scores_dev, c->arena, st, false, /*write_arena=*/true);
  c->train_labels = nullptr;
  if (rc) return rc;
  const DevTables t{c->last_tables, c->last_offsets};
  // ---- loss and d(scores)
  CUDA_TRY(cudaMemsetAsync(gflat_dev, 0, (size_t)c->flat_size * sizeof(float), st));
  CUDA_TRY(cudaMemsetAsync(loss_dev, 0, sizeof(float), st));
  if (dword_dev)
    CUDA_TRY(cudaMemsetAsync(dword_dev, 0, (size_t)T * N * c->cfg.text_dim * sizeof(float), st));
  // VQA: cross-entropy on every row (exp_vqa/train_vqa_rl_gt_layout.py:101-116; invalid_expr_loss
  // only seeds the baseline there)
  TRY(ctx_launch(c, loss_kernel, (N + 7) / 8, 256, 0, st, {}, scores_dev, score_prior_dev,
                 t.at(t.o.labels), t.at(t.o.q_ptr), N, C, invalid_expr_loss, vqa ? 1 : 0, c->dscores,
                 dscores_dev, c->dword_scale, loss_dev + 1, loss_dev));
  prof_mark(c, "loss_kernel", st);
  BwdCtx bc;
  bc.md = c->md; bc.tb = c->tb; bc.arena = c->arena; bc.scores = scores_dev;
  bc.dscores = c->dscores; bc.mbuf = c->mbuf; bc.gflat = gflat_dev; bc.dtau = c->dtau;
  bc.dmap = c->dmap; bc.dstencil = c->dstencil; bc.gmap = c->gmap; bc.phi = c->phi_buf; bc.go = c->go;
  bc.dehat = nullptr;
  // the exact-fp32 verification path keeps the per-root CUDA-core loop of the walk
  if (c->ehat && !(c->cfg.flags & N2NMN_FLAG_PROJ_FP32_SIMT)) {
    TRY(bwd_answer_tail(c, bc, t, N, gflat_dev, st));
    bc.dehat = c->dehat;
  }
  TRY(bwd_walk(c, bc, S, t, st));
  TRY(bwd_text(c, S, t, gflat_dev, dword_dev, st));
  return bwd_features(c, S, t, gflat_dev, st);
}

namespace {
int adam_impl(n2nmn_ctx* c, float* wflat, float* gflat, float* m, float* v, int step, float lr,
              float beta1, float beta2, float eps, float max_norm, float weight_decay, float gscale,
              float* l2_dev, cudaStream_t st) {
  const int nv = (int)c->vars.size();
  if (!c->segs_ready) {
    std::vector<VarSeg> segs(nv);
    for (int i = 0; i < nv; ++i) {
      segs[i].offset = (int)c->flat_offset[i];
      segs[i].count = (int)c->vars[i].count;
      const std::string& n = c->vars[i].name;   // l2_reg covers ".../weights" only
      segs[i].decay = n.size() >= 8 && n.compare(n.size() - 8, 8, "/weights") == 0;
    }
    CUDA_TRY(alloc_once(&c->d_segs, nv * sizeof(VarSeg)));
    CUDA_TRY(cudaMemcpy(c->d_segs, segs.data(), nv * sizeof(VarSeg), cudaMemcpyHostToDevice));
    CUDA_TRY(alloc_once(&c->d_sumsq, nv * sizeof(float)));
    c->segs_ready = true;
  }
  CUDA_TRY(cudaMemsetAsync(c->d_sumsq, 0, nv * sizeof(float), st));
  const dim3 grid(32, nv);
  TRY(ctx_launch(c, grad_norm_kernel, grid, 256, 0, st, {}, wflat, gflat, c->d_segs,
                 weight_decay, gscale, c->d_sumsq, l2_dev));
  const double lr_t = (double)lr * std::sqrt(1.0 - std::pow((double)beta2, step)) /
                      (1.0 - std::pow((double)beta1, step));
  TRY(ensure_repack_tables(c));
  TRY(ctx_launch(c, adam_clip_kernel<true>, grid, 256, 0, st, {}, wflat, gflat, m, v,
                 c->d_segs, c->d_sumsq, (float)lr_t, beta1, beta2, eps, max_norm,
                 c->d_repack, c->wbuf, c->Mp));
  prof_mark(c, "clip_adam_kernels", st);
  const int rc = repack_derived(c, wflat, st);
  prof_mark(c, "repack_kernels", st);
  return rc;
}
}  // namespace

int n2nmn_adam_step(n2nmn_ctx* c, float* wflat, float* gflat, float* m, float* v, int step,
                    float lr, float beta1, float beta2, float eps, float max_norm,
                    float weight_decay, void* stream) {
  if (!c || !wflat || !gflat || !m || !v || step < 1) return fail(N2NMN_ERR_ARG, "bad argument");
  return adam_impl(c, wflat, gflat, m, v, step, lr, beta1, beta2, eps, max_norm, weight_decay, 1.f,
                   nullptr, static_cast<cudaStream_t>(stream));
}

int n2nmn_train_finish(n2nmn_ctx* c, float* wflat, float* gflat, float* m, float* v, int step,
                       float lr, float beta1, float beta2, float eps, float max_norm,
                       float weight_decay, const float* loss_sum_dev, const float* per_sample_dev,
                       const float* log_seq_prob_dev, int N, int world, float baseline_decay,
                       const float* state_in_dev, float* state_out_dev, float* coeff_dev,
                       void* stream) {
  if (!c || !wflat || !gflat || !m || !v || step < 1 || !loss_sum_dev || !per_sample_dev ||
      !state_in_dev || !state_out_dev || N <= 0 || world <= 0)
    return fail(N2NMN_ERR_ARG, "bad argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  TRY(ctx_launch(c, train_scalars_kernel, 1, 256, 0, st, {}, loss_sum_dev, per_sample_dev,
                 log_seq_prob_dev, N, world, baseline_decay, state_in_dev, state_out_dev, coeff_dev));
  return adam_impl(c, wflat, gflat, m, v, step, lr, beta1, beta2, eps, max_norm, weight_decay,
                   1.f / (float)world, state_out_dev + 3, st);
}

int n2nmn_set_grad_scale(n2nmn_ctx* c, float scale) {
  if (!c) return fail(N2NMN_ERR_ARG, "null context");
  c->dword_scale = scale;
  return 0;
}

int n2nmn_set_tree_cluster(n2nmn_ctx* c, int ctas_per_question) {
  if (!c) return fail(N2NMN_ERR_ARG, "n2nmn_set_tree_cluster: null context");
  const int v = ctas_per_question;
  if (!(v == 0 || v == 1 || v == 2 || v == 4 || v == 8))
    return fail(N2NMN_ERR_ARG, "n2nmn_set_tree_cluster: ctas_per_question must be 0, 1, 2, 4 or 8");
  c->tree_cluster = v;
  return 0;
}

int n2nmn_set_proj_ctas(n2nmn_ctx* c, int max_ctas) {
  if (!c) return fail(N2NMN_ERR_ARG, "n2nmn_set_proj_ctas: null context");
  if (max_ctas < 0) return fail(N2NMN_ERR_ARG, "n2nmn_set_proj_ctas: max_ctas must be >= 0");
  c->proj_max_ctas = max_ctas;
  return 0;
}

int n2nmn_set_text_ctas_per_group(n2nmn_ctx* c, int n) {
  if (!c) return fail(N2NMN_ERR_ARG, "n2nmn_set_text_ctas_per_group: null context");
  if (n < 0) return fail(N2NMN_ERR_ARG, "n2nmn_set_text_ctas_per_group: n must be >= 0");
  return 0;   // retired: the text kernel's grid follows the schedule (see the header)
}

int n2nmn_set_profiling(n2nmn_ctx* c, int enabled) {
  if (!c) return fail(N2NMN_ERR_ARG, "null context");
  c->profiling = enabled != 0;
  return 0;
}

int n2nmn_get_launch_times(n2nmn_ctx* c, const char** names, float* us, int cap) {
  if (!c) return fail(N2NMN_ERR_ARG, "null context");
  if (c->ev_used < 2) return 0;
  if (cudaEventSynchronize(c->ev[c->ev_used - 1]) != cudaSuccess)
    return fail(N2NMN_ERR_CUDA, "event sync failed");
  int n = 0;
  for (int i = 1; i < c->ev_used && n < cap; ++i, ++n) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, c->ev[i - 1], c->ev[i]);
    if (names) names[n] = c->ev_names[i];
    if (us) us[n] = ms * 1000.f;
  }
  return n;
}

int64_t n2nmn_launch_count(const n2nmn_ctx* c) { return c ? c->launches : 0; }

}  // extern "C"

