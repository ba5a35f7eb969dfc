// Host-side layout compiler (see schedule.hpp). Plain C++; no CUDA calls.
#include "schedule.hpp"

#include <algorithm>
#include <cstring>

namespace n2nmn {

namespace {

int text_set_of(int op) {
  switch (op) {
    case OP_FIND: case OP_FILTER: return TS_FIND;
    case OP_FIND_SAME_PROPERTY: return TS_FSP;
    case OP_TRANSFORM: return TS_TRANSFORM;
    case OP_SAME_PROPERTY: return TS_SAMEPROP;
    case OP_DESCRIBE: return TS_DESCRIBE;
    default: return -1;
  }
}

}  // namespace

int compile_schedule(const SchedShape& shp, const int32_t* tokens, int T, int N,
                     const int32_t* vocab_ops, int num_vocab, HostSchedule* out,
                     const char** err, bool train) {
  return compile_schedule_group(shp, &tokens, 1, T, N, vocab_ops, num_vocab, out, err, train);
}

int compile_schedule_group(const SchedShape& shp, const int32_t* const* tokens_seg, int num_seg,
                           int T, int N, const int32_t* vocab_ops, int num_vocab,
                           HostSchedule* out, const char** err, bool train, bool pooled_direct) {
  HostSchedule& S = *out;
  S.reset();
  S.N = N; S.T = T; S.num_seg = num_seg;
  S.pooled_direct = pooled_direct && !train;
  const int NQ = num_seg * N;
  S.validity.assign(NQ, 0);
  S.q_ptr.assign(NQ + 1, 0);

  static thread_local std::vector<int32_t> tq;
  tq.resize((size_t)N * T);
  const int scene_bits = [] { float v = 3.0f; int b; std::memcpy(&b, &v, 4); return b; }();
  S.nodes.clear();
  S.depth.clear();
  S.nodes.reserve((size_t)NQ * 8);
  S.depth.reserve((size_t)NQ * 8);
  // node ids of the question's open attention / answer values (at most one push per token)
  static thread_local std::vector<int> stack_buf;
  stack_buf.resize((size_t)T + 1);
  int* stack = stack_buf.data();

  for (int seg = 0; seg < num_seg; ++seg) {
  const int32_t* tokens = tokens_seg[seg];
  // tokens are time-major [T,N]: transpose once so that every question is a contiguous row
  for (int t = 0; t < T; ++t)
    for (int n = 0; n < N; ++n) tq[(size_t)n * T + t] = tokens[(size_t)t * N + n];
  for (int n = 0; n < N; ++n) {
    const int q = seg * N + n;   // question = image index across the segments
    const int32_t* col = tq.data() + (size_t)n * T;
    bool has_eos = false;
    for (int t = 0; t < T; ++t) {
      const int tok = col[t];
      if (tok >= 0 && tok < num_vocab && vocab_ops[tok] < 0) { has_eos = true; break; }
    }
    const int base = (int)S.nodes.size();
    bool ok = has_eos;
    int sp = 0;
    for (int t = 0; t < T && ok; ++t) {
      const int tok = col[t];
      if (tok < 0 || tok >= num_vocab) { ok = false; break; }
      const int op = vocab_ops[tok];
      if (op < 0) break;                       // <eos>
      if (op >= NUM_OPS) { ok = false; break; }
      const int ar = kArity[op];
      if (sp < ar) { ok = false; break; }   // not enough input
      NodeRec nd;
      nd.op = op; nd.t = t; nd.b = q;
      nd.in0 = nd.in1 = -1;
      nd.text = -1;
      nd.aux = (op == OP_SCENE) ? scene_bits : -1;
      nd.aux2 = -1; nd.s0 = nd.s1 = nd.so = -1;
      int depth = 1;
      // operands come off right-to-left: the last popped is input_0
      for (int slot = ar - 1; slot >= 0; --slot) {
        const int child = stack[--sp];
        if (kIsAns[S.nodes[child].op]) { ok = false; break; }  // input must be attention
        (slot == 0 ? nd.in0 : nd.in1) = child;
        depth = std::max(depth, S.depth[child] + 1);
      }
      if (!ok) break;
      const int id = (int)S.nodes.size();
      nd.out = kIsAns[op] ? q : id;
      S.nodes.push_back(nd);
      S.depth.push_back(depth);
      stack[sp++] = id;
    }
    if (ok && !(sp == 1 && kIsAns[S.nodes[stack[0]].op])) ok = false;
    if (ok) {
      S.validity[q] = 1;
      ++S.num_valid;
    } else {
      S.nodes.resize(base);   // an invalid layout contributes no nodes
      S.depth.resize(base);
    }
    S.q_ptr[q + 1] = (int)S.nodes.size();
  }
  }
  (void)err;
  return finalize_schedule(shp, N, out, train);
}

int finalize_schedule(const SchedShape& shp, int images_per_seg, HostSchedule* out, bool train) {
  HostSchedule& S = *out;
  const int N = images_per_seg * std::max(1, S.num_seg);   // images over all segments
  const int NQ = (int)S.q_ptr.size() - 1;   // questions (rows of the score matrix)
  const int num_nodes = (int)S.nodes.size();
  S.max_depth = 0;
  S.groups.clear(); S.work.clear();
  S.num_mslots = 0; S.num_find_nodes = 0;
  for (int k = 0; k < 3; ++k) S.kbytes[k] = S.kflops[k] = 0;
  S.per_node_bytes = S.per_node_flops = 0;
  // ---- text rows, grouped by weight set
  int set_count[NUM_TEXT_SETS] = {0};
  for (const NodeRec& r : S.nodes) if (text_set_of(r.op) >= 0) ++set_count[text_set_of(r.op)];
  int set_start[NUM_TEXT_SETS + 1] = {0};
  for (int s = 0; s < NUM_TEXT_SETS; ++s) set_start[s + 1] = set_start[s] + set_count[s];
  const int num_text = set_start[NUM_TEXT_SETS];
  S.text_t.assign(num_text, 0);
  S.text_b.assign(num_text, 0);
  int cursor[NUM_TEXT_SETS];
  for (int s = 0; s < NUM_TEXT_SETS; ++s) cursor[s] = set_start[s];
  for (int i = 0; i < num_nodes; ++i) {
    NodeRec& r = S.nodes[i];
    const int tset = text_set_of(r.op);
    if (tset >= 0) {
      const int row = cursor[tset]++;
      r.text = row;
      S.text_t[row] = r.t;
      S.text_b[row] = r.b;
    }
    S.max_depth = std::max(S.max_depth, S.depth[i]);
  }
  S.text_set_start.assign(set_start, set_start + NUM_TEXT_SETS + 1);
  for (int s = 0; s < NUM_TEXT_SETS; ++s)
    for (int r = set_start[s]; r < set_start[s + 1]; r += kTextRowsPerCta) {
      TextGroup g;
      g.set = s; g.start = r; g.count = std::min(kTextRowsPerCta, set_start[s + 1] - r); g.pad = 0;
      S.groups.push_back(g);
    }

  // ---- projection work: fused Find/Filter consumers per image; stored maps for the images that
  //      host a FindSameProperty / Describe / SameProperty node (one mbuf slot per image and set)
  const int HW = shp.H * shp.W;
  S.img_ptr.assign(N + 1, 0);
  S.mslot.assign((size_t)NUM_PROJ_SETS * N, -1);
  auto want = [&](int set, int b) -> int {
    int32_t& slot = S.mslot[(size_t)set * N + b];
    if (slot < 0) slot = S.num_mslots++;
    return slot;
  };
  S.train = train;
  if (train) S.pooled_direct = false;
  S.num_pool_rows = 0; S.num_feat_rows = 0;
  S.head_work.clear(); S.head_list.clear(); S.pool_img.clear();
  if (S.pooled_direct) {
    // rows of the root-input buffer: first the roots that pool image features (Describe: 1 row,
    // SameProperty: 2 — the pool kernel's grid covers exactly these), then the other answer roots
    for (int pass = 0; pass < 2; ++pass)
      for (int i = 0; i < num_nodes; ++i) {
        NodeRec& r = S.nodes[i];
        const bool feat = (r.op == OP_DESCRIBE || r.op == OP_SAME_PROPERTY);
        if (r.op < OP_EXIST || feat != (pass == 0)) continue;
        const bool two = (r.op == OP_SAME_PROPERTY || r.op == OP_EQUAL_NUM ||
                          r.op == OP_MORE_NUM || r.op == OP_LESS_NUM);
        r.aux = S.num_pool_rows++;
        r.aux2 = two ? S.num_pool_rows++ : -1;
        if (feat) { S.pool_img.push_back(r.b); if (two) S.pool_img.push_back(r.b); }
      }
    S.num_feat_rows = (int)S.pool_img.size();
  }
  S.entries.clear();
  S.node_entry.assign(train ? num_nodes : 0, -1);
  auto entry = [&](int node, int set, int b) {
    if (!train) return;
    if (S.node_entry[node] < 0) S.node_entry[node] = (int)S.entries.size();
    S.entries.push_back(BwdEntryHost{set, b});
  };
  for (int i = 0; i < num_nodes; ++i) {
    NodeRec& r = S.nodes[i];
    switch (r.op) {
      case OP_FIND: case OP_FILTER:
        ++S.img_ptr[r.b + 1];
        // training keeps the conv_image map of the image: the backward pass needs m[p,:]
        if (train) { r.aux = want(PS_FIND, r.b); entry(i, PS_FIND, r.b); }
        break;
      case OP_FIND_SAME_PROPERTY:
        r.aux = want(PS_FSP_IMG, r.b); r.aux2 = want(PS_FSP_ATT, r.b);
        entry(i, PS_FSP_IMG, r.b); entry(i, PS_FSP_ATT, r.b); break;
      case OP_DESCRIBE:
        if (S.pooled_direct) break;
        r.aux = want(PS_DESC_ATT, r.b); entry(i, PS_DESC_ATT, r.b); break;
      case OP_SAME_PROPERTY:
        if (S.pooled_direct) break;
        r.aux = want(PS_SP_ATT0, r.b); r.aux2 = want(PS_SP_ATT1, r.b);
        entry(i, PS_SP_ATT0, r.b); entry(i, PS_SP_ATT1, r.b); break;
      default: break;
    }
  }
  if (S.pooled_direct) {   // head-kernel work: chunks of root nodes of one type
    const int per = head_nodes_per_cta(shp.Dk, shp.Mp);
    for (int op = OP_EXIST; op < NUM_OPS; ++op) {
      int open = -1;
      for (int i = 0; i < num_nodes; ++i) {
        if (S.nodes[i].op != op) continue;
        if (open < 0 || S.head_work[open].count == per) {
          open = (int)S.head_work.size();
          S.head_work.push_back(HeadWork{(int32_t)S.head_list.size(), 0, op, 0});
        }
        S.head_list.push_back(i);
        ++S.head_work[open].count;
      }
    }
  }
  for (int n = 0; n < N; ++n) S.img_ptr[n + 1] += S.img_ptr[n];
  S.num_find_nodes = S.img_ptr[N];
  S.node_text.assign(S.num_find_nodes, 0);
  S.node_out.assign(S.num_find_nodes, 0);
  {
    static thread_local std::vector<int32_t> fill;
    fill.assign(S.img_ptr.begin(), S.img_ptr.end() - 1);
    for (const NodeRec& r : S.nodes) {
      if (r.op == OP_FIND || r.op == OP_FILTER) {
        const int e = fill[r.b]++;
        S.node_text[e] = r.text;
        S.node_out[e] = r.out;
      }
    }
  }
  int u_set[NUM_PROJ_SETS] = {0}, u_any = 0;
  for (int n = 0; n < N; ++n) {
    bool any = S.img_ptr[n + 1] > S.img_ptr[n];
    if (any) ++u_set[PS_FIND];
    for (int set = 1; set < NUM_PROJ_SETS; ++set)
      if (S.mslot[(size_t)set * N + n] >= 0) { ++u_set[set]; any = true; }
    // (PS_FIND maps stored for training ride along with the fused pass: no extra work items)
    if (any) ++u_any;
  }
  // Tiles (128 rows of one segment x one layer x one pass of <= 8 Find consumers) in tile-major
  // order: the layers that need the same 128 rows of features are handed out at about the same
  // time, so the A tile is fetched from HBM once and the other layers hit it in L2 (matters once
  // the batch no longer fits in L2).
  const int seg_rows = images_per_seg * HW;
  const int tiles_per_seg = (seg_rows + 127) / 128;
  S.work.reserve((size_t)tiles_per_seg * std::max(1, S.num_seg));
  for (int seg = 0; seg < std::max(1, S.num_seg); ++seg) {
    const int g0 = seg * images_per_seg;
    for (int tile = 0; tile < tiles_per_seg; ++tile) {
      const int r0 = tile * 128, r1 = std::min(seg_rows, r0 + 128) - 1;
      const int b0 = g0 + r0 / HW, b1 = g0 + r1 / HW;
      int need[NUM_PROJ_SETS] = {0};     // consumers per layer among the tile's images
      for (int b = b0; b <= b1; ++b) {
        need[PS_FIND] = std::max(need[PS_FIND], S.img_ptr[b + 1] - S.img_ptr[b]);
        for (int set = 1; set < NUM_PROJ_SETS; ++set)
          if (u_set[set] && S.mslot[(size_t)set * N + b] >= 0) need[set] = 1;
      }
      for (int set = 0; set < NUM_PROJ_SETS; ++set) {
        const int passes = (need[set] + kMaxProjNodesPerPass - 1) / kMaxProjNodesPerPass;
        for (int pass = 0; pass < passes; ++pass) S.work.push_back(ProjWork{r0, seg, pass, set});
      }
    }
  }

  // ---- shared-memory stack slots for the tree kernel: a map lives from its producer to its
  //      (single) consumer; inputs are released before the output is placed, so in-place reuse
  //      is allowed (every module copies or finishes reading its inputs before it writes).
  S.max_stack = 0;
  {
    static thread_local std::vector<int> free_slots;
    for (int q = 0; q < NQ; ++q) {
      free_slots.clear();
      int next = 0;
      for (int i = S.q_ptr[q]; i < S.q_ptr[q + 1]; ++i) {
        NodeRec& r = S.nodes[i];
        r.s0 = r.in0 >= 0 ? S.nodes[r.in0].so : -1;
        r.s1 = r.in1 >= 0 ? S.nodes[r.in1].so : -1;
        if (r.s0 >= 0) free_slots.push_back(r.s0);
        if (r.s1 >= 0) free_slots.push_back(r.s1);
        r.so = -1;
        if (r.op <= OP_OR) {   // attention-typed output
          if (!free_slots.empty()) {
            auto it = std::min_element(free_slots.begin(), free_slots.end());
            r.so = *it;
            free_slots.erase(it);
          } else {
            r.so = next++;
          }
        }
      }
      S.max_stack = std::max(S.max_stack, next);
    }
  }

  S.wave_ptr.clear(); S.wave_nodes.clear();   // built on demand (build_waves)
  S.accounted = false;
  S.u_any = u_any;
  for (int set = 0; set < NUM_PROJ_SETS; ++set) S.u_set[set] = u_set[set];
  S.set_count_text = 0;
  for (int st = 0; st < NUM_TEXT_SETS; ++st) S.set_count_text += set_count[st] > 0;
  return 0;
}


// Depth-bucketed waves for the wave executor; the tree executor never needs them.
void build_waves(HostSchedule* out) {
  HostSchedule& S = *out;
  if (!S.wave_ptr.empty()) return;
  const int num_nodes = (int)S.nodes.size();
  // ---- waves (Find is complete after the projection kernel, so it never enters a wave)
  S.wave_ptr.assign(S.max_depth + 2, 0);
  for (int i = 0; i < num_nodes; ++i)
    if (S.nodes[i].op != OP_FIND) ++S.wave_ptr[S.depth[i] + 1];
  for (int d = 0; d <= S.max_depth; ++d) S.wave_ptr[d + 1] += S.wave_ptr[d];
  S.wave_nodes.assign(S.wave_ptr[S.max_depth + 1], 0);
  {
    std::vector<int32_t> fill(S.wave_ptr.begin(), S.wave_ptr.end() - 1);
    for (int i = 0; i < num_nodes; ++i)
      if (S.nodes[i].op != OP_FIND) S.wave_nodes[fill[S.depth[i]]++] = i;
  }

}

void build_bwd_order(HostSchedule* out) {
  HostSchedule& W = *out;
  // bucket 2*depth: the level's Transform nodes (the long CTAs: scheduled first), 2*depth + 1:
  // its other nodes
  const int nb = 2 * (W.max_depth + 1);
  W.bwd_ptr.assign(nb + 1, 0);
  auto bucket = [&](size_t i) { return 2 * W.depth[i] + (W.nodes[i].op == OP_TRANSFORM ? 0 : 1); };
  for (size_t i = 0; i < W.nodes.size(); ++i) ++W.bwd_ptr[bucket(i) + 1];
  for (int b = 0; b < nb; ++b) W.bwd_ptr[b + 1] += W.bwd_ptr[b];
  W.bwd_nodes.assign(W.nodes.size(), 0);
  std::vector<int32_t> fill(W.bwd_ptr.begin(), W.bwd_ptr.end() - 1);
  for (size_t i = 0; i < W.nodes.size(); ++i) W.bwd_nodes[fill[bucket(i)]++] = (int32_t)i;
  W.entry_order.resize(W.entries.size());
  for (size_t i = 0; i < W.entries.size(); ++i) W.entry_order[i] = (int32_t)i;
  std::stable_sort(W.entry_order.begin(), W.entry_order.end(),
                   [&](int32_t a, int32_t b) { return W.entries[a].set < W.entries[b].set; });
}

// §8(d) traffic / work accounting; only needed when statistics are requested, so it is kept off
// the per-step path.
void account_schedule(const SchedShape& shp, HostSchedule* out) {
  HostSchedule& S = *out;
  if (S.accounted) return;
  S.accounted = true;
  const int NQ = (int)S.q_ptr.size() - 1;
  const int HW = shp.H * shp.W;
  const int num_text = (int)S.text_t.size();
  const int sets_used = S.set_count_text;
  const int u_any = S.u_any;
  const int* u_set = S.u_set;
  for (int k = 0; k < 3; ++k) S.kbytes[k] = S.kflops[k] = 0;
  S.per_node_bytes = S.per_node_flops = 0;
  // ---- algorithmic bytes / flops (SURVEY.md §8d, App. D), fp32
  const int64_t D = shp.Dk, M = shp.M, C = shp.C, Dt = shp.Dt, hw = HW;
  const int64_t tile_b = hw * D * 4, att_b = hw * 4, txt_b = Dt * 4;
  const int64_t contraction = 2 * hw * D * M, tail = 6 * hw * M, txt_f = 2 * Dt * M;
  const int64_t pool_f = 2 * hw * D + 2 * D * M;
  int64_t node_bytes = 0, node_flops = 0;      // what the node kernels move / compute
  for (int n = 0; n < NQ; ++n) {
    for (int i = S.q_ptr[n]; i < S.q_ptr[n + 1]; ++i) {
      const int op = S.nodes[i].op;
      int64_t rb = 0, wb = 0, fl = 0, kb = 0, kf = 0;   // per-node figure / node-kernel share
      switch (op) {
        case OP_SCENE: wb = att_b; kb = att_b; break;
        case OP_FIND: rb = tile_b + txt_b; wb = att_b; fl = contraction + txt_f + tail; break;
        case OP_FILTER: rb = tile_b + txt_b + att_b; wb = att_b; fl = contraction + txt_f + tail + hw;
          kb = 3 * att_b; kf = hw; break;
        case OP_FIND_SAME_PROPERTY: rb = tile_b + txt_b + att_b; wb = att_b;
          fl = contraction + txt_f + tail + pool_f; kb = 2 * att_b + 2 * hw * M * 4; kf = tail + 2 * hw * M; break;
        case OP_TRANSFORM: {
          const int64_t stencil = 2 * hw * shp.ksize * shp.ksize * M;
          rb = att_b + txt_b; wb = att_b; fl = stencil + txt_f + tail;
          kb = 2 * att_b; kf = stencil + tail; break;
        }
        case OP_AND: case OP_OR: rb = 2 * att_b; wb = att_b; fl = hw; kb = 3 * att_b; kf = hw; break;
        case OP_EXIST: rb = att_b; wb = C * 4; fl = 6 * C + 3 * hw; kb = rb + wb; kf = fl; break;
        case OP_COUNT: rb = att_b; wb = C * 4; fl = 2 * (hw + 2) * C; kb = rb + wb; kf = fl; break;
        case OP_EQUAL_NUM: case OP_MORE_NUM: case OP_LESS_NUM:
          rb = 2 * att_b; wb = C * 4; fl = 4 * (hw + 2) * C; kb = rb + wb; kf = fl; break;
        // pooled_direct: the node kernels (tree + head) read the feature tile itself and do the
        // fc_att product on the pooled vector; else they read the stored [HW,M] map(s)
        case OP_SAME_PROPERTY: rb = tile_b + txt_b + 2 * att_b; wb = C * 4;
          fl = 2 * pool_f + txt_f + 2 * M * C;
          if (S.pooled_direct) { kb = 2 * att_b + wb + tile_b + txt_b; kf = 2 * pool_f + 2 * M * C; }
          else { kb = 2 * att_b + wb + 2 * hw * M * 4; kf = 4 * hw * M + 2 * M * C; }
          break;
        case OP_DESCRIBE: rb = tile_b + txt_b + att_b; wb = C * 4;
          fl = pool_f + txt_f + 2 * M * C;
          if (S.pooled_direct) { kb = att_b + wb + tile_b + txt_b; kf = pool_f + 2 * M * C; }
          else { kb = att_b + wb + hw * M * 4; kf = 2 * hw * M + 2 * M * C; }
          break;
      }
      S.per_node_bytes += rb + wb;
      S.per_node_flops += fl;
      node_bytes += kb;
      node_flops += kf;
    }
  }
  S.kbytes[0] = (int64_t)num_text * (txt_b + M * 4) + (int64_t)sets_used * Dt * M * 4;
  S.kflops[0] = (int64_t)num_text * txt_f;
  // projection launch: every distinct feature tile once, one weight matrix per set in use,
  // Find outputs + text operands, stored maps of the other sets
  S.kbytes[1] = (int64_t)u_any * tile_b + (int64_t)S.num_find_nodes * (M * 4 + att_b);
  S.kflops[1] = (int64_t)S.num_find_nodes * tail;
  for (int set = 0; set < NUM_PROJ_SETS; ++set) {
    if (!u_set[set]) continue;
    S.kbytes[1] += D * M * 4 + (set == PS_FIND ? 0 : (int64_t)u_set[set] * hw * M * 4);
    S.kflops[1] += (int64_t)u_set[set] * contraction;
  }
  S.kbytes[2] = node_bytes;
  S.kflops[2] = node_flops;
}

}  // namespace n2nmn
