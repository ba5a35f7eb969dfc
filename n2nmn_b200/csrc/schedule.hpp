// Host-side layout compiler: Reverse-Polish layout tokens [T,N] -> launch tables.
//
// Replaces, for the throughput path, the Python `Assembler.assemble`
// (models_clevr/nmn3_assembler.py:153-222: RPN stack decode + validity rules) and TF Fold's
// `compiler.build_feed_dict` (models_clevr/nmn3_model.py:146-159 + loom weaver): no Python dicts,
// no per-node objects — flat int tables that go to the device in ONE copy.
#pragma once
#include <cstdint>
#include <vector>

#include "common.cuh"

namespace n2nmn {

// Per opcode: attention inputs, and whether the module answers (ends a question).
inline constexpr int kArity[NUM_OPS] = {0, 0, 1, 1, 1, 2, 2, 1, 1, 2, 2, 2, 2, 1};
inline constexpr bool kIsAns[NUM_OPS] = {false, false, false, false, false, false, false,
                                         true, true, true, true, true, true, true};

struct SchedShape {
  int family, H, W, Dk, Dt, M, Mp, C, ksize;
  int max_T;
};

struct BwdEntryHost { int32_t set, b; };   // mirrors BwdEntry (backward.cuh)

struct HostSchedule {
  int N = 0, T = 0, num_valid = 0, max_depth = 0;   // N = images (questions) per segment
  int num_seg = 1;                    // batches covered by this schedule (common.cuh: segments)
  std::vector<uint8_t> validity;      // [num_seg*N]
  std::vector<NodeRec> nodes;         // (question, token) order; node id = index = arena slot
  std::vector<int32_t> depth;         // per node
  std::vector<int32_t> q_ptr;         // [N+1]
  std::vector<int32_t> text_t, text_b;
  std::vector<TextGroup> groups;
  std::vector<ProjWork> work;
  std::vector<int32_t> img_ptr, node_text, node_out, mslot;
  int num_mslots = 0;
  int num_find_nodes = 0;
  // Evaluation schedules of the tree executor: the attention-pooled answer roots (Describe,
  // SameProperty) do not get stored fc_att maps from the contraction kernel; the tree kernel writes
  // their pooled feature vectors Σ_p s_p·X[p,:] and a batched head kernel finishes them
  // (head_kernel.cuh). Requested by the caller before finalize_schedule; never with `train`.
  bool pooled_direct = false;
  int num_pool_rows = 0;               // rows of the root-input buffer in use
  int num_feat_rows = 0;               // the first rows: roots that pool image features
  std::vector<int32_t> pool_img;       // per row: image index (across the segments)
  std::vector<HeadWork> head_work;     // one entry per CTA of the head kernel
  std::vector<int32_t> head_list;      // node ids, grouped by head_work
  int max_stack = 0;                  // most attention maps of one question alive at once
  std::vector<int32_t> wave_ptr;      // [max_depth+2], wave d = [wave_ptr[d], wave_ptr[d+1])
  std::vector<int32_t> wave_nodes;
  std::vector<int32_t> bwd_ptr, bwd_nodes;   // training: ALL nodes bucketed by depth (build_bwd_order)
  std::vector<int32_t> entry_order;          // training: B-map entries sorted by weight set
  // training schedules only: one [HW,Mp] gradient map per feature-side layer use
  bool train = false;
  std::vector<BwdEntryHost> entries;
  std::vector<int32_t> node_entry;     // per node: first entry (or -1)
  std::vector<int32_t> text_set_start; // [NUM_TEXT_SETS+1] rows of each text weight set
  // §8(d) algorithmic traffic / work, per kernel: 0 text, 1 projection, 2 node kernels
  int64_t kbytes[3] = {0, 0, 0};
  int64_t kflops[3] = {0, 0, 0};
  int64_t per_node_bytes = 0;         // Σ over nodes of the App. D per-node figure
  int64_t per_node_flops = 0;
  // inputs of the lazy accounting
  bool accounted = false;
  int u_any = 0, u_set[NUM_PROJ_SETS] = {0}, set_count_text = 0;

  // Forget the contents but keep every vector's capacity (the per-step path reuses one object).
  void reset() {
    N = T = num_valid = max_depth = num_mslots = num_find_nodes = max_stack = 0;
    num_seg = 1;
    validity.clear(); nodes.clear(); depth.clear(); q_ptr.clear(); text_t.clear();
    text_b.clear(); groups.clear(); work.clear(); img_ptr.clear(); node_text.clear();
    node_out.clear(); mslot.clear(); wave_ptr.clear(); wave_nodes.clear(); bwd_ptr.clear(); bwd_nodes.clear(); entry_order.clear();
    entries.clear(); node_entry.clear(); text_set_start.clear(); train = false;
    pooled_direct = false; num_pool_rows = 0; num_feat_rows = 0; head_work.clear();
    head_list.clear();
    pool_img.clear();
    for (int k = 0; k < 3; ++k) kbytes[k] = kflops[k] = 0;
    per_node_bytes = per_node_flops = 0;
    accounted = false;
  }
};

// Returns 0 or a negative n2nmn_status; `err` receives a message on failure.
int compile_schedule(const SchedShape& shp, const int32_t* tokens, int T, int N,
                     const int32_t* vocab_ops, int num_vocab, HostSchedule* out,
                     const char** err, bool train = false);
// Same for `num_seg` token matrices [T,N] (independent batches of identical shape evaluated by
// one set of launches): questions and images are numbered seg*N + n.
int compile_schedule_group(const SchedShape& shp, const int32_t* const* tokens, int num_seg, int T,
                           int N, const int32_t* vocab_ops, int num_vocab, HostSchedule* out,
                           const char** err, bool train = false, bool pooled_direct = false);

// Builds every derived table (text rows, projection work, waves, traffic accounting) from
// S.nodes / S.depth / S.q_ptr. `images_per_seg` x S.num_seg bounds NodeRec::b. Used by
// compile_schedule and by the per-module entry point, which fabricates one single-node
// "question" per call row.
int finalize_schedule(const SchedShape& shp, int images_per_seg, HostSchedule* out,
                      bool train = false);

// Fills wave_ptr / wave_nodes (depth-bucketed waves). Idempotent.
void build_waves(HostSchedule* out);

// Fills bwd_ptr / bwd_nodes and entry_order of a training schedule: every node bucketed by depth
// (leaves = 1), since the backward runs one launch per level, top down.
void build_bwd_order(HostSchedule* out);

// Fills kbytes / kflops / per_node_* (SURVEY.md §8d). Idempotent.
void account_schedule(const SchedShape& shp, HostSchedule* out);

}  // namespace n2nmn
