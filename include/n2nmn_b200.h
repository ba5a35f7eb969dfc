/*
 * n2nmn_b200 — C ABI of the H100-native N2NMN module-network hot path.
 *
 * The reference (ronghanghu/n2nmn) has no FFI of its own: its hot path is a chain of TensorFlow
 * graph calls made from Python. Each entry point below therefore names the reference *Python*
 * interface it replaces (paths under the reference repo); INTEGRATION.md shows the ctypes stubs a
 * maintainer of the reference would add to `models_clevr/nmn3_modules.py` / `nmn3_model.py`.
 *
 * Conventions
 *   - every function returns 0 on success, a negative n2nmn_status otherwise; the message of the
 *     last failure on the calling thread is available from n2nmn_last_error(); nothing throws
 *     across this boundary;
 *   - "dev" pointers are CUDA device pointers to contiguous row-major fp32 (NHWC) / int32 data
 *     owned by the caller and valid until the work enqueued on `stream` has finished;
 *     "host" pointers are ordinary host memory read/written before the call returns unless
 *     stated otherwise;
 *   - `stream` is a cudaStream_t passed as void* (0 = legacy default stream). All device work is
 *     enqueued on it; no call synchronises the device except where documented;
 *   - a ctx is not thread-safe: one ctx per GPU per host thread.
 *   - the library runs on sm_90a only and fails with N2NMN_ERR_DEVICE elsewhere. There is no
 *     CPU fallback.
 */
#ifndef N2NMN_B200_H_
#define N2NMN_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define N2NMN_ABI_VERSION 2

typedef struct n2nmn_ctx n2nmn_ctx;
typedef struct n2nmn_sched n2nmn_sched;

enum n2nmn_status {
  N2NMN_OK = 0,
  N2NMN_ERR_ARG = -1,      /* bad argument / shape */
  N2NMN_ERR_CUDA = -2,     /* a CUDA call failed */
  N2NMN_ERR_DEVICE = -3,   /* not an sm_90 device */
  N2NMN_ERR_STATE = -4,    /* weights / inputs not bound yet */
  N2NMN_ERR_CAPACITY = -5  /* batch / T / node count exceeds what the ctx was created for */
};

/* Model families = the three near-identical packages of the reference
 * (models_clevr/, models_shapes/, models_vqa/). */
enum n2nmn_family { N2NMN_CLEVR = 0, N2NMN_SHAPES = 1, N2NMN_VQA = 2 };

/* Module opcodes. One per method of `class Modules`
 * (models_clevr/nmn3_modules.py:60-495). VQA `_Transform` is N2NMN_OP_FIND_SAME_PROPERTY with the
 * TransformModule weights (models_vqa/nmn3_modules.py:123-171); SHAPES `_Answer` is
 * N2NMN_OP_EXIST with the AnswerModule weights (models_shapes/nmn3_modules.py:123-150). */
enum n2nmn_op {
  N2NMN_OP_SCENE = 0,
  N2NMN_OP_FIND = 1,
  N2NMN_OP_FILTER = 2,
  N2NMN_OP_FIND_SAME_PROPERTY = 3,
  N2NMN_OP_TRANSFORM = 4,
  N2NMN_OP_AND = 5,
  N2NMN_OP_OR = 6,
  N2NMN_OP_EXIST = 7,
  N2NMN_OP_COUNT = 8,
  N2NMN_OP_EQUAL_NUM = 9,
  N2NMN_OP_MORE_NUM = 10,
  N2NMN_OP_LESS_NUM = 11,
  N2NMN_OP_SAME_PROPERTY = 12,
  N2NMN_OP_DESCRIBE = 13,
  N2NMN_NUM_OPS = 14
};

enum n2nmn_flags {
  /* Compute the conv_image contraction with the fp32 CUDA-core kernel instead of the wgmma
   * TF32 tensor-core kernel. Verification aid (bit-compatible with nothing, but free of TF32
   * rounding); never the default. */
  N2NMN_FLAG_PROJ_FP32_SIMT = 1,
  /* Execute the layout as depth-bucketed waves (one launch per tree depth over all questions)
   * instead of the default one-CTA-per-question tree walk. Same results. */
  N2NMN_FLAG_WAVE_EXECUTOR = 2
};

typedef struct n2nmn_config {
  int32_t abi_version;   /* N2NMN_ABI_VERSION */
  int32_t family;        /* enum n2nmn_family */
  int32_t H, W, D;       /* feature grid handed to Modules (D excludes the VQA coord channels) */
  int32_t text_dim;      /* 300 */
  int32_t map_dim;       /* 250 (CLEVR) / 500 (SHAPES) / 1024 (VQA) */
  int32_t kernel_size;   /* 5 / 3; unused for VQA */
  int32_t num_choices;
  int32_t max_batch;     /* capacity: questions per bind */
  int32_t max_T;         /* capacity: decoder steps */
  int32_t device;        /* CUDA device ordinal */
  int32_t flags;         /* enum n2nmn_flags */
  int32_t max_group;     /* capacity: independent batches (each <= max_batch questions) that one
                          * n2nmn_forward_group call may evaluate with one set of launches;
                          * 0 or 1 = none, at most 16. Workspaces scale with it. */
} n2nmn_config;

/* Replaces `Modules.__init__` (models_clevr/nmn3_modules.py:12-47): allocates the context,
 * weight storage and workspaces. Weights are NOT initialised here; see n2nmn_set_weight. */
int n2nmn_create(const n2nmn_config* cfg, n2nmn_ctx** out);
int n2nmn_destroy(n2nmn_ctx* ctx);
const char* n2nmn_last_error(void);

/* Number of variables the family owns and their TF names / shapes, in a fixed order
 * (SURVEY.md App. B; scope capture at models_clevr/nmn3_modules.py:17-18,91-92). Names are
 * relative to `.../module_variables/`, e.g. "FindModule/conv_image/weights". */
int n2nmn_num_variables(const n2nmn_ctx* ctx);
int n2nmn_variable_info(const n2nmn_ctx* ctx, int index, const char** name, int64_t shape[4],
                        int* ndim);

/* Replaces tf.get_variable / Saver.restore for one variable: copies `src_dev` (fp32, TF layout)
 * into the context, repacking it for the kernels (K-major padded conv_image matrices etc.).
 * Call again after an optimiser step. */
int n2nmn_set_weight(n2nmn_ctx* ctx, const char* name, const float* src_dev, const int64_t* shape,
                     int ndim, void* stream);

/* Replaces the placeholder feeds of `Modules(image_feat_grid, word_vecs, ...)`
 * (models_clevr/nmn3_modules.py:12-26): image_feat_grid [N,H,W,D], word_vecs [T,N,text_dim].
 * Both stay caller-owned and are read in place (VQA: an augmented copy with the two coordinate
 * channels of models_vqa/nmn3_modules.py:11-31 is built on `stream`). */
int n2nmn_bind_inputs(n2nmn_ctx* ctx, const float* feat_dev, const float* word_vecs_dev, int N,
                      int T, void* stream);

/* One batched module call = one `Modules.<X>Module(...)` invocation with leading dimension n
 * (models_clevr/nmn3_modules.py:60-495): in0/in1 attention maps [n,H,W,1] (NULL when the module
 * takes fewer), time_idx/batch_idx HOST int32 [n] (scheduling metadata), out = attention maps
 * [n,H,W,1] or answer scores [n,num_choices] depending on the op. n == 0 is legal (TF Fold's
 * zero-size batches, util/empty_safe_conv.py:9-11) and does nothing. */
int n2nmn_module_fwd(n2nmn_ctx* ctx, int op, const float* in0_dev, const float* in1_dev,
                     const int32_t* time_idx_host, const int32_t* batch_idx_host, int n,
                     float* out_dev, void* stream);

/* `Modules.SceneModule(time_idx, batch_idx, pos_val)` with an arbitrary constant
 * (models_clevr/nmn3_modules.py:60-72; n2nmn_module_fwd(N2NMN_OP_SCENE) uses the default 3). */
int n2nmn_scene_fwd(n2nmn_ctx* ctx, int n, float pos_val, float* out_dev, void* stream);

/* Replaces `Assembler.assemble` + `td.Compiler.build_feed_dict`
 * (models_clevr/nmn3_assembler.py:153-222, models_clevr/nmn3_model.py:146-159): parses the
 * Reverse-Polish layout tokens [T,N] (host int32, time-major) with the assembler's stack
 * discipline, writes validity_out[N] (1 = valid), and compiles the valid trees into launch tables.
 * `vocab_ops[v]` gives the n2nmn_op of token v, or -1 for <eos>. Host-only, no device sync; the
 * tables are uploaded by the first n2nmn_run_schedule that uses them. */
int n2nmn_compile_schedule(n2nmn_ctx* ctx, const int32_t* tokens_host, int T, int N,
                           const int32_t* vocab_ops, int num_vocab, uint8_t* validity_out,
                           n2nmn_sched** out);
/* n2nmn_compile_schedule without a context or a GPU (pure host logic; used by the CPU tests and
 * by callers that pre-compile layouts on loader threads). Only family/H/W/D/text_dim/map_dim/
 * kernel_size/num_choices/max_T of `cfg` are read. */
int n2nmn_compile_schedule_host(const n2nmn_config* cfg, const int32_t* tokens_host, int T, int N,
                                const int32_t* vocab_ops, int num_vocab, uint8_t* validity_out,
                                n2nmn_sched** out);
/* Diagnostic: average nanoseconds of one host layout compile (no GPU). */
double n2nmn_time_compile(const n2nmn_config* cfg, const int32_t* tokens_host, int T, int N,
                          const int32_t* vocab_ops, int num_vocab, int iters);
/* Same output as n2nmn_compile_schedule, from already-assembled expression trees (what
 * `compiler.build_feed_dict(expr_list)` receives, models_clevr/nmn3_model.py:158): nodes are listed
 * question by question in post-order (operands before their consumer); q_ptr[NQ+1] delimits the
 * questions (an empty range = INVALID_EXPR -> zero scores row); in0/in1 index into the node list
 * (-1 = none). batch_idx may differ from the question index. */
int n2nmn_compile_nodes(n2nmn_ctx* ctx, const int32_t* op, const int32_t* time_idx,
                        const int32_t* batch_idx, const int32_t* in0, const int32_t* in1,
                        int num_nodes, const int32_t* q_ptr, int num_questions,
                        n2nmn_sched** out);
int n2nmn_sched_destroy(n2nmn_sched* sched);

typedef struct n2nmn_sched_info {
  int32_t num_questions, num_valid, num_nodes, max_depth;
  int32_t num_text_nodes, num_find_nodes, num_proj_tiles, num_launches;
  int64_t algorithmic_bytes;   /* SURVEY.md §8(d)/App. D per-node figure summed over the batch */
  int64_t algorithmic_flops;
  /* §8(d) per-launch figures (distinct feature tiles counted once per launch, weights once):
   * [0] text projection kernel, [1] conv_image contraction kernel, [2] node kernel(s) */
  int64_t kernel_bytes[3];
  int64_t kernel_flops[3];
  /* training schedules: 2 * (B maps) * HW * Dk * map_dim, the weight-gradient contraction of the
   * feature-side layers (xtb_mma_kernel<FeatGradSrc>); 0 otherwise */
  int64_t bwd_gemm_flops;
} n2nmn_sched_info;
int n2nmn_sched_get_info(const n2nmn_sched* sched, n2nmn_sched_info* info);
/* Node table in (question, token) order: op, time_idx, batch_idx, depth, in0, in1 (node ids or
 * -1) as 6 int32 per node — lets callers map the attention arena back to expression nodes. */
int n2nmn_sched_get_nodes(const n2nmn_sched* sched, int32_t* out6, int capacity_nodes);

/* Replaces `sess.partial_run(h, scores, feed_dict=expr_feed)` (exp_clevr/eval_clevr.py:132):
 * evaluates every node of the compiled batch against the bound inputs and writes
 * scores_dev [N,num_choices] (rows of invalid layouts = 0, models_clevr/nmn3_model.py:144-155).
 * att_arena_dev, if not NULL, receives every node's attention map, [num_nodes,H,W] indexed by
 * node id (answer nodes' slots are left untouched). Asynchronous on `stream`. */
int n2nmn_run_schedule(n2nmn_ctx* ctx, n2nmn_sched* sched, float* scores_dev,
                       float* att_arena_dev, void* stream);

/* bind + compile + run in one call, for the per-batch loop of exp_clevr/eval_clevr.py:103-135 with
 * device-resident features (the reference keeps image_feat / word_vecs on the device between its
 * two partial_run calls). The compiled tables live in the context and are overwritten by the next
 * call. Asynchronous on `stream`; host cost is one layout compile + four enqueues. */
int n2nmn_forward_tokens(n2nmn_ctx* ctx, const float* feat_dev, const float* word_vecs_dev,
                         const int32_t* tokens_host, int T, int N, const int32_t* vocab_ops,
                         int num_vocab, float* scores_dev, uint8_t* validity_out, void* stream);

/* n2nmn_forward_tokens for `num_batches` (<= cfg.max_group) INDEPENDENT batches of identical shape
 * in one set of launches: batch i has its own feature grid feat_dev[i] [N,H,W,D], word vectors
 * word_vecs_dev[i] [T,N,text_dim], layout tokens tokens_host[i] [T,N] and writes scores_dev[i]
 * [N,num_choices] (validity_out may be NULL, or hold NULL entries). Results are those of
 * num_batches separate n2nmn_forward_tokens calls; the point is that a batch of 64 CLEVR
 * questions is ~4 us of tensor work, far too little to fill the SMs per launch, while the reference's
 * eval loop (exp_clevr/eval_clevr.py:103-135) offers an endless stream of independent batches. */
int n2nmn_forward_group(n2nmn_ctx* ctx, int num_batches, const float* const* feat_dev,
                        const float* const* word_vecs_dev, const int32_t* const* tokens_host,
                        int T, int N, const int32_t* vocab_ops, int num_vocab,
                        float* const* scores_dev, uint8_t* const* validity_out, void* stream);
/* The same with pinned HOST buffers (cf. n2nmn_forward_host_async): H2D copies, kernels and D2H
 * copies are only enqueued on `stream`. */
int n2nmn_forward_group_host_async(n2nmn_ctx* ctx, int num_batches,
                                   const float* const* feat_host,
                                   const float* const* word_vecs_host,
                                   const int32_t* const* tokens_host, int T, int N,
                                   const int32_t* vocab_ops, int num_vocab,
                                   float* const* scores_host, uint8_t* const* validity_out,
                                   void* stream);
/* cfg.max_group as clamped by n2nmn_create. */
int n2nmn_max_group(const n2nmn_ctx* ctx);

/* Statistics of the batch compiled by the last n2nmn_forward_tokens / n2nmn_forward_host. */
int n2nmn_last_step_info(const n2nmn_ctx* ctx, n2nmn_sched_info* info);

/* End-to-end convenience with HOST buffers (what exp_clevr/eval_clevr.py:103-135 does per batch):
 * H2D of features + word vectors, compile, run, D2H of scores; synchronises `stream` before
 * returning. Host buffers should be pinned for full PCIe rate. */
int n2nmn_forward_host(n2nmn_ctx* ctx, const float* feat_host, const float* word_vecs_host,
                       const int32_t* tokens_host, int T, int N, const int32_t* vocab_ops,
                       int num_vocab, float* scores_host, uint8_t* validity_out, void* stream);

/* Same, but returns without synchronising: the H2D copies, the kernels and the D2H copy of the
 * scores are only enqueued on `stream`; `scores_host` is valid once the stream has drained. Host
 * buffers must be pinned and must stay untouched until then. */
int n2nmn_forward_host_async(n2nmn_ctx* ctx, const float* feat_host, const float* word_vecs_host,
                             const int32_t* tokens_host, int T, int N, const int32_t* vocab_ops,
                             int num_vocab, float* scores_host, uint8_t* validity_out,
                             void* stream);

/* n2nmn_forward_group_host_async with the feature grids stored as IEEE fp16 on the host
 * (feat_host_f16[i]: [N][H][W][D] half, pinned): half the PCIe bytes of the fp32 feed, which is
 * what bounds the end-to-end rate (21.2 MB per CLEVR batch of 64). The grids are widened to fp32 on
 * the device (one pass over the staged copy) before the same kernels run; the contraction reads
 * 10-bit mantissas either way, so the outputs move by <= 1e-4 against the fp32 feed at the CLEVR
 * sizes (tests/test_gpu_parity.py), inside the 1e-3 bar. N*H*W*D must be a multiple of 8. No
 * reference counterpart: the reference feeds fp32 `image_feat_batch` (eval_clevr.py:120-123). */
int n2nmn_forward_group_host_f16_async(n2nmn_ctx* ctx, int num_batches,
                                       const uint16_t* const* feat_host_f16,
                                       const float* const* word_vecs_host,
                                       const int32_t* const* tokens_host, int T, int N,
                                       const int32_t* vocab_ops, int num_vocab,
                                       float* const* scores_host, uint8_t* const* validity_out,
                                       void* stream);

/* ---- several batches in flight -------------------------------------------------------------------
 * One worker thread per (context, stream) pair; n2nmn_pool_submit copies the token matrix into a
 * job for worker `slot` and returns. A worker takes up to n2nmn_max_group(ctx) queued jobs of
 * identical shape at a time and runs them as ONE n2nmn_forward_group (host_io == 0: device
 * pointers), n2nmn_forward_group_host_async (host_io == 1: pinned host pointers) or
 * n2nmn_forward_group_host_f16_async (host_io == 2: `feat` points to fp16 grids) on its stream:
 * dynamic batching of whatever the caller has queued, never waiting for more.
 * n2nmn_pool_wait blocks until every submitted batch has been ENQUEUED (not finished) and returns
 * the first error; `validity_out` arrays are valid after it. The contexts must outlive the pool
 * and must not be used directly while jobs are pending. No reference counterpart (the reference
 * evaluates one batch per session.run, exp_clevr/eval_clevr.py:96-133). */
typedef struct n2nmn_pool n2nmn_pool;
int n2nmn_pool_create(n2nmn_ctx** ctxs, void** streams, int num, const int32_t* vocab_ops,
                      int num_vocab, n2nmn_pool** out);
int n2nmn_pool_destroy(n2nmn_pool* pool);
int n2nmn_pool_size(const n2nmn_pool* pool);
int n2nmn_pool_submit(n2nmn_pool* pool, int slot, const float* feat, const float* word_vecs,
                      const int32_t* tokens_host, int T, int N, float* scores,
                      uint8_t* validity_out, int host_io);
/* n batches of identical shape in one call (arrays of n pointers; validity_out may be NULL),
 * dealt to the workers round-robin. Saves the per-batch cost of crossing the FFI. */
int n2nmn_pool_submit_many(n2nmn_pool* pool, int n, const float* const* feat,
                           const float* const* word_vecs, const int32_t* const* tokens_host, int T,
                           int N, float* const* scores, uint8_t* const* validity_out, int host_io);
int n2nmn_pool_wait(n2nmn_pool* pool);
/* How the workers batched the jobs so far: number of n2nmn_forward_group calls and of jobs. */
int n2nmn_pool_group_stats(const n2nmn_pool* pool, int64_t* groups, int64_t* jobs);
const char* n2nmn_pool_last_error(void);


/* ---- training step (exp_clevr/train_clevr_rl_gt_layout.py:108-139) -------------------------------
 * Weights, gradients and the Adam moments live in caller-owned flat fp32 device buffers of
 * n2nmn_flat_size() floats: the variables of n2nmn_variable_info() in order, each in its TF shape
 * at n2nmn_flat_offset(). */
int64_t n2nmn_flat_size(const n2nmn_ctx* ctx);
int n2nmn_flat_offset(const n2nmn_ctx* ctx, int index, int64_t* offset, int64_t* count);
/* n2nmn_set_weight for every variable from one flat buffer. */
int n2nmn_load_flat_weights(n2nmn_ctx* ctx, const float* wflat_dev, void* stream);
/* Forward + backward of one batch: scores_dev [N,C]; loss_dev[0] = Σ_i loss_i with
 * loss_i = softmax cross-entropy for valid layouts and `invalid_expr_loss` otherwise
 * (:108-114), loss_dev[1+i] = loss_i; gflat_dev = d(mean_i loss_i)/d(variables) (overwritten);
 * dword_dev (optional) = d(mean loss)/d(word_vecs) [T,N,text_dim], the gradient handed on to the
 * seq2seq. labels_host int32 [N]. Asynchronous on `stream`. */
int n2nmn_train_backward(n2nmn_ctx* ctx, const float* feat_dev, const float* word_vecs_dev,
                         const int32_t* tokens_host, int T, int N, const int32_t* vocab_ops,
                         int num_vocab, const int32_t* labels_host, float invalid_expr_loss,
                         float* scores_dev, float* gflat_dev, float* dword_dev, float* loss_dev,
                         uint8_t* validity_out, void* stream);
/* n2nmn_train_backward with the answer prior of the VQA training scripts
 * (exp_vqa/train_vqa_rl_gt_layout.py:101-142: scores = scores_nmn + scores_qpn).
 *   score_prior_dev (optional) [N,C]: logits added to the module scores before the loss, e.g. the
 *     output of the caller's question-prior net; scores_dev then holds the sum.
 *   dscores_dev (optional) [N,C]: d(mean loss)/d(scores), the gradient to backpropagate into that
 *     net. Scaled by n2nmn_set_grad_scale like dword_dev, because it is not all-reduced.
 * Loss rule by family: CLEVR / SHAPES charge `invalid_expr_loss` to an invalid layout (its
 * dscores row is zero); VQA takes the softmax cross-entropy on EVERY row, an invalid layout's
 * module scores being zeros (its row is CE(prior, label)), and `invalid_expr_loss` is not used.
 * The VQA family trains at any map_dim; CLEVR / SHAPES (conv Transform) need map_dim <= 512.
 * Batches whose nodes, B maps (feature-side layer uses) or stored maps exceed what the context
 * was created for fail with N2NMN_ERR_CAPACITY. n2nmn_train_backward(...) is
 * n2nmn_train_backward_ex(..., NULL, NULL, stream). */
int n2nmn_train_backward_ex(n2nmn_ctx* ctx, const float* feat_dev, const float* word_vecs_dev,
                            const int32_t* tokens_host, int T, int N, const int32_t* vocab_ops,
                            int num_vocab, const int32_t* labels_host, float invalid_expr_loss,
                            float* scores_dev, float* gflat_dev, float* dword_dev, float* loss_dev,
                            uint8_t* validity_out, const float* score_prior_dev, float* dscores_dev,
                            void* stream);
/* g += weight_decay * w on the ".../weights" variables (l2_reg, nmn3_model.py:163-166), per-tensor
 * tf.clip_by_norm(g, max_norm) (:137-138), Adam step `step` (1-based, :132), then the updated
 * weights are re-packed into the context. In data-parallel training the caller all-reduces
 * gflat_dev (NCCL) between n2nmn_train_backward and this call. */
int n2nmn_adam_step(n2nmn_ctx* ctx, float* wflat_dev, float* gflat_dev, float* m_dev, float* v_dev,
                    int step, float lr, float beta1, float beta2, float eps, float max_norm,
                    float weight_decay, void* stream);

/* The rest of the policy-search step after the (optional) all-reduce, with nothing read back by
 * the host (exp_clevr/train_clevr_rl_gt_layout.py:119-139):
 *   avg_sample_loss = loss_sum / (N*world); coeff_i = (loss_i - baseline) / (N*world) (the
 *   stop_gradient factor of the policy-gradient loss, :123-124); pg = Σ coeff_i*log_seq_prob_i;
 *   baseline EMA (:120-122); g = g/world + weight_decay*w; l2_reg; per-tensor clip; Adam; re-pack.
 * loss_sum_dev: ONE float, Σ of the per-sample losses over all ranks (loss_dev[0] of
 * n2nmn_train_backward, summed by the all-reduce); per_sample_dev [N] this rank's losses
 * (loss_dev + 1); log_seq_prob_dev [N] or NULL; state_in/out_dev: 4 floats {baseline,
 * avg_sample_loss, policy_gradient_loss, l2_reg} (only [0] of state_in is read; in and out may
 * alias); coeff_dev [N] or NULL. */
int n2nmn_train_finish(n2nmn_ctx* ctx, float* wflat_dev, float* gflat_dev, float* m_dev,
                       float* v_dev, int step, float lr, float beta1, float beta2, float eps,
                       float max_norm, float weight_decay, const float* loss_sum_dev,
                       const float* per_sample_dev, const float* log_seq_prob_dev, int N, int world,
                       float baseline_decay, const float* state_in_dev, float* state_out_dev,
                       float* coeff_dev, void* stream);
/* Factor applied to d_word_vecs by n2nmn_train_backward (the one gradient that is not
 * all-reduced): 1/world_size in data-parallel training. Default 1. */
int n2nmn_set_grad_scale(n2nmn_ctx* ctx, float scale);

/* CTAs per question in the layout-executor kernel: 1, 2, 4 or 8 thread-block clusters; 0 (the
 * default) picks from the batch size so that one batch alone spreads over the SMs (lowest latency
 * of a single batch). Callers that keep several batches in flight on different streams get more
 * throughput from smaller clusters. Tuning only: results are identical. No reference counterpart
 * (the reference executor is TensorFlow Fold's scheduler, models_clevr/nmn3_model.py:118-133). */
int n2nmn_set_tree_cluster(n2nmn_ctx* ctx, int ctas_per_question);

/* Cap of the persistent grid of the conv_image contraction kernel; 0 (the default) = one CTA per
 * SM, which gives the shortest kernel for a single batch. With many batches in flight a narrower
 * grid (each CTA then walks several tiles, its epilogue overlapping the next tile's MMAs) leaves
 * the other SMs to the other batches' kernels and raises the throughput. Tuning only: results are
 * identical. */
int n2nmn_set_proj_ctas(n2nmn_ctx* ctx, int max_ctas);

/* Retired tuning knob of the round-1 text-projection kernel (CTAs per group of 8 text rows). The
 * text projection is a tiled GEMM now (64 rows x 32 columns per CTA, csrc/text_proj.cuh); the value
 * is accepted and ignored, the entry point stays for ABI-2 callers. */
int n2nmn_set_text_ctas_per_group(n2nmn_ctx* ctx, int n);

/* CRC-32C (Castagnoli) of a host buffer, continuing from `crc` (0 to start): the checksum of the
 * TensorFlow checkpoint format (tf.train.Saver, exp_clevr/eval_clevr.py:90-91) that
 * n2nmn_b200/checkpoint.py reads and writes. Host only. */
uint32_t n2nmn_crc32c(const void* data, size_t n, uint32_t crc);

/* Per-launch device time of the last n2nmn_run_schedule in microseconds (CUDA events recorded
 * around every launch when enabled). names/us arrays of length >= capacity. */
int n2nmn_set_profiling(n2nmn_ctx* ctx, int enabled);
int n2nmn_get_launch_times(n2nmn_ctx* ctx, const char** names, float* us, int capacity);
/* Count of kernel launches issued by this ctx since creation. */
int64_t n2nmn_launch_count(const n2nmn_ctx* ctx);

/* ---- (f1) attentional seq2seq layout generator --------------------------------------------
 * Replaces `AttentionSeq2Seq` (models_clevr/nmn3_netgen_att.py:46-322; the VQA / SHAPES copies
 * are the same code): greedy decoding under the Assembler's validity masks, `decoder_sampling`
 * (n2nmn_seq2seq_set_sampling) or teacher forcing, with the training scripts' LSTM dropout
 * (`encoder_dropout` / `decoder_dropout`, n2nmn_seq2seq_set_dropout) or without it: the encoder LSTM
 * stack under dynamic_rnn (:73-120) and the raw_rnn attention decoder (:122-322). Training: a recording
 * forward (n2nmn_seq2seq_set_record), n2nmn_seq2seq_backward into a flat gradient buffer and
 * n2nmn_seq2seq_adam_step (DESIGN.md §4c). */
typedef struct n2nmn_seq2seq n2nmn_seq2seq;
typedef struct n2nmn_seq2seq_config {
  int32_t abi_version;     /* N2NMN_ABI_VERSION */
  int32_t num_vocab_txt;   /* nmn3_netgen_att.py:48-52 constructor arguments */
  int32_t embed_dim_txt;
  int32_t num_vocab_nmn;   /* <= 64 */
  int32_t embed_dim_nmn;
  int32_t lstm_dim;        /* multiple of 8 */
  int32_t num_layers;      /* <= 4 */
  int32_t T_encoder;       /* capacity, <= 128 */
  int32_t T_decoder;       /* decoding steps (fixed, as in the reference) */
  int32_t max_batch;
  int32_t device;
  int32_t flags;           /* N2NMN_SEQ2SEQ_FLAG_* */
} n2nmn_seq2seq_config;
/* LSTM / attention-query / h-transform products as ONE TF32 pass (operands rounded to 10-bit
 * mantissas, fp32 accumulate) instead of the default error-compensated three passes (fp32
 * parity). ~1e-3-level differences in probabilities; a decoded token can differ from the fp32
 * result when two scores are within that distance. */
#define N2NMN_SEQ2SEQ_FLAG_TF32 1

int n2nmn_seq2seq_create(const n2nmn_seq2seq_config* cfg, n2nmn_seq2seq** out);
int n2nmn_seq2seq_destroy(n2nmn_seq2seq* s);
/* Variables under the reference's `encoder_decoder/` scope, names relative to it, e.g.
 * "encoder/lstm/multi_rnn_cell/cell_0/basic_lstm_cell/weights" (TF 1.0 BasicLSTMCell:
 * [input+units, 4*units], gate order i, j, f, o). */
int n2nmn_seq2seq_num_variables(const n2nmn_seq2seq* s);
int n2nmn_seq2seq_variable_info(const n2nmn_seq2seq* s, int index, const char** name,
                                int64_t shape[4], int* ndim);
/* src_dev: device pointer, TF layout (what tf.train.Saver stores). */
int n2nmn_seq2seq_set_weight(n2nmn_seq2seq* s, const char* name, const float* src_dev,
                             const int64_t* shape, int ndim, void* stream);
/* The Assembler's decoding-state tables (models_clevr/nmn3_assembler.py:150-222), HOST int32:
 * P [V][3], W [3][V][4], b [V][4] — `_get_valid_tokens` (nmn3_netgen_att.py:8-11) and
 * `_update_decoding_state` (:13-15). Synchronises the stream. */
int n2nmn_seq2seq_set_assembler(n2nmn_seq2seq* s, const int32_t* P, const int32_t* W,
                                const int32_t* b, void* stream);
/* One batch, everything device-resident and time-major as in the reference:
 *   input_seq_dev [T_enc][N] int32, seq_len_dev [N] int32,
 *   gt_layout_dev [T_decoder][N] int32 or NULL (NULL = greedy; non-NULL = `use_gt_layout`),
 *   tokens_dev [T_decoder][N] int32        -> predicted_tokens (:307)
 *   token_probs_dev [T_decoder][N]         -> token_probs (:308); Σ_t log = log_seq_prob
 *   neg_entropy_dev [N]                    -> neg_entropy (:309)
 *   word_vecs_dev [T_decoder][N][embed_dim_txt] -> word_vecs (:312)
 *   atts_dev [T_decoder][T_enc][N] or NULL -> atts (:311)
 * All work is enqueued on `stream`. */
int n2nmn_seq2seq_forward(n2nmn_seq2seq* s, const int32_t* input_seq_dev,
                          const int32_t* seq_len_dev, int T_enc, int N,
                          const int32_t* gt_layout_dev, int32_t* tokens_dev,
                          float* token_probs_dev, float* neg_entropy_dev, float* word_vecs_dev,
                          float* atts_dev, void* stream);
/* n2nmn_seq2seq_forward plus the encoder's final state (models_vqa/nmn3_model.py passes it to the
 * question-prior net): encoder_states_dev [num_layers][2][N][lstm_dim] receives (c, h) of every
 * layer, LSTMStateTuple order, i.e. dynamic_rnn's final state — each question's state at its own
 * length, carried to T_enc - 1 (nmn3_netgen_att.py:95-99), the state the decoder starts from.
 * NULL = n2nmn_seq2seq_forward exactly. Copies only: the kernel launches are the same either way,
 * (T_enc + num_layers - 1) + num_layers·T_decoder + 2·T_decoder + 3 per call. */
int n2nmn_seq2seq_forward_ex(n2nmn_seq2seq* s, const int32_t* input_seq_dev,
                             const int32_t* seq_len_dev, int T_enc, int N,
                             const int32_t* gt_layout_dev, int32_t* tokens_dev,
                             float* token_probs_dev, float* neg_entropy_dev, float* word_vecs_dev,
                             float* atts_dev, void* stream, float* encoder_states_dev);
/* `decoder_sampling=True` (nmn3_netgen_att.py:234-256) for the following forward calls:
 * uniforms_dev [T_decoder][N] fp32 in [0,1) (N = the forward call's N; must stay valid until the
 * forward's work has run), one number per decoding step and question. The token is drawn from
 * softmax(token_scores - 50·invalid) by inverse CDF in vocabulary order (`tf.multinomial`'s
 * distribution; TF's generator itself is not reproducible outside TF) and replaced by the greedy
 * token if it is invalid (:241-256). NULL = back to greedy decoding. gt_layout_dev still wins. */
int n2nmn_seq2seq_set_sampling(n2nmn_seq2seq* s, const float* uniforms_dev);
/* `encoder_dropout` / `decoder_dropout` (nmn3_netgen_att.py:17-44, :91, :303) for the following
 * forward calls: DropoutWrapper(output_keep_prob=0.5) on every layer but the top one. Only the
 * output a layer hands to the layer above is dropped; its state (c, h), the encoder outputs, the
 * attention and the token scores see undropped values, and with num_layers == 1 nothing changes.
 * tf.nn.dropout's rule on given uniform numbers u in [0,1): an element is kept iff
 * floor(0.5 + u) = 1 in fp32 (u >= 0.5 on torch.rand's grid) and a kept element is 2x; TF's
 * generator itself is not reproducible outside TF. Device fp32 uniforms, indexed by (step, layer):
 *   enc_uniforms_dev [T_enc][num_layers-1][N][lstm_dim], dec_uniforms_dev
 *   [T_decoder][num_layers-1][N][lstm_dim]
 * with the forward call's T_enc and N; they must stay valid until the forward's work has run (a
 * recording forward keeps the keep-masks, so the backward does not read them). NULL = no dropout
 * on that side. Same launches as without dropout. */
int n2nmn_seq2seq_set_dropout(n2nmn_seq2seq* s, const float* enc_uniforms_dev,
                              const float* dec_uniforms_dev);
int64_t n2nmn_seq2seq_launch_count(const n2nmn_seq2seq* s);
/* Recording switch for the following forward calls (default off). While on, the forward also
 * keeps what n2nmn_seq2seq_backward needs: every cell's gates and state, every decoding step's
 * attention query, context vector, token scores, validity mask and token, and a copy of the
 * inputs. The workspace (~100 MB at N=64, T_enc=45, T_dec=10, lstm_dim=512, 2 layers) is
 * allocated on first use. The outputs are bit-identical with and without recording. */
int n2nmn_seq2seq_set_record(n2nmn_seq2seq* s, int on);
/* Flat layout of the variables (creation order, n2nmn_seq2seq_variable_info), each in its TF shape
 * and layout at a 16-byte aligned offset: the gradient, weight and Adam moment buffers. */
int64_t n2nmn_seq2seq_flat_size(const n2nmn_seq2seq* s);
int n2nmn_seq2seq_flat_offset(const n2nmn_seq2seq* s, int index, int64_t* offset, int64_t* count);
/* Gradient of the generator's variables, after a recording forward of this batch, as TF 1.0
 * differentiates nmn3_netgen_att.py's graph. Each upstream gradient may be NULL (= zero):
 *   d_log_seq_prob_dev [N]              d total / d log_seq_prob (Σ_t log token_probs, nmn3_model.py:46)
 *   d_neg_entropy_dev  [N]              d total / d neg_entropy
 *   d_word_vecs_dev    [T_dec][N][E_txt] d total / d word_vecs
 * with N the recorded forward's batch. No gradient flows through the validity masks, the decoding
 * state or the chosen tokens. grad_flat_dev (n2nmn_seq2seq_flat_size floats) is overwritten.
 * N2NMN_ERR_STATE if the last forward did not record or a weight was set since. All work is
 * enqueued on `stream`; nothing is read back. */
int n2nmn_seq2seq_backward(n2nmn_seq2seq* s, const float* d_log_seq_prob_dev,
                           const float* d_neg_entropy_dev, const float* d_word_vecs_dev,
                           float* grad_flat_dev, void* stream);
/* n2nmn_seq2seq_backward plus a fourth upstream gradient, d_encoder_states_dev
 * [num_layers][2][N][lstm_dim] (dc, dh): d total / d encoder_states of n2nmn_seq2seq_forward_ex
 * (e.g. from the question-prior net). It is added to the gradient of the encoder's final state that
 * the decoder passes back and flows on through the carried rows in the same way. NULL = zero,
 * i.e. n2nmn_seq2seq_backward exactly; otherwise one more launch. Same N2NMN_ERR_STATE rules. */
int n2nmn_seq2seq_backward_ex(n2nmn_seq2seq* s, const float* d_log_seq_prob_dev,
                              const float* d_neg_entropy_dev, const float* d_word_vecs_dev,
                              float* grad_flat_dev, void* stream,
                              const float* d_encoder_states_dev);
/* All variables from / to one flat buffer (device, n2nmn_seq2seq_flat_offset layout). Loading
 * marks the derived weights for re-preparation at the next forward. */
int n2nmn_seq2seq_load_flat_weights(n2nmn_seq2seq* s, const float* wflat_dev, void* stream);
int n2nmn_seq2seq_get_flat_weights(const n2nmn_seq2seq* s, float* wflat_dev, void* stream);
/* One optimiser step over the flat buffers, as n2nmn_adam_step: g += weight_decay·w on every
 * ".../weights" variable (the reference's l2_reg, nmn3_model.py:161-166), tf.clip_by_norm per
 * tensor to max_norm, Adam with TF's lr_t; then the context takes the new weights
 * (n2nmn_seq2seq_load_flat_weights). gflat_dev is modified (decay term). */
int n2nmn_seq2seq_adam_step(n2nmn_seq2seq* s, float* wflat_dev, float* gflat_dev, float* m_dev,
                            float* v_dev, int step, float lr, float beta1, float beta2, float eps,
                            float max_norm, float weight_decay, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* N2NMN_B200_H_ */
