"""Policy-search train step of the module network (exp_clevr/train_clevr_rl_gt_layout.py:101-139).

    loss_i   = softmax_cross_entropy(scores_i, label_i)  if layout i is valid else 0.5      (:108-114)
    avg      = mean_i loss_i                                                               (:119)
    baseline += (1 - 0.99) * (avg - baseline)             (EMA, not trained)               (:120-122)
    pg       = mean_i stop_gradient(loss_i - baseline) * log_seq_prob_i                    (:123-124)
    total    = pg + avg + 0.005 * entropy_reg + 5e-6 * l2_reg                              (:126-129)
    Adam(1e-4) on per-tensor clip_by_norm(grad, 10)                                        (:132-139)

VQA (exp_vqa/train_vqa{,2}_{gt,rl_gt}_layout.py:101-142) differs in two places: the scores are
`scores_nmn + scores_qpn`, the logits of a question-prior net the caller owns (`score_prior`;
`d_scores` comes back for its backward pass), and loss_i is the cross-entropy on EVERY row (an
invalid layout's module scores are zeros, so its loss is CE(prior, label)): `invalid_expr_loss`
only seeds the baseline. The VQA scripts use weight_decay 0 and clip at 10 (rl) or not at all (gt):
set them on the trainer.

The module network receives gradient only through `avg` and the l2 term; `pg` and the entropy term
reach the seq2seq layout generator, which is off the hot path: this class returns what that
generator needs (d total/d word_vecs and the per-sample REINFORCE coefficients) instead of
differentiating it. Data parallel: every rank holds a shard of the questions; ONE all-reduce over
the flat gradient buffer (+ the loss sum riding in its last element) per step (NCCL via
torch.distributed), then clip + Adam replicated on every rank.

Nothing in a step is read back by the host: the scalar bookkeeping (mean loss, REINFORCE
coefficients, baseline EMA, l2_reg) runs in `n2nmn_train_finish` on the device. `train_step`
returns device tensors with `sync=False` (views into a ring of `RING` result slots, valid for the
next RING-1 steps) and Python floats — one 16-byte read at the end of the step, what the
reference's `sess.run` fetches (train_clevr_rl_gt_layout.py:206-213) — with the default
`sync=True`.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib


class ModuleNetTrainer:
    RING = 64

    def __init__(self, executor, lr=1e-4, beta1=0.9, beta2=0.999, eps=1e-8, max_grad_l2_norm=10.0,
                 weight_decay=5e-6, baseline_decay=0.99, invalid_expr_loss=0.5,
                 lambda_entropy=0.005, process_group=None):
        self.ex = executor
        self.m = executor.modules
        self._lib = executor._lib
        self.hyper = dict(lr=lr, beta1=beta1, beta2=beta2, eps=eps, max_norm=max_grad_l2_norm,
                          weight_decay=weight_decay)
        self.baseline_decay = baseline_decay
        self.invalid_expr_loss = invalid_expr_loss
        self.lambda_entropy = lambda_entropy
        self.step = 0
        self.pg = process_group
        h = self.m._h
        self.flat_size = int(self._lib.n2nmn_flat_size(h))
        dev = self.m.device
        # flat buffers; the last element of `g` carries the loss sum through the all-reduce
        self.w = torch.zeros(self.flat_size, dtype=torch.float32, device=dev)
        # [gradients | Σ loss | per-sample losses]: the loss kernel writes the last two parts, the
        # all-reduce covers the first two (the local per-sample losses stay local)
        self._gbuf = torch.zeros(self.flat_size + 1 + self.m.max_batch, dtype=torch.float32,
                                 device=dev)
        self.g = self._gbuf[:self.flat_size + 1]
        self._loss = self._gbuf[self.flat_size:]
        self.m1 = torch.zeros(self.flat_size, dtype=torch.float32, device=dev)
        self.m2 = torch.zeros(self.flat_size, dtype=torch.float32, device=dev)
        # ring of per-step results: {baseline, avg_sample_loss, policy_gradient_loss, l2_reg}
        self._state = torch.zeros((self.RING, 4), dtype=torch.float32, device=dev)
        self._state[:, 0] = float(invalid_expr_loss)    # tf.Variable(invalid_expr_loss) (:120)
        self._coeff = torch.zeros((self.RING, self.m.max_batch), dtype=torch.float32, device=dev)
        self._slot = 0
        self._world_set = 1
        self.layout = {}
        nvar = self._lib.n2nmn_num_variables(h)
        for i in range(nvar):
            name = C.c_char_p()
            shape = (C.c_int64 * 4)()
            nd = C.c_int()
            _lib.check(self._lib.n2nmn_variable_info(h, i, C.byref(name), shape, C.byref(nd)))
            off, cnt = C.c_int64(), C.c_int64()
            _lib.check(self._lib.n2nmn_flat_offset(h, i, C.byref(off), C.byref(cnt)))
            self.layout[name.value.decode()] = (off.value, cnt.value, tuple(shape[:nd.value]))
        for name, t in self.m.get_weights().items():
            off, cnt, shp = self.layout[name]
            self.w[off:off + cnt] = t.reshape(-1)
        # the context is re-packed from self.w after every step: hand out those values, not the
        # tensors cached by set_weights() at construction time (replicas, checkpoints)
        self.m._weights_source = self.weights
        self._decay_mask = torch.zeros(self.flat_size, dtype=torch.float32, device=dev)
        for name, (off, cnt, _) in self.layout.items():
            if name.endswith('/weights'):
                self._decay_mask[off:off + cnt] = 1.0

    # -- views ------------------------------------------------------------------------------------
    def weights(self):
        return {n: self.w[o:o + c].reshape(s) for n, (o, c, s) in self.layout.items()}

    @property
    def baseline(self):
        """The EMA baseline after the last step (reads the device)."""
        return float(self._state[self._slot, 0])

    def l2_reg(self):
        """Σ tf.nn.l2_loss over the '.../weights' variables (nmn3_model.py:163-166)."""
        return float(0.5 * (self.w * self.w * self._decay_mask).sum())

    def grads(self):
        return {n: self.g[o:o + c].reshape(s) for n, (o, c, s) in self.layout.items()}

    # -- one step ---------------------------------------------------------------------------------
    def forward_backward(self, image_feat_grid, word_vecs, layout_tokens, labels,
                         want_dword=True, score_prior=None):
        """Forward + backward of this rank's shard. Fills self.g (gradient of the LOCAL mean loss)
        and returns (scores, validity, per_sample_loss tensor, d_word_vecs or None).
        score_prior: optional [N, num_choices] CUDA logits added to the module scores before the
        loss (VQA's question-prior net); the returned scores are then the sum, and a fifth
        element d_scores = d(mean loss)/d(scores) [N, num_choices] follows, scaled by 1/world
        like d_word_vecs."""
        m = self.m
        tok = np.ascontiguousarray(layout_tokens, dtype=np.int32)
        T, N = tok.shape
        lab = np.ascontiguousarray(labels, dtype=np.int32)
        assert lab.shape == (N,)
        nc = self.ex.num_choices
        scores = torch.empty((N, nc), dtype=torch.float32, device=m.device)
        dword = torch.empty((T, N, m.text_dim), dtype=torch.float32, device=m.device) \
            if want_dword else None
        prior = dscores = None
        if score_prior is not None:
            prior = score_prior.to(m.device, torch.float32).contiguous()
            if tuple(prior.shape) != (N, nc):
                raise ValueError('score_prior must be [N, num_choices] = [%d, %d], got %r'
                                 % (N, nc, tuple(prior.shape)))
            dscores = torch.empty((N, nc), dtype=torch.float32, device=m.device)
        validity = np.empty(N, np.uint8)
        m.image_feat_grid, m.word_vecs, m.N, m.T = image_feat_grid, word_vecs, N, T
        _lib.check(self._lib.n2nmn_train_backward_ex(
            m._h, image_feat_grid.data_ptr(), word_vecs.data_ptr(), tok.ctypes.data, T, N,
            self.ex._vocab_ptr, len(self.ex.vocab_ops), lab.ctypes.data,
            C.c_float(self.invalid_expr_loss), scores.data_ptr(), self.g.data_ptr(),
            dword.data_ptr() if dword is not None else None, self._loss.data_ptr(),
            validity.ctypes.data, prior.data_ptr() if prior is not None else None,
            dscores.data_ptr() if dscores is not None else None,
            torch.cuda.current_stream(m.device).cuda_stream))
        if prior is not None:
            return scores, validity.view(bool), self._loss[1:1 + N], dword, dscores
        return scores, validity.view(bool), self._loss[1:1 + N], dword

    def train_step(self, image_feat_grid, word_vecs, layout_tokens, labels, log_seq_prob=None,
                   entropy_reg=0.0, sync=True, score_prior=None):
        """One optimiser step. Returns a dict with the reference's logged quantities; with a
        score_prior (see forward_backward) it also carries 'd_scores'."""
        import torch.distributed as dist
        world = 1
        if dist.is_available() and dist.is_initialized() and dist.get_world_size(self.pg) > 1:
            world = dist.get_world_size(self.pg)
        if world != self._world_set:       # d_word_vecs is the one gradient no all-reduce averages
            _lib.check(self._lib.n2nmn_set_grad_scale(self.m._h, C.c_float(1.0 / world)))
            self._world_set = world
        res = self.forward_backward(image_feat_grid, word_vecs, layout_tokens, labels,
                                    score_prior=score_prior)
        scores, validity, per_sample, dword = res[:4]
        N = scores.shape[0]
        if world > 1:
            dist.all_reduce(self.g, op=dist.ReduceOp.SUM, group=self.pg)   # the ONE collective
        prev, cur = self._slot, (self._slot + 1) % self.RING
        self._slot = cur
        self.step += 1
        hp = self.hyper
        lsp = None
        if log_seq_prob is not None:
            lsp = log_seq_prob.to(self.m.device, torch.float32).contiguous()
        _lib.check(self._lib.n2nmn_train_finish(
            self.m._h, self.w.data_ptr(), self.g.data_ptr(), self.m1.data_ptr(),
            self.m2.data_ptr(), self.step, hp['lr'], hp['beta1'], hp['beta2'], hp['eps'],
            hp['max_norm'], hp['weight_decay'], self._loss.data_ptr(),
            self._loss.data_ptr() + 4, lsp.data_ptr() if lsp is not None else None, N, world,
            C.c_float(self.baseline_decay), self._state[prev].data_ptr(),
            self._state[cur].data_ptr(), self._coeff[cur].data_ptr(),
            torch.cuda.current_stream(self.m.device).cuda_stream))
        st = self._state[cur]
        out = {'scores': scores, 'validity': validity, 'd_word_vecs': dword,
               'reinforce_coeff': self._coeff[cur, :N]}
        if score_prior is not None:
            out['d_scores'] = res[4]
        if sync:
            base, avg, pg, l2 = st.tolist()                      # the step's only host read
        else:
            base, avg, pg, l2 = st[0], st[1], st[2], st[3]
        out.update({'avg_sample_loss': avg, 'policy_gradient_loss': pg, 'baseline': base,
                    'l2_reg': l2})
        if sync:      # (:126-129); with sync=False the caller combines the four device scalars
            out['total_loss'] = (pg + avg + self.lambda_entropy * entropy_reg +
                                 hp['weight_decay'] * l2)
        return out


class LayoutGeneratorTrainer:
    """Clip + Adam for the layout generator's variables (`seq2seq.AttentionSeq2Seq`), the
    counterpart of `ModuleNetTrainer` for the other half of the reference's graph. It holds the
    flat weights `w`, the gradient `g` and the Adam moments; `step()` runs the generator's backward
    pass on its last recording forward and one optimiser step, all on the device.

    The reference's two losses map onto the upstream gradients as follows (N = batch size):
      gt-layout (exp_clevr/train_clevr_gt_layout.py:104-124): seq_likelihood_loss =
        mean(-log_seq_prob) -> d_log_seq_prob = -1/N, plus d_word_vecs from
        `ModuleNetTrainer.train_step(...)['d_word_vecs']`;
      policy search (exp_clevr/train_clevr_rl_gt_layout.py:108-139): d_log_seq_prob =
        `train_step(...)['reinforce_coeff']`, d_neg_entropy = lambda_entropy / N, plus
        d_word_vecs.
    weight_decay applies to every `.../weights` variable (the reference's l2_reg,
    nmn3_model.py:161-166), not to the embeddings, go_embedding, v or the biases.
    VQA (exp_vqa/train_vqa*.py, use_qpn=True) adds the question-prior net's input gradient:
    d_encoder_states, the gradient of `generator.encoder_states` (see `AttentionSeq2Seq.backward`)."""

    def __init__(self, generator, lr=1e-4, beta1=0.9, beta2=0.999, eps=1e-8, max_grad_l2_norm=10.0,
                 weight_decay=5e-6):
        self.gen = generator
        self._lib = _lib.lib()
        dev = generator.device
        self.flat_size = generator.flat_layout()[0]
        self.w = generator.get_flat_weights()
        self.g = torch.zeros(self.flat_size, dtype=torch.float32, device=dev)
        self.m1 = torch.zeros(self.flat_size, dtype=torch.float32, device=dev)
        self.m2 = torch.zeros(self.flat_size, dtype=torch.float32, device=dev)
        self.step_count = 0
        self.hyper = dict(lr=lr, beta1=beta1, beta2=beta2, eps=eps, max_norm=max_grad_l2_norm,
                          weight_decay=weight_decay)

    def grads(self):
        return self.gen._views(self.g)

    def step(self, d_log_seq_prob=None, d_neg_entropy=None, d_word_vecs=None,
             d_encoder_states=None):
        """Backward pass of the generator's last `forward(..., record=True)`, then clip + Adam; the
        generator takes the new weights (its next forward re-derives its packed copies)."""
        self.gen.backward(d_log_seq_prob, d_neg_entropy, d_word_vecs, out=self.g,
                          d_encoder_states=d_encoder_states)
        self.step_count += 1
        hp = self.hyper
        dev = self.gen.device
        with torch.cuda.device(dev):
            _lib.check(self._lib.n2nmn_seq2seq_adam_step(
                self.gen._h, self.w.data_ptr(), self.g.data_ptr(), self.m1.data_ptr(),
                self.m2.data_ptr(), self.step_count, hp['lr'], hp['beta1'], hp['beta2'], hp['eps'],
                hp['max_norm'], hp['weight_decay'], torch.cuda.current_stream(dev).cuda_stream))
        self.gen._recorded_N = None
