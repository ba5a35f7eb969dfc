"""CPU ORACLE (test infrastructure, not product code): float64 torch-autograd restatement of the
layout generator ``AttentionSeq2Seq`` (models_clevr/nmn3_netgen_att.py:46-322), the forward pass of
``seq2seq_oracle.py`` written so that autograd yields TF 1.0's registered gradients of the
reference graph:

* no gradient through the validity masks, the decoding state or the chosen / sampled tokens
  (``stop_gradient``, :8-15); under teacher forcing every token is valid (:230-233);
* ``neg_entropy = Σ p·log(max(1e-5, p + 1 - valid))`` (:283-285) with TF's Maximum gradient: the
  second argument receives the gradient only where it is strictly larger than 1e-5
  (``torch.maximum`` would split ties);
* the decoder's inputs are differentiable lookups of ``go_embedding`` and
  ``decoder/embedding_mat`` (:202, :293); the encoder's final state is the decoder's initial state;
* dynamic_rnn past the sequence end carries the state and outputs zeros (:95-99).

Pinned on the CPU against ``seq2seq_oracle.py`` (tokens equal, values within 1e-6) and against
central finite differences (tests/test_seq2seq_oracle_torch.py).

``run(...)`` returns the outputs and, given upstream gradients, the gradient of every variable.
Weights: dict keyed by the TF variable names relative to ``encoder_decoder/``.
"""
from __future__ import annotations

import numpy as np
import torch


def _cell(x, c, h, w, b):
    g = torch.cat([x, h], dim=1) @ w + b
    i, j, f, o = torch.split(g, g.shape[1] // 4, dim=1)
    c2 = c * torch.sigmoid(f + 1.0) + torch.sigmoid(i) * torch.tanh(j)
    return c2, torch.tanh(c2) * torch.sigmoid(o)


def _tf_max_const(a, y):
    """max(a, y) for a constant a with TF's Maximum gradient: y gets it only where y > a."""
    return torch.where(y > a, y, torch.full_like(y, a))


def forward(w, input_seq, seq_length, T_dec, num_layers, P, W, b, use_gt_layout=False,
            gt_layout=None, sample_uniforms=None, tokens=None):
    """w: {name: float64 tensor (requires_grad as wanted)}. tokens [T_dec, N] (optional) overrides
    the chosen tokens (greedy / sampled) — for comparing gradients with a decoder whose choice is
    known; validity is still computed from the decoding state. Returns predicted_tokens (numpy),
    token_probs [T_dec, N], neg_entropy [N], word_vecs [T_dec, N, E], atts [T_dec, T, N]."""
    input_seq = np.asarray(input_seq)
    seq_length = np.asarray(seq_length)
    T, N = input_seq.shape
    L = w['encoder/encoder_h_transform/weights'].shape[0]

    def cell_vars(side, l):
        p = '%s/lstm/multi_rnn_cell/cell_%d/basic_lstm_cell/' % (side, l)
        return w[p + 'weights'], w[p + 'biases']
    seq_t = torch.as_tensor(input_seq.astype(np.int64))
    emb = w['encoder/embedding_mat'][seq_t]                                   # [T, N, E]  :88
    z = torch.zeros(N, L, dtype=torch.float64)
    state = [(z, z) for _ in range(num_layers)]
    outs = []
    for t in range(T):                                                        # :95-99
        live = torch.as_tensor(t < seq_length)[:, None]
        x = emb[t]
        new = []
        for l in range(num_layers):
            wl, bl = cell_vars('encoder', l)
            c2, h2 = _cell(x, state[l][0], state[l][1], wl, bl)
            new.append((torch.where(live, c2, state[l][0]), torch.where(live, h2, state[l][1])))
            x = h2
        outs.append(torch.where(live, x, torch.zeros_like(x)))
        state = new
    outs = torch.stack(outs)                                                  # [T, N, L]
    ht = outs @ w['encoder/encoder_h_transform/weights'] + w['encoder/encoder_h_transform/biases']
    not_finished = torch.as_tensor((np.arange(T)[:, None] < seq_length[None, :]).astype(np.float64))
    Wa, ba, v = (w['decoder/att_prediction/weights'], w['decoder/att_prediction/biases'],
                 w['decoder/att_prediction/v'])
    Wy, by = w['decoder/token_prediction/weights'], w['decoder/token_prediction/biases']
    V = w['decoder/embedding_mat'].shape[0]
    x = w['decoder/go_embedding'].expand(N, -1)                               # :202
    X = np.tile(np.array([[0, 0, T_dec]], np.int64), (N, 1))                  # :293
    P, W, b = np.asarray(P), np.asarray(W).astype(np.int64), np.asarray(b)
    toks, probs, atts = [], [], []
    neg_entropy = torch.zeros(N, dtype=torch.float64)
    rows = torch.arange(N)
    for t in range(T_dec):
        new = []
        for l in range(num_layers):
            wl, bl = cell_vars('decoder', l)
            c2, h2 = _cell(x, state[l][0], state[l][1], wl, bl)
            new.append((c2, h2))
            x = h2
        state = new
        out = x
        att_raw = (torch.tanh((out @ Wa + ba)[None] + ht) * v).sum(2)        # [T, N]  :208-212
        att = torch.softmax(att_raw, dim=0) * not_finished                   # :213-215
        att = att / att.sum(0, keepdim=True)                                  # :216
        d2 = (att[:, :, None] * outs).sum(0)                                  # :218
        scores = torch.cat([out, d2], dim=1) @ Wy + by                        # :221-223
        valid = np.all(np.tensordot(X, W, axes=1) - b >= 0, axis=2)           # :8-11
        if use_gt_layout:
            valid = np.ones_like(valid)                                       # :230-233
        vm = torch.as_tensor(valid.astype(np.float64))
        sc = scores.detach().numpy()
        if tokens is not None:
            pred = np.asarray(tokens[t]).astype(np.int64)
        else:
            masked = np.where(valid, sc, sc.min() - 1)                        # :259-261
            pred = np.argmax(masked, axis=1)
            if sample_uniforms is not None:                                   # :234-256
                zz = sc - (1.0 - valid) * 50.0
                q = np.exp(zz - zz.max(axis=1, keepdims=True))
                cdf = np.cumsum(q, axis=1) / q.sum(axis=1, keepdims=True)
                u = np.asarray(sample_uniforms[t], np.float64)
                samp = np.minimum((cdf <= u[:, None]).sum(axis=1), V - 1)
                pred = np.where(valid[np.arange(N), samp], samp, pred)
            if use_gt_layout:
                pred = np.asarray(gt_layout[t]).astype(np.int64)              # :264-266
        all_p = torch.softmax(scores, dim=1) * vm                             # :270
        all_p = all_p / all_p.sum(1, keepdim=True)                            # :272
        pt = torch.as_tensor(pred)
        probs.append(all_p[rows, pt])                                         # :281
        neg_entropy = neg_entropy + (all_p * torch.log(_tf_max_const(1e-5, all_p + (1 - vm)))).sum(1)
        X = X + P[pred]                                                       # :288-289
        toks.append(pred.astype(np.int32))
        atts.append(att)
        x = w['decoder/embedding_mat'][pt]                                    # :293
    atts = torch.stack(atts)                                                  # [T_dec, T, N]
    word_vecs = (atts[:, :, :, None] * emb[None]).sum(1)                      # :312
    return np.stack(toks), torch.stack(probs), neg_entropy, word_vecs, atts


def run(weights, input_seq, seq_length, T_dec, num_layers, P, W, b, use_gt_layout=False,
        gt_layout=None, sample_uniforms=None, tokens=None, d_log_seq_prob=None,
        d_neg_entropy=None, d_word_vecs=None):
    """Forward in float64 and, if any upstream gradient is given, the gradient of
    Σ d_lsp·log_seq_prob + Σ d_ne·neg_entropy + Σ d_wv·word_vecs for every variable.
    Returns (outputs dict of numpy arrays, grads dict of numpy float64 arrays or None)."""
    w = {k: torch.tensor(np.asarray(v, np.float64), requires_grad=True) for k, v in weights.items()}
    toks, probs, nent, wv, atts = forward(w, input_seq, seq_length, T_dec, num_layers, P, W, b,
                                          use_gt_layout, gt_layout, sample_uniforms, tokens)
    outs = dict(tokens=toks, token_probs=probs.detach().numpy(), neg_entropy=nent.detach().numpy(),
                word_vecs=wv.detach().numpy(), atts=atts.detach().numpy())
    if d_log_seq_prob is None and d_neg_entropy is None and d_word_vecs is None:
        return outs, None
    total = torch.zeros((), dtype=torch.float64)
    if d_log_seq_prob is not None:
        total = total + (torch.log(probs).sum(0) * torch.as_tensor(np.asarray(d_log_seq_prob, np.float64))).sum()
    if d_neg_entropy is not None:
        total = total + (nent * torch.as_tensor(np.asarray(d_neg_entropy, np.float64))).sum()
    if d_word_vecs is not None:
        total = total + (wv * torch.as_tensor(np.asarray(d_word_vecs, np.float64))).sum()
    names = list(w)
    gs = torch.autograd.grad(total, [w[k] for k in names], allow_unused=True)
    grads = {k: (g.numpy() if g is not None else np.zeros(w[k].shape)) for k, g in zip(names, gs)}
    return outs, grads
