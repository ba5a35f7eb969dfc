"""CPU oracle of what VQA's question-prior net takes from the layout generator, on top of the
seq2seq oracles (oracle/seq2seq_oracle.py, oracle/seq2seq_oracle_torch.py):
  * `encoder_states`: the encoder's final state of `seq2seq_oracle.encode(...)` — dynamic_rnn's,
    each question's state at its own length (nmn3_netgen_att.py:95-99) — as one
    [num_layers, 2, N, L] array of (c, h) per layer (LSTMStateTuple order);
  * `states_and_grads`: the same state in float64 with torch autograd (the encoder of
    seq2seq_oracle_torch.forward, restated with its cell) and the gradient of
    Σ d_encoder_states·encoder_states for every variable. The state depends on the encoder alone,
    so the gradient of a total that also has the other three upstreams is this one plus
    seq2seq_oracle_torch.run's (`add_grads`);
  * `greedy_margins`: per decoding step, the gap between the best and the second-best valid token
    score of greedy decoding (inf with one valid token) — how far a greedy token is from flipping
    under another summation order. It replays seq2seq_oracle.decode's score computation along the
    oracle's greedy tokens and checks that they are the argmax."""
import numpy as np
import torch

from oracle import seq2seq_oracle as so
from oracle.seq2seq_oracle_torch import _cell


def encoder_states(enc):
    return np.stack([np.stack([c, h]) for c, h in enc[2]])


def states_and_grads(weights, input_seq, seq_length, num_layers, d_encoder_states=None):
    """(encoder states [num_layers, 2, N, L] float64, {variable: grad} or None)."""
    w = {k: torch.tensor(np.asarray(v, np.float64), requires_grad=True) for k, v in weights.items()}
    input_seq, seq_length = np.asarray(input_seq), np.asarray(seq_length)
    T, N = input_seq.shape
    L = w['encoder/encoder_h_transform/weights'].shape[0]
    emb = w['encoder/embedding_mat'][torch.as_tensor(input_seq.astype(np.int64))]
    z = torch.zeros(N, L, dtype=torch.float64)
    state = [(z, z) for _ in range(num_layers)]
    for t in range(T):                                                        # :95-99
        live = torch.as_tensor(t < seq_length)[:, None]
        x = emb[t]
        new = []
        for l in range(num_layers):
            p = 'encoder/lstm/multi_rnn_cell/cell_%d/basic_lstm_cell/' % l
            c2, h2 = _cell(x, state[l][0], state[l][1], w[p + 'weights'], w[p + 'biases'])
            new.append((torch.where(live, c2, state[l][0]), torch.where(live, h2, state[l][1])))
            x = h2
        state = new
    st = torch.stack([torch.stack([c, h]) for c, h in state])
    if d_encoder_states is None:
        return st.detach().numpy(), None
    total = (st * torch.as_tensor(np.asarray(d_encoder_states, np.float64))).sum()
    names = list(w)
    gs = torch.autograd.grad(total, [w[k] for k in names], allow_unused=True)
    return st.detach().numpy(), {k: (g.numpy() if g is not None else np.zeros(w[k].shape))
                                 for k, g in zip(names, gs)}


def add_grads(a, b):
    return {k: a[k] + b[k] for k in a}


def greedy_margins(w, enc, tokens, T_dec, num_layers, P, W, b):
    """[T_dec, N] top-2 valid score gaps along the greedy tokens `tokens` of seq2seq_oracle.decode
    (same formulas, :205-293); asserts that each token is the masked argmax."""
    emb, outs, state, ht, not_finished = enc
    N = emb.shape[1]
    Wa, ba, v = (w['decoder/att_prediction/weights'], w['decoder/att_prediction/biases'],
                 w['decoder/att_prediction/v'])
    Wy, by = w['decoder/token_prediction/weights'], w['decoder/token_prediction/biases']
    x = np.tile(w['decoder/go_embedding'], (N, 1))
    X = np.tile(np.array([[0, 0, T_dec]], np.int64), (N, 1))
    P, W, b = np.asarray(P), np.asarray(W).astype(np.int64), np.asarray(b)
    gaps = []
    for t in range(T_dec):
        new = []
        for l in range(num_layers):
            p = 'decoder/lstm/multi_rnn_cell/cell_%d/basic_lstm_cell/' % l
            c2, h2 = so.lstm_cell(x, state[l][0], state[l][1], w[p + 'weights'], w[p + 'biases'])
            new.append((c2, h2))
            x = h2
        state = new
        att_raw = np.sum(np.tanh((x @ Wa + ba) + ht) * v, axis=2, keepdims=True)
        e = np.exp(att_raw - att_raw.max(axis=0, keepdims=True))
        att = e / e.sum(axis=0, keepdims=True) * not_finished
        att = att / att.sum(axis=0, keepdims=True)
        d2 = np.sum(att * outs, axis=0)
        scores = (np.concatenate([x, d2], axis=1) @ Wy + by).astype(np.float32)
        valid = np.all(np.tensordot(X, W, axes=1) - b >= 0, axis=2)
        masked = np.where(valid, scores, scores.min() - 1)
        pred = np.asarray(tokens[t]).astype(np.int64)
        assert np.array_equal(np.argmax(masked, axis=1), pred)
        top2 = np.sort(np.where(valid, scores, -np.inf), axis=1)[:, -2:]
        gaps.append(top2[:, 1] - top2[:, 0])
        X = X + P[pred]
        x = w['decoder/embedding_mat'][pred]
    return np.stack(gaps)
