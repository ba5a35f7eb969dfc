"""CPU oracle of the layout generator's LSTM dropout (`encoder_dropout` / `decoder_dropout`,
models_clevr/nmn3_netgen_att.py:17-44, :91, :303). It runs the seq2seq oracles themselves
(oracle/seq2seq_oracle.py, oracle/seq2seq_oracle_torch.py, and tests/seq2seq_states_oracle.py for
the encoder state's gradient) with their LSTM cell function hooked for the duration of one call;
nothing of their forward is restated here, so a fix to them reaches these results too:
  * `dropout`: tf.nn.dropout(x, 0.5) on given uniform numbers, as TF 1.0 computes it in fp32:
    x / 0.5 · floor(0.5 + u), i.e. kept iff u >= 0.5, a kept element is 2x (exact);
  * the hook: the oracles call the cell in loop order (every encoder step, then every decoder
    step; layer by layer inside a step), so the k-th call is one (side, step, layer). For a layer
    below the top one the hook attaches the dropped copy of the cell's output to it, and the next
    call, the layer above, takes that copy as its input x. The output itself, which the oracle
    keeps as the layer's state h (and, on the top layer, as the encoder output / attention query),
    stays undropped: DropoutWrapper drops only what the layer above reads. The number of calls is
    checked against the shapes after every run;
  * `run` / `encode`: seq2seq_oracle.run / encode with uniforms enc [T_enc, num_layers-1, N, L]
    and dec [T_dec, num_layers-1, N, L], one [N, L] draw per (step, dropped layer); None = no
    dropout on that side;
  * `run_torch`: seq2seq_oracle_torch.run (float64 autograd, TF's gradient conventions) under the
    same hook, so dropout's gradient is d·2·mask; d_encoder_states adds the gradient of the
    (undropped) encoder state, from seq2seq_states_oracle.states_and_grads under the hook;
  * `DropoutWrapper` / `install_shim_dropout` / `set_dropout_uniforms`: the TF 1.0 symbols for the
    numpy TF shim (oracle/tf1_shim_rnn.py) that let the reference file run with dropout on
    (tests/golden/make_golden_seq2seq_dropout.py). The wrapper adds no variable scope (TF 1.0's
    DropoutWrapper does not), so variable names do not change. Each call takes the next stored
    [N, units] uniform array, in call order. The shim's dynamic_rnn calls the cell at every step,
    where TF 1.0 skips steps past the longest sequence; that changes no output, since those steps'
    numbers are unused either way (the rows are past their ends)."""
import contextlib

import numpy as np
import torch

from oracle import seq2seq_oracle as so
from oracle import seq2seq_oracle_torch as sot
from tests import seq2seq_states_oracle as sso


def keep_mask(u):
    """floor(0.5 + u) in fp32: 1 where the element is kept."""
    return np.floor(np.float32(0.5) + np.asarray(u, np.float32)).astype(np.float32)


def dropout(x, u):
    return (np.asarray(x, np.float32) / np.float32(0.5) * keep_mask(u)).astype(np.float32)


class _Out(np.ndarray):
    """A numpy cell output that also carries the dropped copy the layer above reads."""
    dropped = None


def _np_attach(h, u):
    out = np.asarray(h).view(_Out)
    out.dropped = dropout(h, u)
    return out


def _np_input(x):
    return x.dropped if getattr(x, 'dropped', None) is not None else np.asarray(x)


def _torch_attach(h, u):
    h.dropped = h * torch.as_tensor(2.0 * keep_mask(u).astype(np.float64))   # d·2·mask backward
    return h


def _torch_input(x):
    return x.dropped if getattr(x, 'dropped', None) is not None else x


@contextlib.contextmanager
def _hooked(module, name, numpy, enc_u, dec_u, T_enc, T_dec, num_layers):
    """module.<name> (the oracle's cell function) drops the outputs of the layers below the top
    while the block runs; the block must make T_enc·layers encoder and T_dec·layers decoder calls."""
    cell = getattr(module, name)
    attach, take = (_np_attach, _np_input) if numpy else (_torch_attach, _torch_input)
    us = [None if u is None else np.asarray(u, np.float32) for u in (enc_u, dec_u)]
    for u, T in zip(us, (T_enc, T_dec)):
        assert u is None or u.shape[:2] == (T, num_layers - 1), u.shape
    calls = [0]

    def hooked(x, c, h, w, b):
        k = calls[0]
        calls[0] += 1
        side = 0 if k < T_enc * num_layers else 1
        t, l = divmod(k - side * T_enc * num_layers, num_layers)
        if numpy:
            c, h = np.asarray(c), np.asarray(h)
        c2, h2 = cell(take(x), c, h, w, b)
        if us[side] is not None and l < num_layers - 1:
            assert us[side][t, l].shape == tuple(h2.shape), (us[side].shape, h2.shape)
            h2 = attach(h2, us[side][t, l])
        return c2, h2
    setattr(module, name, hooked)
    try:
        yield
    finally:
        setattr(module, name, cell)
    assert calls[0] == (T_enc + T_dec) * num_layers, (calls[0], T_enc, T_dec, num_layers)


def encode(w, input_seq, seq_length, num_layers, enc_u=None):
    """seq2seq_oracle.encode with dropout between the layers."""
    input_seq = np.asarray(input_seq)
    with _hooked(so, 'lstm_cell', True, enc_u, None, input_seq.shape[0], 0, num_layers):
        return so.encode(w, input_seq, np.asarray(seq_length), num_layers)


def run(w, input_seq, seq_length, T_dec, num_layers, P, W, b, enc_u=None, dec_u=None, **kw):
    """seq2seq_oracle.run (same keywords) with dropout between the layers."""
    input_seq = np.asarray(input_seq)
    with _hooked(so, 'lstm_cell', True, enc_u, dec_u, input_seq.shape[0], T_dec, num_layers):
        return so.run(w, input_seq, seq_length, T_dec, num_layers, P, W, b, **kw)


def run_torch(weights, input_seq, seq_length, T_dec, num_layers, P, W, b, enc_u=None, dec_u=None,
              d_encoder_states=None, **kw):
    """seq2seq_oracle_torch.run (same keywords) with dropout between the layers: (outputs dict,
    grads dict or None). d_encoder_states [num_layers, 2, N, L] adds Σ d_encoder_states·
    encoder_states, the encoder's final (c, h), to the total; the outputs then also hold
    `encoder_states`."""
    input_seq = np.asarray(input_seq)
    T_enc = input_seq.shape[0]
    with _hooked(sot, '_cell', False, enc_u, dec_u, T_enc, T_dec, num_layers):
        outs, grads = sot.run(weights, input_seq, seq_length, T_dec, num_layers, P, W, b, **kw)
    if d_encoder_states is None:
        return outs, grads
    with _hooked(sso, '_cell', False, enc_u, None, T_enc, 0, num_layers):
        st, g_st = sso.states_and_grads(weights, input_seq, seq_length, num_layers, d_encoder_states)
    outs['encoder_states'] = st
    return outs, (g_st if grads is None else sso.add_grads(grads, g_st))




def golden_uniforms(seed, T_enc, T_dec, num_layers, N, L):
    """The uniform numbers of one case of golden_seq2seq_dropout.npz: (enc [T_enc, layers-1, N, L],
    dec [T_dec, layers-1, N, L], sampling [T_dec, N]), fp32."""
    rng = np.random.RandomState(seed)
    enc = rng.random_sample((T_enc, num_layers - 1, N, L)).astype(np.float32)
    dec = rng.random_sample((T_dec, num_layers - 1, N, L)).astype(np.float32)
    return enc, dec, rng.random_sample((T_dec, N)).astype(np.float32)


# ---- the numpy TF shim's DropoutWrapper ------------------------------------------------------------
_DROPOUT_UNIFORMS = []


def set_dropout_uniforms(rows):
    """Uniform arrays [N, units] that the shim's DropoutWrapper consumes, one per call, in call
    order (the encoder's steps, then the decoder's; layer by layer inside a step)."""
    _DROPOUT_UNIFORMS[:] = [np.asarray(r, np.float32) for r in rows]


def pending_dropout_uniforms():
    return len(_DROPOUT_UNIFORMS)


def shim_dropout(x, keep_prob):
    """tf.nn.dropout (TF 1.0 nn_ops.dropout): x / keep_prob · floor(keep_prob + u), in fp32."""
    u = _DROPOUT_UNIFORMS.pop(0)
    x = np.asarray(x, np.float32)
    assert u.shape == x.shape, (u.shape, x.shape)
    binary = np.floor(np.float32(keep_prob) + u).astype(np.float32)
    return (x / np.float32(keep_prob) * binary).astype(np.float32)


class DropoutWrapper:
    """TF 1.0 DropoutWrapper(cell, output_keep_prob): runs the cell in the caller's scope (no scope
    of its own) and applies tf.nn.dropout to the output only; the state passes through."""

    def __init__(self, cell, output_keep_prob=1.0):
        self.cell, self.output_keep_prob = cell, float(output_keep_prob)
        self.output_size = cell.output_size

    def __call__(self, inputs, state):
        out, new_state = self.cell(inputs, state)
        if self.output_keep_prob < 1.0:
            from oracle.tf1_shim import _t
            out = _t(shim_dropout(out, self.output_keep_prob))
        return out, new_state

    def zero_state(self, n):
        return self.cell.zero_state(n)


def install_shim_dropout(tf):
    """Adds DropoutWrapper and tf.nn.dropout to the fake module of tf1_shim_rnn.install_rnn()."""
    tf.contrib.rnn.DropoutWrapper = DropoutWrapper
    tf.nn.dropout = shim_dropout
    return tf
