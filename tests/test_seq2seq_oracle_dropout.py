"""CPU: the dropout oracle of the layout generator (tests/seq2seq_dropout_oracle.py):
  * the numpy forward equals the goldens produced by executing the reference's nmn3_netgen_att.py
    with encoder_dropout = decoder_dropout = True on the TF shim (golden_seq2seq_dropout.npz):
    tokens equal, values within 1e-6, at 2 and 3 layers in greedy, forced and sampled decoding;
  * the float64 autograd forward equals the numpy forward, and its gradients equal central finite
    differences with the masks fixed, for every variable;
  * with no uniforms both are the dropout-free oracles, and the shim's LSTM stack with the
    DropoutWrapper symbols installed still reproduces golden_seq2seq.npz."""
import os

import numpy as np
import pytest

from n2nmn_b200 import synth
from n2nmn_b200.assembler import Assembler
from n2nmn_b200.weights import init_seq2seq_weights
from oracle import seq2seq_oracle as so
from oracle import seq2seq_oracle_torch as sot
from tests import seq2seq_dropout_oracle as sdo

GOLDEN = os.path.join(os.path.dirname(__file__), 'golden')
ZD = np.load(os.path.join(GOLDEN, 'golden_seq2seq_dropout.npz'))
Z = np.load(os.path.join(GOLDEN, 'golden_seq2seq.npz'))


def golden_case(layers, case):
    """(weights, seq, lens, T_dec, kwargs of sdo.run, prefix) of one golden case."""
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, seed = [int(v) for v in ZD['cfg']]
    pre = 'l%d_' % layers
    w = {k[len(pre) + 2 + len('encoder_decoder/'):]: ZD[k] for k in ZD.files
         if k.startswith(pre + 'w:')}
    enc_u, dec_u, samp_u = sdo.golden_uniforms(int(ZD[pre + case + '_uniform_seed']), T_enc, T_dec,
                                               layers, N, L)
    kw = dict(enc_u=enc_u, dec_u=dec_u)
    if case == 'gt':
        kw.update(use_gt_layout=True, gt_layout=ZD['gt_layout'])
    elif case == 'sample':
        kw.update(sample_uniforms=samp_u)
    return w, ZD[pre + 'input_seq'], ZD[pre + 'seq_length'], T_dec, kw, pre + case + '_'


@pytest.mark.parametrize('layers', [2, 3])
@pytest.mark.parametrize('case', ['greedy', 'gt', 'sample'])
def test_numpy_oracle_matches_reference_golden(layers, case):
    asm = Assembler(synth.vocab_file('clevr'))
    w, seq, lens, T_dec, kw, p = golden_case(layers, case)
    enc, dec = sdo.run(w, seq, lens, T_dec, layers, asm.P, asm.W, asm.b, **kw)
    _, outs, state, _, _ = enc
    np.testing.assert_allclose(outs, ZD[p + 'encoder_outputs'], atol=1e-6)
    for l in range(layers):
        np.testing.assert_allclose(state[l][0], ZD[p + 'encoder_c%d' % l], atol=1e-6)
        np.testing.assert_allclose(state[l][1], ZD[p + 'encoder_h%d' % l], atol=1e-6)
    tokens, probs, nent, wv, atts = dec
    assert np.array_equal(tokens, ZD[p + 'predicted_tokens'])
    np.testing.assert_allclose(probs, ZD[p + 'token_probs'], atol=1e-6)
    np.testing.assert_allclose(nent, ZD[p + 'neg_entropy'], atol=1e-6)
    np.testing.assert_allclose(wv, ZD[p + 'word_vecs'], atol=1e-6)
    np.testing.assert_allclose(atts, ZD[p + 'atts'], atol=1e-6)
    # dropout changed the run: the same case without it decodes other values
    _, dec0 = so.run(w, seq, lens, T_dec, layers, asm.P, asm.W, asm.b,
                     **{k: v for k, v in kw.items() if k not in ('enc_u', 'dec_u')})
    assert np.abs(dec0[1] - probs).max() > 1e-3


@pytest.mark.parametrize('layers', [2, 3])
@pytest.mark.parametrize('case', ['greedy', 'gt', 'sample'])
def test_torch_forward_matches_numpy(layers, case):
    asm = Assembler(synth.vocab_file('clevr'))
    w, seq, lens, T_dec, kw, _ = golden_case(layers, case)
    _, dec = sdo.run(w, seq, lens, T_dec, layers, asm.P, asm.W, asm.b, **kw)
    out, _ = sdo.run_torch(w, seq, lens, T_dec, layers, asm.P, asm.W, asm.b, **kw)
    assert np.array_equal(out['tokens'], dec[0])
    np.testing.assert_allclose(out['token_probs'], dec[1], atol=1e-6)
    np.testing.assert_allclose(out['neg_entropy'], dec[2], atol=1e-6)
    np.testing.assert_allclose(out['word_vecs'], dec[3], atol=1e-6)
    np.testing.assert_allclose(out['atts'], dec[4][..., 0], atol=1e-6)


def test_without_uniforms_is_the_dropout_free_oracle():
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers, seed = [int(v) for v in Z['cfg']]
    asm = Assembler(synth.vocab_file('clevr'))
    w = {k[2 + len('encoder_decoder/'):]: Z[k] for k in Z.files if k.startswith('w:')}
    kw = dict(sample_uniforms=Z['sample_uniforms'])
    _, a = so.run(w, Z['input_seq'], Z['seq_length'], T_dec, layers, asm.P, asm.W, asm.b, **kw)
    _, b = sdo.run(w, Z['input_seq'], Z['seq_length'], T_dec, layers, asm.P, asm.W, asm.b, **kw)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    o1, _ = sot.run(w, Z['input_seq'], Z['seq_length'], T_dec, layers, asm.P, asm.W, asm.b, **kw)
    o2, _ = sdo.run_torch(w, Z['input_seq'], Z['seq_length'], T_dec, layers, asm.P, asm.W, asm.b, **kw)
    for k in o1:
        assert np.array_equal(o1[k], o2[k])
    # all-kept uniforms double every dropped value, all-dropped zero it: both differ from no dropout
    ones = np.full((T_enc, layers - 1, N, L), 0.75, np.float32)
    _, kept = sdo.run(w, Z['input_seq'], Z['seq_length'], T_dec, layers, asm.P, asm.W, asm.b,
                      enc_u=ones, **kw)
    assert not np.array_equal(kept[1], a[1])


def test_shim_stack_without_dropout_reproduces_golden():
    """The shim's MultiRNNCell + dynamic_rnn, with the DropoutWrapper symbols installed and no
    dropout asked for, gives golden_seq2seq.npz's encoder outputs and final states."""
    from oracle import tf1_shim, tf1_shim_rnn
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers, seed = [int(v) for v in Z['cfg']]
    weights = {k[2:]: Z[k] for k in Z.files if k.startswith('w:')}
    tf = sdo.install_shim_dropout(tf1_shim_rnn.install_rnn(tf1_shim.install(weights)))
    try:
        sdo.set_dropout_uniforms([])
        cell = tf.contrib.rnn.MultiRNNCell([tf.contrib.rnn.BasicLSTMCell(L)] * layers)
        emb = Z['w:encoder_decoder/encoder/embedding_mat'][Z['input_seq']]
        with tf1_shim.variable_scope('encoder_decoder'), tf1_shim.variable_scope('encoder'):
            outs, states = tf.nn.dynamic_rnn(cell, emb, Z['seq_length'], time_major=True, scope='lstm')
        np.testing.assert_allclose(np.asarray(outs), Z['encoder_outputs'], atol=1e-6)
        for l in range(layers):
            np.testing.assert_allclose(np.asarray(states[l][0]), Z['encoder_c%d' % l], atol=1e-6)
            np.testing.assert_allclose(np.asarray(states[l][1]), Z['encoder_h%d' % l], atol=1e-6)
        # a wrapper at keep_prob 1 draws nothing and changes nothing; at 0.5 it draws one per call
        wrapped = tf.contrib.rnn.MultiRNNCell([tf.contrib.rnn.DropoutWrapper(
            tf.contrib.rnn.BasicLSTMCell(L), output_keep_prob=1.0)] * layers)
        with tf1_shim.variable_scope('encoder_decoder'), tf1_shim.variable_scope('encoder'):
            outs1, _ = tf.nn.dynamic_rnn(wrapped, emb, Z['seq_length'], time_major=True, scope='lstm')
        assert np.array_equal(np.asarray(outs1), np.asarray(outs))
        u = np.random.RandomState(0).random_sample((T_enc, layers - 1, N, L)).astype(np.float32)
        sdo.set_dropout_uniforms(list(u.reshape(-1, N, L)))
        dropped = tf.contrib.rnn.MultiRNNCell(
            [tf.contrib.rnn.DropoutWrapper(tf.contrib.rnn.BasicLSTMCell(L), output_keep_prob=0.5)] *
            (layers - 1) + [tf.contrib.rnn.BasicLSTMCell(L)])
        with tf1_shim.variable_scope('encoder_decoder'), tf1_shim.variable_scope('encoder'):
            outs2, _ = tf.nn.dynamic_rnn(dropped, emb, Z['seq_length'], time_major=True, scope='lstm')
        assert sdo.pending_dropout_uniforms() == 0
        w = {k[len('encoder_decoder/'):]: v for k, v in weights.items()}
        enc = sdo.encode(w, Z['input_seq'], Z['seq_length'], layers, u)
        np.testing.assert_allclose(np.asarray(outs2), enc[1], atol=1e-6)
    finally:
        tf1_shim.uninstall()


def test_dropout_rule():
    u = np.array([0.0, 0.25, 0.49999994, 0.5, 0.75, 0.99999994], np.float32)
    assert np.array_equal(sdo.keep_mask(u), [0, 0, 0, 1, 1, 1])
    x = np.array([1.5, -2.0, 3.0, -0.1, 1e-30, 7.0], np.float32)
    assert np.array_equal(sdo.dropout(x, u), np.array([0, 0, 0, -0.2, 2e-30, 14.0], np.float32))


@pytest.mark.parametrize('sides', ['enc', 'dec', 'both'])
def test_gradients_match_finite_differences(sides):
    """Teacher forcing at a tiny size, 3 layers, masks fixed: every variable, a few sampled
    coordinates each, all four upstream gradients at once (d_encoder_states included), ragged
    lengths."""
    asm = Assembler(synth.vocab_file('clevr'))
    V = asm.num_vocab_nmn
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers = 4, 5, 4, 7, 4, 4, 4, 3
    w = {k: v.astype(np.float64) for k, v in
         init_seq2seq_weights(V_txt, E_txt, V, E_nmn, L, layers, seed=5).items()}
    rng = np.random.RandomState(1)
    seq = rng.randint(0, V_txt, size=(T_enc, N))
    lens = np.array([1, T_enc, 3, 2])
    gt = rng.randint(0, V, size=(T_dec, N))
    dlp, dne, dwv = rng.randn(N), rng.randn(N), rng.randn(T_dec, N, E_txt)
    dst = rng.randn(layers, 2, N, L)
    kw = dict(use_gt_layout=True, gt_layout=gt)
    if sides in ('enc', 'both'):
        kw['enc_u'] = rng.random_sample((T_enc, layers - 1, N, L)).astype(np.float32)
    if sides in ('dec', 'both'):
        kw['dec_u'] = rng.random_sample((T_dec, layers - 1, N, L)).astype(np.float32)

    def total(ws):
        out, _ = sdo.run_torch(ws, seq, lens, T_dec, layers, asm.P, asm.W, asm.b,
                               d_encoder_states=dst, **kw)
        return (np.sum(np.log(out['token_probs']).sum(0) * dlp) + np.sum(out['neg_entropy'] * dne) +
                np.sum(out['word_vecs'] * dwv) + np.sum(out['encoder_states'] * dst))
    _, g = sdo.run_torch(w, seq, lens, T_dec, layers, asm.P, asm.W, asm.b, d_log_seq_prob=dlp,
                         d_neg_entropy=dne, d_word_vecs=dwv, d_encoder_states=dst, **kw)
    eps = 1e-6
    for name, val in w.items():
        flat = val.reshape(-1)
        for i in rng.choice(flat.size, size=min(6, flat.size), replace=False):
            wp, wm = dict(w), dict(w)
            a = flat.copy(); a[i] += eps; wp[name] = a.reshape(val.shape)
            b = flat.copy(); b[i] -= eps; wm[name] = b.reshape(val.shape)
            fd = (total(wp) - total(wm)) / (2 * eps)
            an = g[name].reshape(-1)[i]
            assert abs(fd - an) / max(1.0, abs(fd)) < 1e-6, (name, i, fd, an)
