"""CPU: the encoder's final state of the layout generator, the input of VQA's question-prior net
(models_vqa/nmn3_model.py, use_qpn=True), in the test oracle tests/seq2seq_states_oracle.py:
  * the numpy and the float64 states equal the reference's own `encoder_states` (encoder_c%d /
    encoder_h%d of tests/golden/golden_seq2seq.npz, from executing nmn3_netgen_att.py on the shim);
  * the gradient for an upstream on those states, alone and added to seq2seq_oracle_torch's
    gradient of the other three upstreams, equals central finite differences at lstm_dim 24 (a
    multiple of 8, not of 16), two layers and ragged lengths including 1 and T_enc;
  * the greedy top-2 score gaps replay the numpy oracle's greedy tokens."""
import os

import numpy as np

from n2nmn_b200 import synth
from n2nmn_b200.assembler import Assembler
from n2nmn_b200.weights import init_seq2seq_weights
from oracle import seq2seq_oracle as so
from oracle import seq2seq_oracle_torch as sot
from tests import seq2seq_states_oracle as sso

Z = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'golden_seq2seq.npz'))


def golden_weights():
    return {k[2 + len('encoder_decoder/'):]: Z[k] for k in Z.files if k.startswith('w:')}


def test_encoder_states_match_reference_goldens():
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers, seed = [int(v) for v in Z['cfg']]
    asm = Assembler(synth.vocab_file('clevr'))
    want = np.stack([np.stack([Z['encoder_c%d' % l], Z['encoder_h%d' % l]]) for l in range(layers)])
    enc, dec = so.run(golden_weights(), Z['input_seq'], Z['seq_length'], T_dec, layers, asm.P,
                      asm.W, asm.b)
    got = sso.encoder_states(enc)
    assert got.shape == (layers, 2, N, L)
    np.testing.assert_allclose(got, want, atol=1e-6)
    st, _ = sso.states_and_grads(golden_weights(), Z['input_seq'], Z['seq_length'], layers)
    np.testing.assert_allclose(st, want, atol=1e-6)
    # a question shorter than T_enc carries its state: it is not the state after T_enc steps
    assert (Z['seq_length'] < T_enc).any()
    gaps = sso.greedy_margins(golden_weights(), enc, dec[0], T_dec, layers, asm.P, asm.W, asm.b)
    assert gaps.shape == (T_dec, N) and (gaps >= 0).all()


def test_encoder_state_gradients_match_finite_differences():
    asm = Assembler(synth.vocab_file('vqa'))
    V = asm.num_vocab_nmn
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers = 4, 5, 4, 7, 4, 4, 24, 2
    w = {k: v.astype(np.float64) for k, v in
         init_seq2seq_weights(V_txt, E_txt, V, E_nmn, L, layers, seed=4).items()}
    rng = np.random.RandomState(1)
    seq = rng.randint(0, V_txt, size=(T_enc, N))
    lens = np.array([1, T_enc, 3, 2])
    gt = rng.randint(0, V, size=(T_dec, N))
    dlp, dne = rng.randn(N), rng.randn(N)
    dwv = rng.randn(T_dec, N, E_txt)
    des = rng.randn(layers, 2, N, L)
    kw = dict(use_gt_layout=True, gt_layout=gt)

    def total(ws, all_four):
        t = np.sum(sso.states_and_grads(ws, seq, lens, layers)[0] * des)
        if all_four:
            out, _ = sot.run(ws, seq, lens, T_dec, layers, asm.P, asm.W, asm.b, **kw)
            t += (np.sum(np.log(out['token_probs']).sum(0) * dlp) +
                  np.sum(out['neg_entropy'] * dne) + np.sum(out['word_vecs'] * dwv))
        return t
    eps = 1e-6
    for all_four in (False, True):
        _, g = sso.states_and_grads(w, seq, lens, layers, des)
        if all_four:
            _, g3 = sot.run(w, seq, lens, T_dec, layers, asm.P, asm.W, asm.b, d_log_seq_prob=dlp,
                            d_neg_entropy=dne, d_word_vecs=dwv, **kw)
            g = sso.add_grads(g3, g)
        else:
            # the encoder's state feeds no decoder variable
            assert all(np.abs(g[k]).max() == 0 for k in g if k.startswith('decoder/'))
            assert np.abs(g['encoder/lstm/multi_rnn_cell/cell_0/basic_lstm_cell/weights']).max() > 0
        worst = 0.0
        for name, val in w.items():
            flat = val.reshape(-1)
            for i in rng.choice(flat.size, size=min(5, flat.size), replace=False):
                wp, wm = dict(w), dict(w)
                a = flat.copy(); a[i] += eps; wp[name] = a.reshape(val.shape)
                b = flat.copy(); b[i] -= eps; wm[name] = b.reshape(val.shape)
                fd = (total(wp, all_four) - total(wm, all_four)) / (2 * eps)
                an = g[name].reshape(-1)[i]
                err = abs(fd - an) / max(1.0, abs(fd))
                worst = max(worst, err)
                assert err < 1e-6, (all_four, name, i, fd, an)
        print('all four upstreams' if all_four else 'd_encoder_states alone',
              'worst finite-difference error %.2e' % worst)
