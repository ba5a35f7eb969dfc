"""CPU: the float64 autograd restatement of AttentionSeq2Seq (oracle/seq2seq_oracle_torch.py), the
reference the GPU backward pass is measured against:
  * its forward equals the numpy oracle (itself pinned to the reference file's goldens) in greedy,
    teacher-forced and sampled decoding: tokens equal, values within 1e-6;
  * its gradients equal central finite differences on sampled coordinates of every variable
    (teacher forcing, tiny size, float64)."""
import os

import numpy as np
import pytest

from n2nmn_b200 import synth
from n2nmn_b200.assembler import Assembler
from n2nmn_b200.weights import init_seq2seq_weights
from oracle import seq2seq_oracle as so
from oracle import seq2seq_oracle_torch as sot

Z = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'golden_seq2seq.npz'))


def golden_weights():
    return {k[2 + len('encoder_decoder/'):]: Z[k] for k in Z.files if k.startswith('w:')}


@pytest.mark.parametrize('mode', ['greedy', 'gt', 'sample'])
def test_forward_matches_numpy_oracle(mode):
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers, seed = [int(v) for v in Z['cfg']]
    asm = Assembler(synth.vocab_file('clevr'))
    kw = {}
    if mode == 'gt':
        kw = dict(use_gt_layout=True, gt_layout=Z['gt_layout'])
    elif mode == 'sample':
        kw = dict(sample_uniforms=Z['sample_uniforms'])
    w = golden_weights()
    _, dec = so.run(w, Z['input_seq'], Z['seq_length'], T_dec, layers, asm.P, asm.W, asm.b, **kw)
    out, _ = sot.run(w, Z['input_seq'], Z['seq_length'], T_dec, layers, asm.P, asm.W, asm.b, **kw)
    assert np.array_equal(out['tokens'], dec[0])
    np.testing.assert_allclose(out['token_probs'], dec[1], atol=1e-6)
    np.testing.assert_allclose(out['neg_entropy'], dec[2], atol=1e-6)
    np.testing.assert_allclose(out['word_vecs'], dec[3], atol=1e-6)
    np.testing.assert_allclose(out['atts'], dec[4][..., 0], atol=1e-6)


def test_gradients_match_finite_differences():
    """Teacher forcing at a tiny size: every variable, a few sampled coordinates each, all three
    upstream gradients at once, ragged lengths (1 and T_enc included)."""
    asm = Assembler(synth.vocab_file('clevr'))
    V = asm.num_vocab_nmn
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers = 4, 5, 4, 7, 4, 4, 4, 2
    w = {k: v.astype(np.float64) for k, v in
         init_seq2seq_weights(V_txt, E_txt, V, E_nmn, L, layers, seed=3).items()}
    rng = np.random.RandomState(0)
    seq = rng.randint(0, V_txt, size=(T_enc, N))
    lens = np.array([1, T_enc, 3, 2])
    gt = rng.randint(0, V, size=(T_dec, N))
    dlp = rng.randn(N)
    dne = rng.randn(N)
    dwv = rng.randn(T_dec, N, E_txt)
    kw = dict(use_gt_layout=True, gt_layout=gt)

    def total(ws):
        out, _ = sot.run(ws, seq, lens, T_dec, layers, asm.P, asm.W, asm.b, **kw)
        return (np.sum(np.log(out['token_probs']).sum(0) * dlp) + np.sum(out['neg_entropy'] * dne) +
                np.sum(out['word_vecs'] * dwv))
    _, g = sot.run(w, seq, lens, T_dec, layers, asm.P, asm.W, asm.b, d_log_seq_prob=dlp,
                   d_neg_entropy=dne, d_word_vecs=dwv, **kw)
    eps = 1e-6
    worst = 0.0
    for name, val in w.items():
        flat = val.reshape(-1)
        for i in rng.choice(flat.size, size=min(6, flat.size), replace=False):
            wp = dict(w); wm = dict(w)
            a = flat.copy(); a[i] += eps; wp[name] = a.reshape(val.shape)
            b = flat.copy(); b[i] -= eps; wm[name] = b.reshape(val.shape)
            fd = (total(wp) - total(wm)) / (2 * eps)
            an = g[name].reshape(-1)[i]
            err = abs(fd - an) / max(1.0, abs(fd))
            worst = max(worst, err)
            assert err < 1e-6, (name, i, fd, an)
    print('worst finite-difference error %.2e' % worst)
