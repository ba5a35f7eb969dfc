"""CPU: the VQA loss oracle (tests/vqa_loss_oracle.py) — question prior added to the module
scores, cross-entropy on every row — and that with its defaults it is the CLEVR rule of
oracle/nmn_oracle_torch.py::loss_and_grads, bit for bit."""
import numpy as np
import torch
import torch.nn.functional as F

from n2nmn_b200 import synth, weights as wts
from n2nmn_b200.assembler import Assembler
from oracle import nmn_oracle_torch as ot
from tests import vqa_loss_oracle as vo


def _case(N=6, H=3, Wd=3, D=10, T=8, Cc=7, seed=0):
    feat, word_vecs = synth.make_inputs(N, H, Wd, D, T, seed=20 + seed, text_dim=12)
    W = wts.init_weights('vqa', H, Wd, D, Cc, seed=seed, bias_std=0.1, text_dim=12)
    asm = Assembler(synth.vocab_file('vqa'))
    layouts = [l for l, _ in synth.VQA_LAYOUTS][:N - 1] + [['_Find', '_Transform']]
    tokens = synth.tokens_from_layouts(asm, layouts, T)
    exprs, valid = asm.assemble(tokens)
    assert not valid[-1] and valid[:-1].all()
    labels = (np.arange(N) * 3) % Cc
    return feat, word_vecs, W, exprs, valid, labels, Cc


def test_prior_gradient_is_softmax_minus_onehot_on_every_row():
    feat, word_vecs, W, exprs, valid, labels, Cc = _case()
    N = len(exprs)
    prior = np.random.RandomState(1).standard_normal((N, Cc)).astype(np.float32)
    m = ot.TorchOracleModules(feat, word_vecs, Cc, W, family='vqa')
    s, per, avg, g, g_wv, g_prior = vo.loss_and_grads(m, exprs, valid, labels, score_prior=prior,
                                                      ce_every_row=True)
    module = ot.forward_scores(ot.TorchOracleModules(feat, word_vecs, Cc, W, family='vqa'),
                               exprs).detach().numpy()
    np.testing.assert_allclose(s, module + prior, rtol=0, atol=1e-6)
    assert np.all(module[-1] == 0)                      # invalid layout: zero module scores
    p = torch.softmax(torch.as_tensor(s, dtype=torch.float64), dim=1).numpy()
    want = (p - np.eye(Cc)[labels]) / N
    np.testing.assert_allclose(g_prior, want, rtol=0, atol=1e-6)
    assert np.abs(g_prior[-1]).max() > 0                # the invalid row is trained too
    ce = F.cross_entropy(torch.as_tensor(s, dtype=torch.float64),
                         torch.as_tensor(labels, dtype=torch.long), reduction='none').numpy()
    np.testing.assert_allclose(per, ce, rtol=1e-5, atol=1e-6)
    assert abs(avg - float(ce.mean())) < 1e-5


def test_defaults_reproduce_the_clevr_rule_bit_for_bit():
    feat, word_vecs, W, exprs, valid, labels, Cc = _case(seed=2)

    def fresh():
        return ot.TorchOracleModules(feat, word_vecs, Cc, W, family='vqa')
    want = ot.loss_and_grads(fresh(), exprs, valid, labels)
    for got in (vo.loss_and_grads(fresh(), exprs, valid, labels),
                vo.loss_and_grads(fresh(), exprs, valid, labels, score_prior=None,
                                  ce_every_row=False)):
        assert len(got) == 5
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
        assert got[2] == want[2]
        assert set(got[3]) == set(want[3])
        for n in want[3]:
            assert np.array_equal(got[3][n], want[3][n]), n
        assert np.array_equal(got[4], want[4])
    assert want[1][-1] == 0.5
