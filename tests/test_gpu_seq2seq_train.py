"""GPU: training the seq2seq layout generator (n2nmn_seq2seq_set_record / _backward / _adam_step):
  * every variable's gradient against the float64 autograd oracle (oracle/seq2seq_oracle_torch.py,
    TF 1.0's gradients of nmn3_netgen_att.py): rel_err = max|Δ| / max|ref| <= 5e-3, for teacher
    forcing, sampled and greedy decoding, at the golden config, CLEVR training sizes (N=64,
    T_enc=45, T_dec=10, lstm 512, 2 layers, ragged lengths with 1 and T_enc), N=37 / T_enc=26 /
    T_dec=13 / lstm 208 / 1 layer, and a 3-layer tiny case;
  * NULL upstream gradients, recording leaves the forward bit-identical, loud errors, launch
    counts, the clip + Adam step against TF's formula, and learning runs."""
import os

import numpy as np
import pytest
import torch

from n2nmn_b200 import synth, _lib
from n2nmn_b200.assembler import Assembler
from n2nmn_b200.weights import init_seq2seq_weights
from oracle import seq2seq_oracle_torch as sot

pytestmark = pytest.mark.gpu
Z = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'golden_seq2seq.npz'))
BAR = 5e-3


def golden_weights():
    return {k[2 + len('encoder_decoder/'):]: Z[k] for k in Z.files if k.startswith('w:')}


def make(asm, w, T_enc, N, T_dec, V_txt, E_txt, E_nmn, L, layers, decoder_sampling=False):
    from n2nmn_b200.seq2seq import AttentionSeq2Seq
    return AttentionSeq2Seq(None, None, T_dec, V_txt, E_txt, asm.num_vocab_nmn, E_nmn, L, layers,
                            asm, T_encoder=T_enc, max_batch=N, weights=w, device='cuda:0',
                            decoder_sampling=decoder_sampling)


def problem(cfg, seed=0):
    """(asm, weights, inputs) for cfg = (N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers)."""
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers = cfg
    asm = Assembler(synth.vocab_file('clevr'))
    if cfg == golden_cfg():
        w = golden_weights()
        seq, lens = Z['input_seq'], Z['seq_length']
    else:
        w = init_seq2seq_weights(V_txt, E_txt, asm.num_vocab_nmn, E_nmn, L, layers, seed=seed)
        rng = np.random.RandomState(seed + 1)
        seq = rng.randint(0, V_txt, size=(T_enc, N)).astype(np.int32)
        lens = rng.randint(1, T_enc + 1, size=N).astype(np.int32)
        lens[0], lens[-1] = 1, T_enc
    return asm, w, seq, lens


def golden_cfg():
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers, _ = [int(v) for v in Z['cfg']]
    return (N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers)


CFGS = {
    'golden': golden_cfg(),
    'clevr': (64, 45, 10, 90, 300, 300, 512, 2),
    'odd': (37, 26, 13, 50, 64, 32, 208, 1),
    'deep': (5, 7, 5, 11, 8, 12, 32, 3),
}


def compare(s, ref_grads, label):
    torch.cuda.synchronize()
    worst = []
    for name, g in s.grads().items():
        ref = ref_grads[name]
        scale = np.abs(ref).max()
        err = np.abs(g.cpu().numpy().astype(np.float64) - ref).max()
        rel = err / scale if scale > 0 else err
        worst.append((rel, name))
    worst.sort(reverse=True)
    print('%s: worst rel_err %s' % (label, ', '.join('%.2e %s' % w for w in worst[:3])))
    assert worst[0][0] <= BAR, worst[:3]


@pytest.mark.parametrize('size', list(CFGS))
@pytest.mark.parametrize('mode', ['gt', 'sample', 'greedy'])
def test_gradients_match_oracle(size, mode):
    cfg = CFGS[size]
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers = cfg
    asm, w, seq, lens = problem(cfg)
    rng = np.random.RandomState(7)
    V = asm.num_vocab_nmn
    kw, up = {}, {}
    dlp = rng.randn(N).astype(np.float32)
    if mode == 'gt':
        kw = dict(use_gt_layout=True, gt_layout_batch=rng.randint(0, V, size=(T_dec, N)).astype(np.int32))
        up = dict(d_log_seq_prob=dlp)
    else:
        up = dict(d_log_seq_prob=dlp, d_neg_entropy=rng.randn(N).astype(np.float32),
                  d_word_vecs=rng.randn(T_dec, N, E_txt).astype(np.float32))
    u = rng.uniform(size=(T_dec, N)).astype(np.float32) if mode == 'sample' else None
    s = make(asm, w, T_enc, N, T_dec, V_txt, E_txt, E_nmn, L, layers, decoder_sampling=mode == 'sample')
    tokens = s.forward(seq, lens, sample_uniforms=u, record=True, **kw)[0]
    s.backward(**{k: torch.as_tensor(v).cuda() for k, v in up.items()})
    tok = tokens.cpu().numpy()
    okw = dict(use_gt_layout=True, gt_layout=kw['gt_layout_batch']) if mode == 'gt' else dict(tokens=tok)
    _, ref = sot.run(w, seq, lens, T_dec, layers, asm.P, asm.W, asm.b, **okw,
                     **{k: v.astype(np.float64) for k, v in up.items()})
    compare(s, ref, '%s/%s' % (size, mode))


def test_null_upstreams():
    cfg = CFGS['golden']
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers = cfg
    asm, w, seq, lens = problem(cfg)
    s = make(asm, w, T_enc, N, T_dec, V_txt, E_txt, E_nmn, L, layers)
    s.forward(seq, lens, record=True)
    dwv = torch.randn(T_dec, N, E_txt, device='cuda')
    s.backward(d_word_vecs=dwv)
    g = s.grads()
    assert (g['decoder/token_prediction/weights'] == 0).all()
    assert (g['decoder/token_prediction/biases'] == 0).all()
    assert (g['encoder/embedding_mat'] != 0).any()
    s.backward()
    assert all((v == 0).all() for v in s.grads().values())


def test_recording_leaves_forward_bit_identical_and_launch_counts():
    from n2nmn_b200.trainer import LayoutGeneratorTrainer
    for size in ('clevr', 'golden'):
        cfg = CFGS[size]
        N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers = cfg
        asm, w, seq, lens = problem(cfg)
        s = make(asm, w, T_enc, N, T_dec, V_txt, E_txt, E_nmn, L, layers)
        n_set = s.launch_count()
        a = [o.clone() for o in s.forward(seq, lens)]
        n0 = s.launch_count()
        a2 = [o.clone() for o in s.forward(seq, lens)]
        n_off = s.launch_count() - n0
        # recording off: (T_enc + layers - 1) + layers·T_dec + 2·T_dec + 3 launches, as before
        assert n_off == (T_enc + layers - 1) + layers * T_dec + 2 * T_dec + 3
        # the first forward after set_weights also re-derives the packed weights: two regroups per
        # cell, the two input tables and the transposed token_prediction matrix
        assert n0 - n_set - n_off == 4 * layers + 3
        n1 = s.launch_count()
        b = [o.clone() for o in s.forward(seq, lens, record=True)]
        assert s.launch_count() - n1 == n_off
        torch.cuda.synchronize()
        for x, y, z in zip(a, a2, b):
            assert torch.equal(x, y) and torch.equal(x, z)
        n2 = s.launch_count()
        s.backward(d_log_seq_prob=torch.ones(N, device='cuda'))
        first = s.launch_count() - n2
        s.forward(seq, lens, record=True)
        n3 = s.launch_count()
        s.backward(d_log_seq_prob=torch.ones(N, device='cuda'))
        per = s.launch_count() - n3
        want = 14 + 2 * layers * T_dec + 2 * (T_enc + layers - 1) + 4 * layers
        assert per == want, (per, want)
        assert first == want + 2 * layers + 2      # the transposed matrices, once per weight change
        tr = LayoutGeneratorTrainer(s)
        s.forward(seq, lens, record=True)
        n4 = s.launch_count()
        tr.step(d_log_seq_prob=torch.ones(N, device='cuda'))
        assert s.launch_count() - n4 == per + 2    # the backward, then grad_norm and adam_clip
        print('%s: forward %d launches, backward %d' % (size, n_off, per))


def test_errors_are_loud():
    cfg = CFGS['golden']
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers = cfg
    asm, w, seq, lens = problem(cfg)
    s = make(asm, w, T_enc, N, T_dec, V_txt, E_txt, E_nmn, L, layers)
    with pytest.raises(_lib.N2NMNError):
        s.backward(d_log_seq_prob=torch.ones(N, device='cuda'))
    s.forward(seq, lens)
    with pytest.raises(_lib.N2NMNError):
        s.backward(d_log_seq_prob=torch.ones(N, device='cuda'))
    s.forward(seq, lens, record=True)
    with pytest.raises(ValueError):
        s.backward(d_log_seq_prob=torch.ones(N - 1, device='cuda'))
    s.set_weights(w)
    with pytest.raises(_lib.N2NMNError):
        s.backward(d_log_seq_prob=torch.ones(N, device='cuda'))
    # and at the C level: the ABI refuses a backward after a non-recording forward
    s.forward(seq, lens)
    out = torch.empty(s.flat_layout()[0], device='cuda')
    rc = s._L.n2nmn_seq2seq_backward(s._h, None, None, None, out.data_ptr(), s._stream())
    assert rc != 0


def test_adam_step_matches_tf_formula_and_refreshes_the_forward():
    from n2nmn_b200.trainer import LayoutGeneratorTrainer
    cfg = CFGS['odd']
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers = cfg
    asm, w, seq, lens = problem(cfg)
    s = make(asm, w, T_enc, N, T_dec, V_txt, E_txt, E_nmn, L, layers)
    hp = dict(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, max_grad_l2_norm=0.5, weight_decay=1e-2)
    tr = LayoutGeneratorTrainer(s, **hp)
    w0 = {k: v.cpu().numpy().astype(np.float64) for k, v in s.get_weights().items()}
    s.forward(seq, lens, record=True)
    tr.step(d_log_seq_prob=torch.full((N,), -1.0 / N, device='cuda'))
    torch.cuda.synchronize()
    g = {k: v.cpu().numpy().astype(np.float64) for k, v in tr.grads().items()}   # (decay included)
    w1 = {k: v.cpu().numpy() for k, v in s.get_weights().items()}
    lr_t = hp['lr'] * np.sqrt(1 - hp['beta2']) / (1 - hp['beta1'])
    for name in w0:
        gd = g[name]
        # the gradient buffer holds g + wd·w on '/weights' variables (the reference's l2_reg)
        nrm = np.sqrt((gd ** 2).sum())
        gc = gd * (hp['max_grad_l2_norm'] / nrm if nrm > hp['max_grad_l2_norm'] else 1.0)
        m = (1 - hp['beta1']) * gc
        v = (1 - hp['beta2']) * gc * gc
        want = w0[name] - lr_t * m / (np.sqrt(v) + hp['eps'])
        np.testing.assert_allclose(w1[name], want, atol=2e-6, err_msg=name)
    # weight decay only on '/weights': recompute the raw gradient and compare the difference
    s.forward(seq, lens, record=True)
    s.backward(d_log_seq_prob=torch.full((N,), -1.0 / N, device='cuda'))
    # a forward after the step equals a fresh context given the new weights, bit for bit
    s2 = make(asm, {k: v for k, v in w1.items()}, T_enc, N, T_dec, V_txt, E_txt, E_nmn, L, layers)
    a = s.forward(seq, lens)
    b = s2.forward(seq, lens)
    torch.cuda.synchronize()
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def test_weight_decay_only_on_weights_variables():
    from n2nmn_b200.trainer import LayoutGeneratorTrainer
    cfg = CFGS['deep']
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers = cfg
    asm, w, seq, lens = problem(cfg)
    s = make(asm, w, T_enc, N, T_dec, V_txt, E_txt, E_nmn, L, layers)
    tr = LayoutGeneratorTrainer(s, lr=1e-3, max_grad_l2_norm=1e9, weight_decay=0.5)
    s.forward(seq, lens, record=True)
    s.backward(d_log_seq_prob=torch.full((N,), -1.0 / N, device='cuda'))
    raw = {k: v.clone() for k, v in s.grads().items()}
    wts = {k: v.clone() for k, v in s.get_weights().items()}
    s.forward(seq, lens, record=True)
    tr.step(d_log_seq_prob=torch.full((N,), -1.0 / N, device='cuda'))
    torch.cuda.synchronize()
    for name, g in tr.grads().items():
        extra = (g - raw[name]).cpu().numpy()
        if name.endswith('/weights'):
            np.testing.assert_allclose(extra, 0.5 * wts[name].cpu().numpy(), rtol=1e-5, atol=1e-6)
        else:   # (embedding rows are summed with atomics: the order, not the value, may differ)
            assert np.abs(extra).max() <= 1e-6 * max(1e-3, float(raw[name].abs().max())), name


def test_gt_layout_nll_falls():
    from n2nmn_b200.trainer import LayoutGeneratorTrainer
    cfg = CFGS['odd']
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers = cfg
    asm, w, seq, lens = problem(cfg)
    s = make(asm, w, T_enc, N, T_dec, V_txt, E_txt, E_nmn, L, layers)
    tr = LayoutGeneratorTrainer(s, lr=1e-3)
    gt = np.random.RandomState(3).randint(0, asm.num_vocab_nmn, size=(T_dec, N)).astype(np.int32)
    nll = []
    for _ in range(50):
        s.forward(seq, lens, use_gt_layout=True, gt_layout_batch=gt, record=True)
        nll.append(float(-s.log_seq_prob.mean()))
        tr.step(d_log_seq_prob=torch.full((N,), -1.0 / N, device='cuda'))
    print('gt-layout NLL %.3f -> %.3f' % (nll[0], nll[-1]))
    assert nll[-1] < 0.5 * nll[0]


def test_joint_gt_layout_step_lowers_total_loss():
    """One composed gt-layout step of the reference (exp_clevr/train_clevr_gt_layout.py:104-124):
    total = avg_sample_loss + seq_likelihood_loss; the module trainer's d_word_vecs handed to the
    generator's trainer."""
    from n2nmn_b200.executor import LayoutExecutor
    from n2nmn_b200.trainer import ModuleNetTrainer, LayoutGeneratorTrainer
    from n2nmn_b200 import weights as wts
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers = 16, 12, 10, 40, 300, 32, 64, 2
    H, W, D, C = 10, 15, 512, 28
    asm = Assembler(synth.vocab_file('clevr'))
    feat, _ = synth.make_inputs(N, H, W, D, T_dec, seed=1)
    gt = synth.expert_mix_tokens(asm, N, T_dec)
    labels = np.random.RandomState(0).randint(0, C, size=N).astype(np.int32)
    w = init_seq2seq_weights(V_txt, E_txt, asm.num_vocab_nmn, E_nmn, L, layers, seed=0)
    rng = np.random.RandomState(1)
    seq = rng.randint(0, V_txt, size=(T_enc, N)).astype(np.int32)
    lens = rng.randint(1, T_enc + 1, size=N).astype(np.int32)
    s = make(asm, w, T_enc, N, T_dec, V_txt, E_txt, E_nmn, L, layers)
    gen_tr = LayoutGeneratorTrainer(s, lr=1e-3)
    featd = torch.from_numpy(feat).cuda()
    wv = s.forward(seq, lens, use_gt_layout=True, gt_layout_batch=gt)[3]
    ex = LayoutExecutor('clevr', featd, wv, C, asm,
                        weights=wts.init_weights('clevr', H, W, D, C, seed=0, bias_std=0.1),
                        max_batch=N, max_T=T_dec)
    mod_tr = ModuleNetTrainer(ex, lr=1e-3)
    totals = []
    for _ in range(20):
        wv = s.forward(seq, lens, use_gt_layout=True, gt_layout_batch=gt, record=True)[3]
        out = mod_tr.train_step(featd, wv, gt, labels)
        nll = float(-s.log_seq_prob.mean())
        totals.append(out['avg_sample_loss'] + nll)
        gen_tr.step(d_log_seq_prob=torch.full((N,), -1.0 / N, device='cuda'),
                    d_word_vecs=out['d_word_vecs'])
    print('joint gt-layout total %.3f -> %.3f' % (totals[0], totals[-1]))
    assert totals[-1] < totals[0]


def test_policy_search_keeps_layouts_valid():
    from n2nmn_b200.trainer import LayoutGeneratorTrainer
    cfg = CFGS['odd']
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers = cfg
    asm, w, seq, lens = problem(cfg)
    s = make(asm, w, T_enc, N, T_dec, V_txt, E_txt, E_nmn, L, layers, decoder_sampling=True)
    tr = LayoutGeneratorTrainer(s, lr=1e-3)
    torch.manual_seed(0)
    for _ in range(15):
        tok = s.forward(seq, lens, record=True)[0]
        assert asm.assemble(tok.cpu().numpy())[1].all()
        coeff = torch.randn(N, device='cuda') / N
        tr.step(d_log_seq_prob=coeff, d_neg_entropy=torch.full((N,), 0.005 / N, device='cuda'))
