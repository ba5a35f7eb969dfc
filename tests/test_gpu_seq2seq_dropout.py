"""GPU: the layout generator's LSTM dropout (encoder_dropout / decoder_dropout,
n2nmn_seq2seq_set_dropout) against the oracle of tests/seq2seq_dropout_oracle.py:
  * the reference's goldens (golden_seq2seq_dropout.npz, 2 and 3 layers, greedy / forced /
    sampled): tokens bit-exact, values within 2e-5 (tests/test_gpu_seq2seq.py's bar);
  * the forward at the CLEVR training size (N=64, T 45/10, lstm 512) and the VQA size (lstm 1000,
    T 26/13, 17,742 words) with encoder-only, decoder-only and both dropouts, forced and sampled,
    ragged lengths, and 3 layers;
  * every variable's gradient within rel_err 5e-3 of the float64 oracle, with d_encoder_states;
  * invariants: flags off = a generator without dropout bit for bit, one layer = no dropout,
    layer 0's encoder state untouched by encoder dropout, all-kept / all-dropped uniforms;
  * default draws in the documented order, launch counts, shape errors, a joint VQA step."""
import os

import numpy as np
import pytest
import torch

from n2nmn_b200 import synth
from n2nmn_b200.assembler import Assembler
from n2nmn_b200.weights import init_seq2seq_weights
from tests import seq2seq_dropout_oracle as sdo

pytestmark = pytest.mark.gpu
ZD = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'golden_seq2seq_dropout.npz'))
ATOL = 2e-5
BAR = 5e-3
#         N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers
CFGS = {'clevr': (64, 45, 10, 90, 300, 300, 512, 2),
        'vqa': (64, 26, 13, 17742, 300, 300, 1000, 2),
        'deep': (37, 26, 13, 90, 300, 300, 40, 3)}


def make(asm, w, cfg, enc=False, dec=False, decoder_sampling=False):
    from n2nmn_b200.seq2seq import AttentionSeq2Seq
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers = cfg
    return AttentionSeq2Seq(None, None, T_dec, V_txt, E_txt, asm.num_vocab_nmn, E_nmn, L, layers,
                            asm, encoder_dropout=enc, decoder_dropout=dec,
                            decoder_sampling=decoder_sampling, T_encoder=T_enc, max_batch=N,
                            weights=w, device='cuda:0')


def problem(cfg, seed=0):
    """(asm, weights, input_seq, lengths 1 ... T_enc)."""
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers = cfg
    asm = Assembler(synth.vocab_file('vqa' if V_txt > 10000 else 'clevr'))
    w = init_seq2seq_weights(V_txt, E_txt, asm.num_vocab_nmn, E_nmn, L, layers, seed=seed)
    rng = np.random.RandomState(seed + 1)
    seq = rng.randint(0, V_txt, size=(T_enc, N)).astype(np.int32)
    lens = ((np.arange(N) * 7) % T_enc + 1).astype(np.int32)
    lens[-1] = T_enc
    return asm, w, seq, lens


def uniforms(cfg, rng, enc, dec):
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers = cfg
    eu = rng.random_sample((T_enc, layers - 1, N, L)).astype(np.float32) if enc else None
    du = rng.random_sample((T_dec, layers - 1, N, L)).astype(np.float32) if dec else None
    return eu, du


def check_forward(out, dec):
    g = [o.cpu().numpy() for o in out]
    assert np.array_equal(g[0], dec[0])
    np.testing.assert_allclose(g[1], dec[1], atol=ATOL)
    np.testing.assert_allclose(g[2], dec[2], atol=10 * ATOL)
    np.testing.assert_allclose(g[3], dec[3], atol=ATOL)
    np.testing.assert_allclose(g[4], dec[4], atol=ATOL)


@pytest.mark.parametrize('layers', [2, 3])
@pytest.mark.parametrize('case', ['greedy', 'gt', 'sample'])
def test_matches_reference_golden(layers, case):
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, _ = [int(v) for v in ZD['cfg']]
    pre = 'l%d_' % layers
    p = pre + case + '_'
    w = {k[len(pre) + 2:]: ZD[k] for k in ZD.files if k.startswith(pre + 'w:')}
    eu, du, su = sdo.golden_uniforms(int(ZD[p + 'uniform_seed']), T_enc, T_dec, layers, N, L)
    asm = Assembler(synth.vocab_file('clevr'))
    cfg = (N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers)
    s = make(asm, w, cfg, True, True, decoder_sampling=case == 'sample')
    kw = dict(use_gt_layout=True, gt_layout_batch=ZD['gt_layout']) if case == 'gt' else {}
    out = s.forward(ZD[pre + 'input_seq'], ZD[pre + 'seq_length'], dropout_uniforms=(eu, du),
                    sample_uniforms=su if case == 'sample' else None, with_encoder_states=True, **kw)
    torch.cuda.synchronize()
    check_forward(out, [ZD[p + k] for k in ('predicted_tokens', 'token_probs', 'neg_entropy',
                                             'word_vecs', 'atts')])
    for l in range(layers):
        np.testing.assert_allclose(s.encoder_states[l][0].cpu().numpy(), ZD[p + 'encoder_c%d' % l], atol=ATOL)
        np.testing.assert_allclose(s.encoder_states[l][1].cpu().numpy(), ZD[p + 'encoder_h%d' % l], atol=ATOL)


FWD = [('clevr', 'enc', 'gt'), ('clevr', 'dec', 'sample'), ('clevr', 'both', 'gt'),
       ('clevr', 'both', 'sample'), ('vqa', 'enc', 'sample'), ('vqa', 'dec', 'gt'),
       ('vqa', 'both', 'gt'), ('vqa', 'both', 'sample'), ('deep', 'both', 'gt'),
       ('deep', 'both', 'sample')]


@pytest.mark.parametrize('size,sides,mode', FWD)
def test_forward_matches_oracle(size, sides, mode):
    cfg = CFGS[size]
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers = cfg
    asm, w, seq, lens = problem(cfg, seed=12)
    rng = np.random.RandomState(20)
    enc, dec = sides in ('enc', 'both'), sides in ('dec', 'both')
    eu, du = uniforms(cfg, rng, enc, dec)
    kw, okw, margins = {}, {}, []
    if mode == 'gt':
        gt = synth.histogram_tokens(asm, synth.VQA_LAYOUTS, N, T_dec, seed=3) if size == 'vqa' \
            else synth.expert_mix_tokens(asm, N, T_dec)
        kw, okw = dict(use_gt_layout=True, gt_layout_batch=gt), dict(use_gt_layout=True, gt_layout=gt)
    else:
        u = rng.random_sample((T_dec, N)).astype(np.float32)
        kw, okw = dict(sample_uniforms=u), dict(sample_uniforms=u, margins=margins)
    _, ref = sdo.run(w, seq, lens, T_dec, layers, asm.P, asm.W, asm.b, enc_u=eu, dec_u=du, **okw)
    if mode == 'sample':
        assert np.min(margins) > 1e-4, np.min(margins)
    s = make(asm, w, cfg, enc, dec, decoder_sampling=mode == 'sample')
    out = s.forward(seq, lens, dropout_uniforms=(eu, du), **kw)
    torch.cuda.synchronize()
    check_forward(out, ref)


def compare(s, ref, label):
    torch.cuda.synchronize()
    worst = []
    for name, g in s.grads().items():
        scale = np.abs(ref[name]).max()
        err = np.abs(g.cpu().numpy().astype(np.float64) - ref[name]).max()
        worst.append((err / scale if scale > 0 else err, name))
    worst.sort(reverse=True)
    print('%s: worst rel_err %s' % (label, ', '.join('%.2e %s' % x for x in worst[:3])))
    assert worst[0][0] <= BAR, worst[:3]


@pytest.mark.parametrize('size,sides,mode', [('clevr', 'both', 'gt'), ('clevr', 'enc', 'sample'),
                                             ('vqa', 'both', 'gt'), ('vqa', 'dec', 'sample'),
                                             ('deep', 'both', 'sample')])
def test_gradients_match_oracle(size, sides, mode):
    cfg = CFGS[size]
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers = cfg
    asm, w, seq, lens = problem(cfg, seed=30)
    rng = np.random.RandomState(31)
    enc, dec = sides in ('enc', 'both'), sides in ('dec', 'both')
    eu, du = uniforms(cfg, rng, enc, dec)
    kw = {}
    if mode == 'gt':
        kw = dict(use_gt_layout=True,
                  gt_layout_batch=rng.randint(0, asm.num_vocab_nmn, size=(T_dec, N)).astype(np.int32))
    u = rng.uniform(size=(T_dec, N)).astype(np.float32) if mode == 'sample' else None
    up = dict(d_log_seq_prob=rng.randn(N).astype(np.float32),
              d_neg_entropy=rng.randn(N).astype(np.float32),
              d_word_vecs=rng.randn(T_dec, N, E_txt).astype(np.float32),
              d_encoder_states=rng.randn(layers, 2, N, L).astype(np.float32))
    s = make(asm, w, cfg, enc, dec, decoder_sampling=mode == 'sample')
    eu_d = torch.as_tensor(eu).cuda() if enc else None
    du_d = torch.as_tensor(du).cuda() if dec else None
    tok = s.forward(seq, lens, sample_uniforms=u, record=True, dropout_uniforms=(eu_d, du_d),
                    **kw)[0].cpu().numpy()
    # the backward reads the recorded keep-masks, not the caller's uniforms: overwrite them (every
    # element dropped) once the forward has read them
    for d in (eu_d, du_d):
        if d is not None:
            d.fill_(0.0)
    torch.cuda.synchronize()
    s.backward(**{k: torch.as_tensor(v).cuda() for k, v in up.items()})
    okw = (dict(use_gt_layout=True, gt_layout=kw['gt_layout_batch']) if mode == 'gt'
           else dict(tokens=tok))
    _, ref = sdo.run_torch(w, seq, lens, T_dec, layers, asm.P, asm.W, asm.b, enc_u=eu, dec_u=du,
                           **okw, **{k: v.astype(np.float64) for k, v in up.items()})
    compare(s, ref, '%s/%s/%s' % (size, sides, mode))


def test_invariants():
    cfg = CFGS['clevr']
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers = cfg
    asm, w, seq, lens = problem(cfg, seed=40)
    gt = synth.expert_mix_tokens(asm, N, T_dec)
    plain = make(asm, w, cfg)
    a = [o.clone() for o in plain.forward(seq, lens, True, gt, with_encoder_states=True)]
    st_a = [x.clone() for x in plain.encoder_states[0]]
    # both flags off: bit-identical to a generator that never had dropout, after dropout forwards
    s = make(asm, w, cfg, True, True)
    s.forward(seq, lens, True, gt)
    s.encoder_dropout = s.decoder_dropout = False
    b = [o.clone() for o in s.forward(seq, lens, True, gt)]
    torch.cuda.synchronize()
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    # encoder dropout leaves layer 0's final state alone (and changes the outputs)
    s.encoder_dropout = True
    c = s.forward(seq, lens, True, gt, with_encoder_states=True)
    torch.cuda.synchronize()
    assert torch.equal(s.encoder_states[0][0], st_a[0]) and torch.equal(s.encoder_states[0][1], st_a[1])
    assert not torch.equal(s.encoder_states[1][1], plain.encoder_states[1][1])
    assert not torch.equal(c[1], a[1])
    # all kept / all dropped against the oracle
    for val in (0.5, 0.4999):
        eu = np.full((T_enc, layers - 1, N, L), val, np.float32)
        du = np.full((T_dec, layers - 1, N, L), val, np.float32)
        s.encoder_dropout = s.decoder_dropout = True
        out = s.forward(seq, lens, True, gt, dropout_uniforms=(eu, du))
        _, ref = sdo.run(w, seq, lens, T_dec, layers, asm.P, asm.W, asm.b, use_gt_layout=True,
                         gt_layout=gt, enc_u=eu, dec_u=du)
        torch.cuda.synchronize()
        check_forward(out, ref)
    # one layer: dropout on changes nothing and draws nothing
    cfg1 = (N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, 1)
    asm1, w1, _, _ = problem(cfg1, seed=42)
    one = make(asm1, w1, cfg1)
    one_d = make(asm1, w1, cfg1, True, True)
    x = [o.clone() for o in one.forward(seq, lens, True, gt)]
    torch.manual_seed(3)
    y = [o.clone() for o in one_d.forward(seq, lens, True, gt)]
    after = torch.rand(4, device='cuda')
    torch.manual_seed(3)
    torch.cuda.synchronize()
    assert torch.equal(after, torch.rand(4, device='cuda'))
    for p, q in zip(x, y):
        assert torch.equal(p, q)


def test_default_draws_follow_the_documented_order():
    cfg = CFGS['deep']
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers = cfg
    asm, w, seq, lens = problem(cfg, seed=60)
    s = make(asm, w, cfg, True, True, decoder_sampling=True)
    torch.manual_seed(5)
    a = [o.clone() for o in s.forward(seq, lens)]
    torch.manual_seed(5)
    u = torch.rand((T_dec, N), device='cuda')
    eu = torch.rand((T_enc, layers - 1, N, L), device='cuda')
    du = torch.rand((T_dec, layers - 1, N, L), device='cuda')
    b = [o.clone() for o in s.forward(seq, lens, sample_uniforms=u, dropout_uniforms=(eu, du))]
    torch.cuda.synchronize()
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    # without dropout the generator is consumed exactly as before: one [T_dec, N] draw
    s.encoder_dropout = s.decoder_dropout = False
    torch.manual_seed(6)
    c = [o.clone() for o in s.forward(seq, lens)]
    after = torch.rand(3, device='cuda')
    torch.manual_seed(6)
    u = torch.rand((T_dec, N), device='cuda')
    d = [o.clone() for o in s.forward(seq, lens, sample_uniforms=u)]
    torch.cuda.synchronize()
    assert torch.equal(after, torch.rand(3, device='cuda'))
    for x, y in zip(c, d):
        assert torch.equal(x, y)


@pytest.mark.parametrize('size', ['clevr', 'deep'])
def test_launch_counts_do_not_change(size):
    cfg = CFGS[size]
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers = cfg
    asm, w, seq, lens = problem(cfg, seed=70)
    gt = synth.expert_mix_tokens(asm, N, T_dec)
    dlp = torch.full((N,), -1.0 / N, device='cuda')
    counts = []
    for enc, dec in ((False, False), (True, True), (True, False), (False, True)):
        s = make(asm, w, cfg, enc, dec)
        s.forward(seq, lens, True, gt, record=True)
        s.backward(d_log_seq_prob=dlp)                      # prepare() and the transposes, once
        n0 = s.launch_count()
        s.forward(seq, lens, True, gt, record=True)
        n1 = s.launch_count()
        s.backward(d_log_seq_prob=dlp)
        n2 = s.launch_count()
        counts.append((n1 - n0, n2 - n1))
    fwd = (T_enc + layers - 1) + layers * T_dec + 2 * T_dec + 3
    bwd = 14 + 2 * layers * T_dec + 2 * (T_enc + layers - 1) + 4 * layers
    assert all(c == (fwd, bwd) for c in counts), (counts, fwd, bwd)
    print('%s: forward %d, backward %d launches with and without dropout' % (size, fwd, bwd))


def test_wrong_uniform_shapes_raise():
    cfg = CFGS['deep']
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers = cfg
    asm, w, seq, lens = problem(cfg, seed=80)
    s = make(asm, w, cfg, True, True)
    good_e = np.zeros((T_enc, layers - 1, N, L), np.float32)
    good_d = np.zeros((T_dec, layers - 1, N, L), np.float32)
    for bad in [(good_e[:, :1], good_d), (good_e, good_d[1:]), (good_e[..., :8], good_d),
                (good_e, good_d[:, :, :5]), (good_e,)]:
        with pytest.raises(ValueError):
            s.forward(seq, lens, dropout_uniforms=bad)
    s.decoder_dropout = False
    with pytest.raises(ValueError):
        s.forward(seq, lens, dropout_uniforms=(good_e, good_d))   # numbers for a side that is off
    s.forward(seq, lens, dropout_uniforms=(good_e, None))


def test_joint_vqa_gt_layout_step_with_dropout():
    """INTEGRATION §2b's joint step (exp_vqa/train_vqa_gt_layout.py, use_qpn) with the scripts'
    encoder_dropout = decoder_dropout = True: the module network's trainer gives d_word_vecs and
    d_scores, d_scores goes back through a torch question-prior net to the encoder states. The
    generator's gradient matches the oracle's for the same upstreams and uniforms, and its clip +
    Adam step runs after the dropout forward."""
    from n2nmn_b200 import weights as wts
    from n2nmn_b200.executor import LayoutExecutor
    from n2nmn_b200.trainer import LayoutGeneratorTrainer, ModuleNetTrainer
    cfg = CFGS['vqa']
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers = cfg
    H, W, D, C = 14, 14, 2048, 3001
    asm, w, seq, lens = problem(cfg, seed=50)
    feat, _ = synth.make_inputs(N, H, W, D, T_dec, seed=51)
    gt = synth.histogram_tokens(asm, synth.VQA_LAYOUTS, N, T_dec, seed=52)
    labels = np.random.RandomState(53).randint(0, C, size=N).astype(np.int32)
    s = make(asm, w, cfg, True, True)
    gen_tr = LayoutGeneratorTrainer(s, lr=1e-3, weight_decay=0.0)
    eu, du = uniforms(cfg, np.random.RandomState(54), True, True)
    featd = torch.from_numpy(feat).cuda()
    wv = s.forward(seq, lens, use_gt_layout=True, gt_layout_batch=gt, record=True,
                   with_encoder_states=True, dropout_uniforms=(eu, du))[3]
    ex = LayoutExecutor('vqa', featd, wv, C, asm,
                        weights=wts.init_weights('vqa', H, W, D, C, seed=0, bias_std=0.1),
                        max_batch=N, max_T=T_dec)
    mod_tr = ModuleNetTrainer(ex, lr=1e-3, weight_decay=0.0)
    torch.manual_seed(0)
    qpn = torch.nn.Sequential(torch.nn.Linear(layers * L, 500), torch.nn.ReLU(),
                              torch.nn.Linear(500, C)).cuda()
    h = torch.cat([hl for _, hl in s.encoder_states], dim=1).detach().requires_grad_(True)
    prior = qpn(h)
    out = mod_tr.train_step(featd, wv, gt, labels, score_prior=prior.detach())
    prior.backward(out['d_scores'])
    d_states = torch.zeros(layers, 2, N, L, device='cuda')
    d_states[:, 1] = h.grad.view(N, layers, L).permute(1, 0, 2)
    dlp = torch.full((N,), -1.0 / N, device='cuda')
    s.backward(d_log_seq_prob=dlp, d_word_vecs=out['d_word_vecs'], d_encoder_states=d_states)
    torch.cuda.synchronize()
    _, ref = sdo.run_torch(w, seq, lens, T_dec, layers, asm.P, asm.W, asm.b, use_gt_layout=True,
                           gt_layout=gt, enc_u=eu, dec_u=du,
                           d_log_seq_prob=dlp.cpu().numpy().astype(np.float64),
                           d_word_vecs=out['d_word_vecs'].cpu().numpy().astype(np.float64),
                           d_encoder_states=d_states.cpu().numpy().astype(np.float64))
    compare(s, ref, 'joint vqa step')
    w0 = gen_tr.w.clone()
    gen_tr.step(d_log_seq_prob=dlp, d_word_vecs=out['d_word_vecs'], d_encoder_states=d_states)
    torch.cuda.synchronize()
    assert torch.isfinite(gen_tr.w).all() and not torch.equal(gen_tr.w, w0)
