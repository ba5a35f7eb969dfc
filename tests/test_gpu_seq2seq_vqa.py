"""GPU: the layout generator at the VQA scripts' size (exp_vqa/train_vqa*.py, eval_vqa*.py:
lstm_dim 1000, 2 layers, T_encoder 26, T_decoder 13, embed_dim_txt 300 over the 17,742-word
vocabulary_vqa.txt; batch 64; the VQA Assembler's 5 layout tokens) with random weights:
  * forward against the numpy oracle in greedy, sampled and teacher-forced decoding (tokens
    bit-exact, guarded by the greedy top-2 score gap and the sampled draws' distance from a CDF
    boundary; values within tests/test_gpu_seq2seq.py's 2e-5), the encoder's final state included;
    also at N = 1 and at N = 37 / lstm_dim 40 / 3 layers, with lengths 1 ... T_enc;
  * every variable's gradient against the float64 oracle with all four upstreams (d_log_seq_prob,
    d_neg_entropy, d_word_vecs, d_encoder_states): max|Δ| / max|ref| <= 5e-3;
  * the encoder states and their gradient leave everything else bit-identical, launch counts;
  * a joint VQA gt-layout step with a question-prior net over the encoder states, and
    evaluate_split with score_prior_fn."""
import numpy as np
import pytest
import torch

from n2nmn_b200 import _lib, synth
from n2nmn_b200.assembler import Assembler
from n2nmn_b200.weights import init_seq2seq_weights
from oracle import seq2seq_oracle as so
from oracle import seq2seq_oracle_torch as sot
from tests import seq2seq_states_oracle as sso

pytestmark = pytest.mark.gpu
ATOL = 2e-5
BAR = 5e-3
#        N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers
CFGS = {'vqa': (64, 26, 13, 17742, 300, 300, 1000, 2),
        'one': (1, 26, 13, 17742, 300, 300, 1000, 2),
        'small': (37, 26, 13, 90, 300, 300, 40, 3)}


def make(asm, w, cfg, decoder_sampling=False):
    from n2nmn_b200.seq2seq import AttentionSeq2Seq
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers = cfg
    return AttentionSeq2Seq(None, None, T_dec, V_txt, E_txt, asm.num_vocab_nmn, E_nmn, L, layers,
                            asm, T_encoder=T_enc, max_batch=N, weights=w, device='cuda:0',
                            decoder_sampling=decoder_sampling)


def problem(cfg, seed=0):
    """(asm, weights, input_seq, lengths): lengths cycle through 1 ... T_enc."""
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers = cfg
    asm = Assembler(synth.vocab_file('vqa'))
    w = init_seq2seq_weights(V_txt, E_txt, asm.num_vocab_nmn, E_nmn, L, layers, seed=seed)
    rng = np.random.RandomState(seed + 1)
    seq = rng.randint(0, V_txt, size=(T_enc, N)).astype(np.int32)
    lens = ((np.arange(N) * 7) % T_enc + 1).astype(np.int32)
    lens[-1] = T_enc
    return asm, w, seq, lens


def states_of(s):
    return torch.stack([torch.stack([c, h]) for c, h in s.encoder_states]).cpu().numpy()


@pytest.mark.parametrize('size', list(CFGS))
@pytest.mark.parametrize('mode', ['greedy', 'sample', 'gt'])
def test_forward_matches_oracle(size, mode):
    cfg = CFGS[size]
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers = cfg
    asm, w, seq, lens = problem(cfg, seed=12)
    rng = np.random.RandomState(20)
    kw, okw, margins = {}, {}, []
    if mode == 'gt':
        gt = synth.histogram_tokens(asm, synth.VQA_LAYOUTS, N, T_dec, seed=3)
        kw = dict(use_gt_layout=True, gt_layout_batch=gt)
        okw = dict(use_gt_layout=True, gt_layout=gt)
    elif mode == 'sample':
        u = rng.random_sample((T_dec, N)).astype(np.float32)
        kw = dict(sample_uniforms=u)
        okw = dict(sample_uniforms=u, margins=margins)
    enc, dec = so.run(w, seq, lens, T_dec, layers, asm.P, asm.W, asm.b, **okw)
    if mode == 'sample':
        assert np.min(margins) > 1e-4, np.min(margins)
    if mode == 'greedy':
        gaps = sso.greedy_margins(w, enc, dec[0], T_dec, layers, asm.P, asm.W, asm.b)
        assert np.min(gaps) > 1e-4, np.min(gaps)
    s = make(asm, w, cfg, decoder_sampling=mode == 'sample')
    out = s.forward(seq, lens, with_encoder_states=True, **kw)
    torch.cuda.synchronize()
    g = [o.cpu().numpy() for o in out]
    assert np.array_equal(g[0], dec[0])
    np.testing.assert_allclose(g[1], dec[1], atol=ATOL)
    np.testing.assert_allclose(g[2], dec[2], atol=10 * ATOL)
    np.testing.assert_allclose(g[3], dec[3], atol=ATOL)
    np.testing.assert_allclose(g[4], dec[4], atol=ATOL)
    assert len(s.encoder_states) == layers
    assert all(c.shape == (N, L) and h.shape == (N, L) for c, h in s.encoder_states)
    np.testing.assert_allclose(states_of(s), sso.encoder_states(enc), atol=ATOL)
    if mode != 'gt':
        assert asm.assemble(g[0])[1].all()


def upstreams(cfg, rng):
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers = cfg
    return dict(d_log_seq_prob=rng.randn(N).astype(np.float32),
                d_neg_entropy=rng.randn(N).astype(np.float32),
                d_word_vecs=rng.randn(T_dec, N, E_txt).astype(np.float32),
                d_encoder_states=rng.randn(layers, 2, N, L).astype(np.float32))


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


@pytest.mark.parametrize('size', ['vqa', 'small'])
@pytest.mark.parametrize('mode', ['gt', 'sample', 'greedy'])
def test_gradients_match_oracle(size, mode):
    cfg = CFGS[size]
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers = cfg
    asm, w, seq, lens = problem(cfg, seed=30)
    rng = np.random.RandomState(31)
    kw = {}
    if mode == 'gt':
        kw = dict(use_gt_layout=True,
                  gt_layout_batch=rng.randint(0, asm.num_vocab_nmn, size=(T_dec, N)).astype(np.int32))
    u = rng.uniform(size=(T_dec, N)).astype(np.float32) if mode == 'sample' else None
    up = upstreams(cfg, rng)
    s = make(asm, w, cfg, decoder_sampling=mode == 'sample')
    tok = s.forward(seq, lens, sample_uniforms=u, record=True, **kw)[0].cpu().numpy()
    d_states = torch.as_tensor(up['d_encoder_states']).cuda()
    s.backward(**{k: torch.as_tensor(v).cuda() for k, v in up.items() if k != 'd_encoder_states'},
               d_encoder_states=tuple((d_states[l, 0], d_states[l, 1]) for l in range(layers)))
    okw = (dict(use_gt_layout=True, gt_layout=kw['gt_layout_batch']) if mode == 'gt'
           else dict(tokens=tok))
    _, ref = sot.run(w, seq, lens, T_dec, layers, asm.P, asm.W, asm.b, **okw,
                     **{k: v.astype(np.float64) for k, v in up.items() if k != 'd_encoder_states'})
    _, ref_st = sso.states_and_grads(w, seq, lens, layers,
                                     up['d_encoder_states'].astype(np.float64))
    ref = sso.add_grads(ref, ref_st)
    compare(s, ref, '%s/%s' % (size, mode))


def test_encoder_states_leave_everything_else_bit_identical_and_launch_counts():
    cfg = CFGS['vqa']
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers = cfg
    asm, w, seq, lens = problem(cfg, seed=40)
    s = make(asm, w, cfg)
    s.forward(seq, lens)                                  # prepare() runs here
    n0 = s.launch_count()
    a = [o.clone() for o in s.forward(seq, lens)]
    n1 = s.launch_count()
    assert s.encoder_states is None
    b = [o.clone() for o in s.forward(seq, lens, with_encoder_states=True)]
    n2 = s.launch_count()
    want = (T_enc + layers - 1) + layers * T_dec + 2 * T_dec + 3
    assert want == 82
    assert n1 - n0 == want and n2 - n1 == want, (n1 - n0, n2 - n1)
    c = [o.clone() for o in s.forward(seq, lens, record=True, with_encoder_states=True)]
    torch.cuda.synchronize()
    for x, y, z in zip(a, b, c):
        assert torch.equal(x, y) and torch.equal(x, z)
    # backward: a zero d_encoder_states gives the NULL call's gradient, one launch more. The
    # LSTM cell matrices' gradients have no atomics at this size (s2s_xtb_kernel has >= 1323 tiles
    # per matrix, so it does not split the rows): they are the same bit for bit. The others are
    # summed with atomics in an order that varies from call to call, even between two NULL calls:
    # they agree to summation-order rounding (a bias gradient is a sum that largely cancels, so
    # that rounding is ~1e-5 of its largest entry).
    dlp = torch.full((N,), -1.0 / N, device='cuda')
    dwv = torch.randn(T_dec, N, E_txt, device='cuda')
    s.backward(d_log_seq_prob=dlp, d_word_vecs=dwv)       # the transposes, once
    n3 = s.launch_count()
    g0 = s.backward(d_log_seq_prob=dlp, d_word_vecs=dwv).clone()
    n4 = s.launch_count()
    g1 = s.backward(d_log_seq_prob=dlp, d_word_vecs=dwv,
                    d_encoder_states=torch.zeros(layers, 2, N, L, device='cuda')).clone()
    n5 = s.launch_count()
    torch.cuda.synchronize()
    v0, v1 = s._views(g0), s._views(g1)
    exact = [n for n in v0 if n.endswith('/basic_lstm_cell/weights')]
    assert len(exact) == 2 * layers
    for name in v0:
        if name in exact:
            assert torch.equal(v0[name], v1[name]), name
        else:
            scale = float(v0[name].abs().max())
            assert float((v0[name] - v1[name]).abs().max()) <= 1e-3 * scale, name
    assert n4 - n3 == 14 + 2 * layers * T_dec + 2 * (T_enc + layers - 1) + 4 * layers
    assert n5 - n4 == n4 - n3 + 1
    print('VQA size: forward %d launches, backward %d (+1 with d_encoder_states)' % (want, n4 - n3))
    # d_encoder_states alone reaches exactly the encoder's LSTM variables and embedding
    s.backward(d_encoder_states=torch.randn(layers, 2, N, L, device='cuda'))
    g = s.grads()
    for name, v in g.items():
        if name.startswith('encoder/lstm/') or name == 'encoder/embedding_mat':
            assert (v != 0).any(), name
        else:
            assert (v == 0).all(), name


def test_lstm_dim_not_a_multiple_of_8_is_refused():
    cfg = (4, 26, 13, 100, 300, 300, 1004, 2)
    asm, w, seq, lens = problem(cfg)
    with pytest.raises(_lib.N2NMNError, match='multiple of 8'):
        make(asm, None, cfg)
    s = make(asm, None, (4, 26, 13, 100, 300, 300, 1000, 2))     # 1000 is accepted
    assert s.lstm_dim == 1000


class QuestionPriorNet(torch.nn.Module):
    """models_vqa/question_prior_net.py without dropout: fc_relu(500) and fc(num_choices) over
    the concatenated h of every encoder layer."""

    def __init__(self, in_dim, num_choices, hidden_dim=500):
        super().__init__()
        self.fc1 = torch.nn.Linear(in_dim, hidden_dim)
        self.fc2 = torch.nn.Linear(hidden_dim, num_choices)

    def forward(self, h_concat):
        return self.fc2(torch.relu(self.fc1(h_concat)))


def test_joint_vqa_gt_layout_step_lowers_total_loss():
    """exp_vqa/train_vqa_gt_layout.py with use_qpn: scores = scores_nmn + question_prior_net(
    encoder_states), total = avg_sample_loss + seq_likelihood_loss. The module network's trainer
    gives d_scores and d_word_vecs; d_scores runs back through the prior net (torch) to the
    encoder states, whose gradient goes to the generator's trainer with d_log_seq_prob = -1/N."""
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
    s = make(asm, w, cfg)
    gen_tr = LayoutGeneratorTrainer(s, lr=1e-3, weight_decay=0.0)
    featd = torch.from_numpy(feat).cuda()
    wv = s.forward(seq, lens, use_gt_layout=True, gt_layout_batch=gt)[3]
    ex = LayoutExecutor('vqa', featd, wv, C, asm,
                        weights=wts.init_weights('vqa', H, W, D, C, seed=0, bias_std=0.1),
                        max_batch=N, max_T=T_dec)
    mod_tr = ModuleNetTrainer(ex, lr=1e-3, weight_decay=0.0)
    torch.manual_seed(0)
    qpn = QuestionPriorNet(layers * L, C).cuda()
    qpn_opt = torch.optim.Adam(qpn.parameters(), lr=1e-3)
    totals = []
    for _ in range(30):
        wv = s.forward(seq, lens, use_gt_layout=True, gt_layout_batch=gt, record=True,
                       with_encoder_states=True)[3]
        h = torch.cat([hl for _, hl in s.encoder_states], dim=1).detach().requires_grad_(True)
        prior = qpn(h)
        out = mod_tr.train_step(featd, wv, gt, labels, score_prior=prior.detach())
        nll = float(-s.log_seq_prob.mean())
        totals.append(out['avg_sample_loss'] + nll)
        qpn_opt.zero_grad()
        prior.backward(out['d_scores'])
        qpn_opt.step()
        dh = h.grad.view(N, layers, L)
        d_states = torch.zeros(layers, 2, N, L, device='cuda')
        d_states[:, 1] = dh.permute(1, 0, 2)
        gen_tr.step(d_log_seq_prob=torch.full((N,), -1.0 / N, device='cuda'),
                    d_word_vecs=out['d_word_vecs'], d_encoder_states=d_states)
    print('joint VQA gt-layout total %.3f -> %.3f' % (totals[0], totals[-1]))
    assert np.isfinite(totals).all()
    assert totals[-1] < totals[0]


def test_evaluate_split_adds_the_score_prior():
    """eval_vqa.py with use_qpn: the answer is argmax(scores_nmn + scores_qpn)."""
    from n2nmn_b200 import evaluate as ev
    from n2nmn_b200 import weights as wts
    from n2nmn_b200.executor import ExecutorPool, LayoutExecutor
    N, H, W, D, T, C = 16, 14, 14, 64, 13, 37
    asm = Assembler(synth.vocab_file('vqa'))
    weights = wts.init_weights('vqa', H, W, D, C, seed=1, bias_std=0.1)
    rng = np.random.RandomState(60)
    batches, wvs, priors, want_nmn, want_sum = [], [], [], [], []
    for i in range(3):
        feat, wv = synth.make_inputs(N, H, W, D, T, seed=61 + i)
        tok = synth.histogram_tokens(asm, synth.VQA_LAYOUTS, N, T, seed=70 + i)
        batches.append({'image_feat_batch': feat, 'gt_layout_batch': tok,
                        'answer_label_batch': rng.randint(0, C, size=N).astype(np.int32), 'i': i})
        wvs.append(torch.from_numpy(wv).cuda())
        ex = LayoutExecutor('vqa', torch.from_numpy(feat).cuda(), wvs[-1], C, asm, weights=weights)
        sc = ex.forward_tokens(tok)[0]
        torch.cuda.synchronize()
        sc = sc.cpu().numpy()
        prior = (3 * rng.standard_normal((N, C))).astype(np.float32)
        priors.append(prior)
        want_nmn.extend(np.argmax(sc, axis=1))
        want_sum.extend(np.argmax(sc + prior, axis=1))
    answers = [str(c) for c in range(C)]
    pool = ExecutorPool('vqa', torch.from_numpy(batches[0]['image_feat_batch']).cuda(), wvs[0], C,
                        asm, weights=weights, num_streams=2)
    res = ev.evaluate_split(pool, batches, asm, answers, 'synthetic',
                            word_vecs_fn=lambda b: wvs[b['i']])
    assert res['output_answers'] == [str(a) for a in want_nmn]
    res = ev.evaluate_split(pool, batches, asm, answers, 'synthetic',
                            word_vecs_fn=lambda b: wvs[b['i']],
                            score_prior_fn=lambda b: torch.from_numpy(priors[b['i']]).cuda())
    assert res['output_answers'] == [str(a) for a in want_sum]
    assert want_sum != want_nmn
