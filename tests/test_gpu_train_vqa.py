"""GPU: VQA training — backward pass at map_dim 1024 with many-class answer heads and the
question-prior logits (exp_vqa/train_vqa_rl_gt_layout.py:101-142) vs the torch-autograd oracle
(oracle/nmn_oracle_torch.py, family='vqa', with the VQA loss of tests/vqa_loss_oracle.py)."""
import numpy as np
import pytest
import torch

from n2nmn_b200 import _lib, synth, weights as wts
from n2nmn_b200.assembler import Assembler
from oracle import nmn_oracle_torch as ot
from tests import vqa_loss_oracle as vo

pytestmark = pytest.mark.gpu

INVALID = ['_Find', '_Transform']     # no answer module: does not assemble


def make(N, H, Wd, D, T, Cc, flags=0, seed=0, **ctx):
    from n2nmn_b200.executor import LayoutExecutor
    from n2nmn_b200.trainer import ModuleNetTrainer
    feat, word_vecs = synth.make_inputs(N, H, Wd, D, T, seed=60 + seed)
    W = wts.init_weights('vqa', H, Wd, D, Cc, seed=seed, bias_std=0.1)
    asm = Assembler(synth.vocab_file('vqa'))
    ex = LayoutExecutor('vqa', torch.from_numpy(feat).cuda(), torch.from_numpy(word_vecs).cuda(),
                        Cc, asm, weights=W, flags=flags, **ctx)
    return feat, word_vecs, W, asm, ex, ModuleNetTrainer(ex, weight_decay=0.0)


def rel_err(a, b, scale=0.0):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b)) / (max(np.max(np.abs(b)), scale) + 1e-12))


def grad_errs(got, ref):
    """Relative error of every variable's gradient. conv_eltwise/biases is the exception: its
    gradient is Σ_p d loss / d map[p] over the Find / Transform maps, and in these layouts every
    map reaches the loss through the softmax of an attention pooling (Describe, Transform), whose
    input gradient sums to zero over the pixels (And passes each pixel to one input). The
    reference is then rounding noise (~1e-10), so the error is taken on the scale of the
    layer's weight gradient."""
    errs = {}
    for n, g in got.items():
        scale = 0.0
        if n.endswith('conv_eltwise/biases'):
            scale = float(np.max(np.abs(ref[n[:-len('biases')] + 'weights'])))
        errs[n] = rel_err(g, ref[n], scale)
    return errs


def layouts_with_invalid(N):
    real = [l for l, _ in synth.VQA_LAYOUTS]
    return [real[i % len(real)] for i in range(N - 1)] + [INVALID]


def check_against_autograd(N, H, Wd, D, T, Cc, flags, tol, seed):
    feat, word_vecs, W, asm, ex, tr = make(N, H, Wd, D, T, Cc, flags=flags, seed=seed)
    tokens = synth.tokens_from_layouts(asm, layouts_with_invalid(N), T)
    labels = (np.arange(N) * 7 + 3) % Cc
    prior = np.random.RandomState(seed).standard_normal((N, Cc)).astype(np.float32)
    scores, valid, per_sample, dword, dscores = tr.forward_backward(
        torch.from_numpy(feat).cuda(), torch.from_numpy(word_vecs).cuda(), tokens, labels,
        score_prior=torch.from_numpy(prior).cuda())
    torch.cuda.synchronize()
    exprs, pv = asm.assemble(tokens)
    assert valid.tolist() == pv.tolist() and not valid[-1] and valid[:-1].all()
    m = ot.TorchOracleModules(feat, word_vecs, Cc, W, family='vqa')
    ref_s, ref_per, ref_avg, ref_g, ref_gwv, ref_gprior = vo.loss_and_grads(
        m, exprs, pv, labels, score_prior=prior, ce_every_row=True)
    assert np.max(np.abs(scores.cpu().numpy() - ref_s)) <= 1e-3
    np.testing.assert_allclose(per_sample.cpu().numpy(), ref_per, atol=1e-3)
    assert abs(float(tr._loss[0]) / N - ref_avg) <= 1e-3
    errs = grad_errs({n: g.cpu().numpy() for n, g in tr.grads().items()}, ref_g)
    errs['word_vecs'] = rel_err(dword.cpu().numpy(), ref_gwv)
    errs['d_scores'] = rel_err(dscores.cpu().numpy(), ref_gprior)
    print('flags', flags, 'worst relative gradient errors:',
          sorted(errs.items(), key=lambda kv: -kv[1])[:6])
    bad = {k: v for k, v in errs.items() if not v <= tol}
    assert not bad, bad
    # every weight matrix of the family is trained (image_feat_grid itself gets no gradient)
    assert all(np.abs(ref_g[n]).max() > 0 for n in ref_g if n.endswith('weights'))


@pytest.mark.parametrize('flags,tol', [(_lib.FLAG_PROJ_FP32_SIMT, 2e-4), (0, 5e-3)])
def test_vqa_backward_matches_autograd(flags, tol):
    check_against_autograd(12, 14, 14, 512, 13, 3001, flags, tol, seed=3)


def test_vqa_backward_matches_autograd_at_reference_depth_2048():
    """res5c depth: Dk = 2050, a ragged last 128-feature slab of the wgmma weight gradient."""
    check_against_autograd(6, 14, 14, 2048, 13, 3001, 0, 5e-3, seed=4)


def test_vqa_backward_small_odd_shapes():
    """The golden VQA sizes: Dk = 40 (mma.sync weight gradient over a re-pitched copy) and the
    many-class tail at a small C."""
    check_against_autograd(6, 14, 14, 38, 8, 37, 0, 5e-3, seed=5)


def test_vqa_wgmma_weight_gradient_equals_mma_sync_path_at_batch_64(monkeypatch):
    """The wgmma weight gradient at the VQA shapes (Mp = 1024: four 256-channel tiles; Dk = 2050:
    ragged last slab; coordinate-augmented feature copy) against xtb_mma_kernel
    (N2NMN_WGRAD_MMA_SYNC=1). TF32 operands truncated vs rounded: 2e-3 of the largest entry for
    the weights, fp32 accuracy for the biases; the two must differ, or the wgmma path was not
    taken."""
    N, H, Wd, D, T, Cc = 64, 14, 14, 2048, 13, 3001
    feat, word_vecs, W, asm, ex, tr = make(N, H, Wd, D, T, Cc, seed=11)
    tokens = synth.histogram_tokens(asm, synth.VQA_LAYOUTS, N, T, seed=12)
    labels = (np.arange(N) * 13) % Cc
    f, w = torch.from_numpy(feat).cuda(), torch.from_numpy(word_vecs).cuda()

    def grads():
        tr.forward_backward(f, w, tokens, labels)
        torch.cuda.synchronize()
        return {n: g.cpu().numpy().copy() for n, g in tr.grads().items()}
    monkeypatch.setenv('N2NMN_WGRAD_MMA_SYNC', '1')
    ref = grads()
    monkeypatch.delenv('N2NMN_WGRAD_MMA_SYNC')
    new = grads()
    checked = differ = 0
    errs = grad_errs(new, ref)
    for n in ref:
        if 'conv_image' in n or 'fc_att' in n:
            tol = 2e-3 if n.endswith('weights') else 1e-5
            assert rel_err(new[n], ref[n]) <= tol, (n, rel_err(new[n], ref[n]))
            assert np.abs(ref[n]).max() > 0
            if n.endswith('weights'):
                differ += int(not np.array_equal(new[n], ref[n]))
                # the coordinate channels (last two rows) are trained
                assert np.abs(ref[n][-2:]).max() > 0, n
            checked += 1
        else:   # same kernels, fp32 atomics in a different order
            assert errs[n] <= 3e-4, (n, errs[n])
    assert checked == 8 and differ == 4


def test_vqa_train_steps_reduce_the_loss():
    N, H, Wd, D, T, Cc = 32, 14, 14, 512, 13, 37
    feat, word_vecs, W, asm, ex, tr = make(N, H, Wd, D, T, Cc, seed=9)
    tr.hyper['lr'] = 1e-3
    tokens = synth.histogram_tokens(asm, synth.VQA_LAYOUTS, N, T, seed=10)
    labels = np.arange(N) % Cc
    f, w = torch.from_numpy(feat).cuda(), torch.from_numpy(word_vecs).cuda()
    prior = torch.from_numpy(
        0.1 * np.random.RandomState(2).standard_normal((N, Cc)).astype(np.float32)).cuda()
    lsp = torch.full((N,), -3.0, device='cuda')
    losses = []
    for _ in range(30):
        out = tr.train_step(f, w, tokens, labels, log_seq_prob=lsp, score_prior=prior)
        losses.append(out['avg_sample_loss'])
    print('loss curve', [round(l, 3) for l in losses[::5]])
    assert losses[-1] < 0.6 * losses[0]
    assert out['d_scores'].shape == (N, Cc) and np.isfinite(out['total_loss'])


def test_vqa_capacity_overflow_raises():
    """Long Transform chains need two B maps per Transform node: 14 per question, more than the
    context made for T = 9 holds."""
    N, H, Wd, D, T, Cc = 4, 14, 14, 64, 9, 37
    feat, word_vecs, W, asm, ex, tr = make(N, H, Wd, D, T, Cc, seed=13, max_batch=N, max_T=T)
    chain = ['_Find'] + ['_Transform'] * 6 + ['_Describe']
    tokens = synth.tokens_from_layouts(asm, [chain] * N, T)
    with pytest.raises(_lib.N2NMNError, match='error -5'):
        tr.forward_backward(torch.from_numpy(feat).cuda(), torch.from_numpy(word_vecs).cuda(),
                            tokens, np.zeros(N, np.int32))
