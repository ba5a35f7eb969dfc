"""GPU: backward pass and optimiser step (SURVEY.md §8 a20 / config 3) vs the torch-autograd
oracle with TF's gradient conventions (oracle/nmn_oracle_torch.py)."""
import ctypes as C

import numpy as np
import pytest
import torch

from n2nmn_b200 import _lib, synth, weights as wts
from n2nmn_b200.assembler import Assembler
from oracle import nmn_oracle_torch as ot

pytestmark = pytest.mark.gpu


def make(family, N, H, Wd, D, T, Cc, flags=0, seed=0, tokens_fn=None):
    from n2nmn_b200.executor import LayoutExecutor
    from n2nmn_b200.trainer import ModuleNetTrainer
    feat, word_vecs = synth.make_inputs(N, H, Wd, D, T, seed=50 + seed)
    W = wts.init_weights(family, H, Wd, D, Cc, seed=seed, bias_std=0.1)
    asm = Assembler(synth.vocab_file(family))
    ex = LayoutExecutor(family, torch.from_numpy(feat).cuda(), torch.from_numpy(word_vecs).cuda(),
                        Cc, asm, weights=W, flags=flags)
    return feat, word_vecs, W, asm, ex, ModuleNetTrainer(ex)


def rel_err(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b)) / (np.max(np.abs(b)) + 1e-12))


@pytest.mark.parametrize('flags,tol', [(_lib.FLAG_PROJ_FP32_SIMT, 2e-4), (0, 5e-3)])
def test_clevr_backward_matches_autograd(flags, tol):
    N, H, Wd, D, T, Cc = 12, 10, 15, 512, 12, 28
    feat, word_vecs, W, asm, ex, tr = make('clevr', N, H, Wd, D, T, Cc, flags=flags, seed=3)
    layouts = [synth.CLEVR_EXPERT_MIX[i % 10] for i in range(10)] + \
        [['_Find', '_Find', '_Or', '_Find', '_Filter', '_MoreNum'], ['_Find', '_Transform']]
    tokens = synth.tokens_from_layouts(asm, layouts, T)
    labels = (np.arange(N) * 5) % Cc
    scores, valid, per_sample, dword = tr.forward_backward(
        torch.from_numpy(feat).cuda(), torch.from_numpy(word_vecs).cuda(), tokens, labels)
    torch.cuda.synchronize()
    exprs, pv = asm.assemble(tokens)
    assert valid.tolist() == pv.tolist() and not valid[-1]
    m = ot.TorchOracleModules(feat, word_vecs, Cc, W)
    ref_s, ref_per, ref_avg, ref_g, ref_gwv = ot.loss_and_grads(m, exprs, pv, labels)
    assert np.max(np.abs(scores.cpu().numpy() - ref_s)) <= 1e-3
    np.testing.assert_allclose(per_sample.cpu().numpy(), ref_per, atol=1e-3)
    assert abs(float(tr._loss[0]) / N - ref_avg) <= 1e-3
    errs = {n: rel_err(g.cpu().numpy(), ref_g[n]) for n, g in tr.grads().items()}
    errs['word_vecs'] = rel_err(dword.cpu().numpy(), ref_gwv)
    print('flags', flags, 'worst relative gradient errors:',
          sorted(errs.items(), key=lambda kv: -kv[1])[:6])
    bad = {k: v for k, v in errs.items() if not v <= tol}
    assert not bad, bad


def test_shapes_backward_matches_autograd():
    N, H, Wd, D, T, Cc = 6, 3, 3, 64, 8, 2
    feat, word_vecs, W, asm, ex, tr = make('shapes', N, H, Wd, D, T, Cc,
                                           flags=_lib.FLAG_PROJ_FP32_SIMT, seed=5)
    layouts = [l for l, _ in synth.SHAPES_LAYOUTS] * 2
    tokens = synth.tokens_from_layouts(asm, layouts, T)
    labels = np.arange(N) % Cc
    scores, valid, per_sample, dword = tr.forward_backward(
        torch.from_numpy(feat).cuda(), torch.from_numpy(word_vecs).cuda(), tokens, labels)
    exprs, pv = asm.assemble(tokens)
    m = ot.TorchOracleModules(feat, word_vecs, Cc, W, family='shapes')
    _, _, _, ref_g, ref_gwv = ot.loss_and_grads(m, exprs, pv, labels)
    errs = {n: rel_err(g.cpu().numpy(), ref_g[n]) for n, g in tr.grads().items()}
    errs['word_vecs'] = rel_err(dword.cpu().numpy(), ref_gwv)
    bad = {k: v for k, v in errs.items() if not v <= 5e-4}
    assert not bad, bad


def test_adam_clip_kernel_matches_tf_formula():
    N, H, Wd, D, T, Cc = 4, 10, 15, 512, 6, 28
    feat, word_vecs, W, asm, ex, tr = make('clevr', N, H, Wd, D, T, Cc, seed=7)
    rng = np.random.RandomState(0)
    w0 = {n: v.cpu().numpy().copy() for n, v in tr.weights().items()}
    state = {}
    ref = dict(w0)
    for step in range(1, 4):
        g = {n: (rng.standard_normal(v.shape) * (3.0 if 'conv_image' in n else 0.01)).astype(np.float32)
             for n, v in w0.items()}      # conv_image grads exceed the clip norm of 10
        for n, (off, cnt, shp) in tr.layout.items():
            tr.g[off:off + cnt] = torch.from_numpy(g[n].reshape(-1)).cuda()
        hp = tr.hyper
        tr.step = step
        _lib.check(tr._lib.n2nmn_adam_step(
            tr.m._h, tr.w.data_ptr(), tr.g.data_ptr(), tr.m1.data_ptr(), tr.m2.data_ptr(), step,
            hp['lr'], hp['beta1'], hp['beta2'], hp['eps'], hp['max_norm'], hp['weight_decay'],
            torch.cuda.current_stream().cuda_stream))
        gd = {n: g[n] + (hp['weight_decay'] * ref[n] if n.endswith('/weights') else 0) for n in g}
        ref = ot.adam_clip_step(ref, gd, state, lr=hp['lr'], max_norm=hp['max_norm'])
    torch.cuda.synchronize()
    for n, v in tr.weights().items():
        np.testing.assert_allclose(v.cpu().numpy(), ref[n], rtol=0, atol=2e-6, err_msg=n)
    # the re-packed weights are the ones the forward now uses
    tokens = synth.expert_mix_tokens(asm, N, T)
    s_new, _ = ex.forward_tokens(tokens)
    exprs, _ = asm.assemble(tokens)
    m = ot.TorchOracleModules(feat, word_vecs, Cc, ref)
    want = ot.forward_scores(m, exprs).detach().numpy()
    assert np.max(np.abs(s_new.cpu().numpy() - want)) <= 1e-3


def test_train_steps_reduce_the_loss():
    N, H, Wd, D, T, Cc = 32, 10, 15, 512, 10, 28
    feat, word_vecs, W, asm, ex, tr = make('clevr', N, H, Wd, D, T, Cc, seed=9)
    tr.hyper['lr'] = 1e-3
    tokens = synth.expert_mix_tokens(asm, N, T)
    labels = np.arange(N) % Cc
    f, w = torch.from_numpy(feat).cuda(), torch.from_numpy(word_vecs).cuda()
    lsp = torch.full((N,), -3.0, device='cuda')
    losses = []
    for _ in range(30):
        out = tr.train_step(f, w, tokens, labels, log_seq_prob=lsp, entropy_reg=-1.0)
        losses.append(out['avg_sample_loss'])
    print('loss curve', [round(l, 3) for l in losses[::5]])
    assert losses[-1] < 0.6 * losses[0]
    assert abs(tr.baseline - 0.5) > 1e-3 and np.isfinite(out['total_loss'])



def test_wgmma_weight_gradient_equals_mma_sync_path_at_batch_64(monkeypatch):
    """The wgmma weight-gradient kernel (wgrad_wgmma.cuh: operands staged transposed into K-major
    tiles) against the mma.sync kernel (xtb_mma_kernel, N2NMN_WGRAD_MMA_SYNC=1) on the BASELINE
    train batch (64 questions, T=10: ~160 B maps, several entries and weight-set changes per CTA).
    Both read TF32 operands (one truncates, one rounds): 2e-3 of the largest gradient entry;
    biases to fp32 accuracy."""
    N, H, Wd, D, T, Cc = 64, 10, 15, 512, 10, 28
    feat, word_vecs, W, asm, ex, tr = make('clevr', N, H, Wd, D, T, Cc, seed=11)
    tokens = synth.expert_mix_tokens(asm, N, T)
    labels = (np.arange(N) * 7) % Cc
    f, w = torch.from_numpy(feat).cuda(), torch.from_numpy(word_vecs).cuda()

    def grads():
        tr.forward_backward(f, w, tokens, labels)
        torch.cuda.synchronize()
        return {n: g.cpu().numpy().copy() for n, g in tr.grads().items()}
    monkeypatch.setenv('N2NMN_WGRAD_MMA_SYNC', '1')
    ref = grads()
    monkeypatch.delenv('N2NMN_WGRAD_MMA_SYNC')
    new = grads()
    checked = 0
    for n in ref:
        if 'conv_image' in n or 'fc_att' in n:
            tol = 2e-3 if n.endswith('weights') else 1e-5
            assert rel_err(new[n], ref[n]) <= tol, (n, rel_err(new[n], ref[n]))
            assert np.abs(ref[n]).max() > 0
            checked += 1
        else:
            # (everything else: same kernels, fp32 atomics in a different order)
            assert rel_err(new[n], ref[n]) <= 1e-4, n
    assert checked >= 8
