"""GPU: launch accounting of the C ABI and context setup that cannot leak.

For fixed seeded workloads, how many kernels each entry point launches (n2nmn_launch_count) and
which profile regions it records (n2nmn_set_profiling / n2nmn_get_launch_times) are pinned: the
benchmark's kernel pass keys on those region names, and the counts show a launch that went missing
or was added. A failed n2nmn_create or n2nmn_seq2seq_create must free everything it allocated
before it failed."""
import ctypes as C

import numpy as np
import pytest
import torch

from n2nmn_b200 import _lib, synth, weights as wts
from n2nmn_b200.assembler import Assembler
from n2nmn_b200.executor import LayoutExecutor
from n2nmn_b200.trainer import ModuleNetTrainer

pytestmark = pytest.mark.gpu

CLEVR = dict(family='clevr', N=16, H=10, W=15, D=512, T=12, C=28)
VQA = dict(family='vqa', N=16, H=7, W=7, D=256, T=8, C=100)


def make(family, N, H, W, D, T, C, seed=0, **ctx):
    feat, wv = synth.make_inputs(N, H, W, D, T, seed=seed)
    weights = wts.init_weights(family, H, W, D, C, seed=seed, bias_std=0.1)
    asm = Assembler(synth.vocab_file(family))
    ex = LayoutExecutor(family, torch.from_numpy(feat).cuda(), torch.from_numpy(wv).cuda(), C, asm,
                        weights=weights, **ctx)
    if family == 'vqa':
        real = [l for l, _ in synth.VQA_LAYOUTS]
        tokens = synth.tokens_from_layouts(asm, [real[i % len(real)] for i in range(N)], T)
    else:
        tokens = synth.expert_mix_tokens(asm, N, T)
    return ex, np.ascontiguousarray(tokens, np.int32), feat, wv


def accounting(ex, fn):
    """(kernel launches, profile region names) of one call of fn."""
    torch.cuda.synchronize()
    ex.set_profiling(True)
    n0 = ex.launch_count()
    fn()
    torch.cuda.synchronize()
    n = ex.launch_count() - n0
    names = [name for name, _ in ex.launch_times()]
    ex.set_profiling(False)
    return n, names


def clevr_forward_group():
    ex, tok, feat, wv = make(**CLEVR, max_group=2)
    f = [torch.from_numpy(feat).cuda(), torch.from_numpy(feat[::-1].copy()).cuda()]
    w = [torch.from_numpy(wv).cuda(), torch.from_numpy(wv[:, ::-1].copy()).cuda()]
    return accounting(ex, lambda: ex.forward_group(f, w, [tok, tok[:, ::-1].copy()]))


def vqa_forward():
    ex, tok, _, _ = make(**VQA)
    return accounting(ex, lambda: ex.forward_tokens(tok))


def wave_forward():
    ex, tok, _, _ = make(**CLEVR, flags=_lib.FLAG_WAVE_EXECUTOR)
    return accounting(ex, lambda: ex.forward_tokens(tok))


def module_call():
    ex, _, _, _ = make(**CLEVR)
    att = torch.rand((8, CLEVR['H'], CLEVR['W'], 1), device='cuda')
    t, b = np.arange(8) % CLEVR['T'], np.arange(8) % CLEVR['N']
    return accounting(ex, lambda: ex.modules.TransformModule(att, t, b))


def trainer(cfg):
    ex, tok, feat, wv = make(**cfg)
    tr = ModuleNetTrainer(ex, weight_decay=0.0)
    labels = (np.arange(cfg['N']) * 7 + 3) % cfg['C']
    return ex, tr, (torch.from_numpy(feat).cuda(), torch.from_numpy(wv).cuda(), tok, labels)


def clevr_forward_backward():
    ex, tr, args = trainer(CLEVR)
    return accounting(ex, lambda: tr.forward_backward(*args))


def vqa_forward_backward():
    ex, tr, args = trainer(VQA)
    return accounting(ex, lambda: tr.forward_backward(*args))


def adam_step():
    """n2nmn_train_finish after a backward pass: scalars, clip + Adam and the re-pack."""
    ex, tr, args = trainer(VQA)
    tr.forward_backward(*args)
    return accounting(ex, lambda: tr.train_step(*args))


WORKLOADS = [clevr_forward_group, vqa_forward, wave_forward, module_call, clevr_forward_backward,
             vqa_forward_backward, adam_step]

# Recorded at the parent of the launch-helper refactor; adam_step counted 22 there, one less,
# because the re-pack counted the pitched copy and the TF32 split of W_out as one launch.
TEXT = ['text_proj_kernel', 'quad_kernel']
VQA_BWD = ['text_proj_kernel', 'proj_wgmma_kernel', 'tree_kernel', 'loss_kernel',
           'tail_prep_kernel', 'tail_dehat_kernel', 'tail_wgrad_kernel', 'tree_bwd_kernel',
           'text_grad_kernels', 'feat_grad_kernel', 'bias_grad_kernel']
PINS = {
    'clevr_forward_group': (6, TEXT + ['proj_wgmma_kernel', 'tree_kernel', 'pool_kernel',
                                       'head_kernel']),
    'vqa_forward': (6, ['text_proj_kernel', 'proj_wgmma_kernel', 'tree_kernel', 'pool_kernel',
                        'head_kernel', 'head_tail_gemm_kernel']),
    'wave_forward': (9, TEXT + ['proj_wgmma_kernel'] + ['wave_kernel'] * 6),
    'module_call': (3, TEXT + ['wave_kernel']),
    'clevr_forward_backward': (15, TEXT + ['proj_wgmma_kernel', 'tree_kernel', 'loss_kernel',
                                           'tree_bwd_kernel', 'text_grad_kernels',
                                           'feat_grad_kernel', 'bias_grad_kernel']),
    'vqa_forward_backward': (17, VQA_BWD),
    'adam_step': (23, VQA_BWD + ['clip_adam_kernels', 'repack_kernels']),
}


@pytest.mark.parametrize('workload', WORKLOADS, ids=[w.__name__ for w in WORKLOADS])
def test_launch_accounting(workload):
    assert workload() == PINS[workload.__name__]


def test_failed_create_frees_its_allocations():
    """text_dim = 302 is refused only after the weights, workspaces and table slots exist
    (about 130 MB at the CLEVR benchmark's sizes with two batches per launch)."""
    lib = _lib.lib()
    cfg = _lib.Config(abi_version=_lib.ABI_VERSION, family=_lib.FAMILY_ID['clevr'], H=10, W=15,
                      D=512, text_dim=302, map_dim=250, kernel_size=5, num_choices=28,
                      max_batch=64, max_T=20, device=torch.cuda.current_device(), flags=0,
                      max_group=2)
    torch.cuda.synchronize()
    free0, _ = torch.cuda.mem_get_info()
    for _ in range(10):
        h = C.c_void_p()
        assert lib.n2nmn_create(C.byref(cfg), C.byref(h)) == -1   # N2NMN_ERR_ARG
        assert b'text_dim' in lib.n2nmn_last_error()
        assert not h.value
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info()
    assert free0 - free1 < 256 << 20, (free0 - free1) / 2**20


def test_failed_seq2seq_create_frees_its_allocations():
    """A 64-token layout vocabulary at lstm_dim 512 needs about 284 KB of shared memory in the
    decoder step kernel: refused, with nothing left allocated (a context of this size holds about
    240 MB, most of it the 17,742-row input table of the question vocabulary)."""
    lib = _lib.lib()
    cfg = _lib.Seq2SeqConfig(abi_version=_lib.ABI_VERSION, num_vocab_txt=17742, embed_dim_txt=300,
                             num_vocab_nmn=64, embed_dim_nmn=300, lstm_dim=512, num_layers=2,
                             T_encoder=45, T_decoder=10, max_batch=64,
                             device=torch.cuda.current_device(), flags=0)
    torch.cuda.synchronize()
    free0, _ = torch.cuda.mem_get_info()
    for _ in range(5):
        h = C.c_void_p()
        assert lib.n2nmn_seq2seq_create(C.byref(cfg), C.byref(h)) == -1   # N2NMN_ERR_ARG
        assert b'decoder step kernel' in lib.n2nmn_last_error()
        assert not h.value
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info()
    assert free0 - free1 < 64 << 20, (free0 - free1) / 2**20
