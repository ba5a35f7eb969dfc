#!/usr/bin/env python
"""Per-launch CUDA-event timing of the three forward kernels when ONE set of launches covers G
batches (n2nmn_forward_group), G = 1, 2, 4, 8 (GB_ONLY=8: one G only). Env: GB_BATCH, GB_LAYOUT (expert|find), GB_ONLY, GB_ITERS,
GB_CLUSTER (tree CTAs per question, default 1)."""
import os, sys
import numpy as np
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from n2nmn_b200 import synth, weights as wts
from n2nmn_b200.assembler import Assembler
from n2nmn_b200.executor import LayoutExecutor

B = int(os.environ.get('GB_BATCH', 64))
H, W, D, T, C = 10, 15, 512, 20, 28
asm = Assembler(synth.vocab_file('clevr'))
layout = os.environ.get('GB_LAYOUT', 'expert')
weights = wts.init_weights('clevr', H, W, D, C, seed=0, bias_std=0.1)
P = 16
feats, wvs, toks = [], [], []
for i in range(P):
    f, w = synth.make_inputs(B, H, W, D, T, seed=1234 + i)
    feats.append(torch.from_numpy(f).cuda()); wvs.append(torch.from_numpy(w).cuda())
    if layout == 'find':
        toks.append(synth.tokens_from_layouts(asm, [['_Find', '_Exist']] * B, T))
    else:
        t = synth.expert_mix_tokens(asm, B, T)
        toks.append(np.ascontiguousarray(t[:, np.random.RandomState(i).permutation(B)]))
ex = LayoutExecutor('clevr', feats[0], wvs[0], C, asm, weights=weights, max_batch=B, max_T=T,
                    max_group=int(os.environ.get('GB_MAXG', 16)))
ex.set_tree_cluster(int(os.environ.get('GB_CLUSTER', 1)))
only = os.environ.get('GB_ONLY')
iters = int(os.environ.get('GB_ITERS', 40))
pk_tf32, pk_hbm = 840.25, 6581.6
for G in ([int(only)] if only else [1, 2, 4, 8, 16]):
    def run(i):
        idx = [(i * G + g) % P for g in range(G)]
        return ex.forward_group([feats[j] for j in idx], [wvs[j] for j in idx], [toks[j] for j in idx])
    for i in range(4):
        run(i)
    torch.cuda.synchronize()
    ex.set_profiling(True)
    acc = {}
    for i in range(iters):
        run(i)
        for name, us in ex.launch_times():
            acc.setdefault(name, []).append(us)
    info = ex.last_step_info()
    ex.set_profiling(False)
    med = {k: float(np.median(v)) for k, v in acc.items()}
    fl, by = info['kernel_flops'][1], info['kernel_bytes'][1]
    pu = med.get('proj_wgmma_kernel', float('nan'))
    print('G=%d B=%d %s | us per launch (median): %s | per batch: %s | proj: %.1f TF/s = %.3f of TF32 '
          'peak, %.0f GB/s = %.3f of HBM peak, tiles %d' % (
              G, B, layout, {k: round(v, 1) for k, v in med.items()},
              {k: round(v / G, 2) for k, v in med.items()}, fl / pu / 1e6, fl / pu / 1e6 / pk_tf32,
              by / pu / 1e3, by / pu / 1e3 / pk_hbm, info['num_proj_tiles']), flush=True)
