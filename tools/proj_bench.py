#!/usr/bin/env python
"""Kernel-only timing of the conv_image contraction as the benchmark's timed region runs it: one
context evaluating groups of `max_group` (16) resident batches of the CLEVR expert mix at the
headline shape (64 x 10x15x512, T=20) per set of launches (n2nmn_forward_group), per-launch CUDA
events (library profiling mode). Prints the median us per launch of every kernel, the card and its
power limit.

    python tools/proj_bench.py [--groups 40] [--proj-ctas 0]"""
import argparse, json, os, subprocess, sys
import numpy as np
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from n2nmn_b200 import synth, weights as wts
from n2nmn_b200.assembler import Assembler
from n2nmn_b200.executor import ExecutorPool

ap = argparse.ArgumentParser()
ap.add_argument('--groups', type=int, default=40, help='timed launch sets')
ap.add_argument('--proj-ctas', type=int, default=0, help='n2nmn_set_proj_ctas cap (0 = all SMs)')
ap.add_argument('--resident', type=int, default=10, help='resident batches the groups walk')
args = ap.parse_args()

B, H, W, D, T, C = 64, 10, 15, 512, 20, 28
asm = Assembler(synth.vocab_file('clevr'))
weights = wts.init_weights('clevr', H, W, D, C, seed=0, bias_std=0.1)
feats, wvs, toks = [], [], []
for i in range(args.resident):
    f, w = synth.make_inputs(B, H, W, D, T, seed=1234 + i)
    feats.append(torch.from_numpy(f).cuda())
    wvs.append(torch.from_numpy(w).cuda())
    t = synth.expert_mix_tokens(asm, B, T)    # the benchmark's mix, question order per batch
    toks.append(np.ascontiguousarray(t[:, np.random.RandomState(100 + i).permutation(B)]))
pool = ExecutorPool('clevr', feats[0], wvs[0], C, asm, weights=weights, max_batch=B, max_T=T,
                    proj_ctas=args.proj_ctas)
ex, G = pool.executors[0], pool.max_group
outs = [torch.empty((B, C), dtype=torch.float32, device='cuda') for _ in range(G)]


def run(i):
    idx = [(i * G + g) % args.resident for g in range(G)]
    ex.forward_group([feats[j] for j in idx], [wvs[j] for j in idx], [toks[j] for j in idx],
                     outs=outs)


for i in range(5):
    run(i)
torch.cuda.synchronize()
ex.set_profiling(True)
acc = {}
for i in range(args.groups):
    run(i)
    for name, us in ex.launch_times():
        acc.setdefault(name, []).append(us)
ex.set_profiling(False)
try:
    smi = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
except Exception as e:   # noqa: BLE001
    smi = 'unknown (%s)' % e
med = {k: round(float(np.median(v)), 1) for k, v in acc.items()}
print(json.dumps({'card': torch.cuda.get_device_name(),
                  'power_limit_and_max_sm_clock': smi, 'batches_per_launch': G,
                  'proj_ctas': args.proj_ctas, 'groups': args.groups,
                  'proj_wgmma_kernel_us': med.get('proj_wgmma_kernel'), 'median_us': med}))
