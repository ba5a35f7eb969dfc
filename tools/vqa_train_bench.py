"""VQA train-step benchmark (exp_vqa/train_vqa_rl_gt_layout.py shapes): B=64 questions,
14x14x2048 res5c grid (+2 coordinate channels), T=13, 3001 answers, map_dim 1024, layouts drawn
from the real gt-layout histogram (synth.VQA_LAYOUTS), a question-prior logit input.

Prints one JSON line: the card and its power limit (read in the same run), the median step time
of the wgmma weight-gradient path and of the mma.sync path (N2NMN_WGRAD_MMA_SYNC=1), timed in
alternating windows, the per-kernel device times of the library's profiling mode, and the
weight-gradient kernel's achieved TFLOP/s from the FLOPs computed from the shapes
(2 * H*W * Dk * map_dim per B map; a Find, Describe = 1 B map, a Transform = 2).

    python tools/vqa_train_bench.py [--steps 10] [--windows 5] [--out result.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from n2nmn_b200 import synth, weights as wts  # noqa: E402
from n2nmn_b200.assembler import Assembler  # noqa: E402
from n2nmn_b200.executor import LayoutExecutor  # noqa: E402
from n2nmn_b200.trainer import ModuleNetTrainer  # noqa: E402

B, H, W, D, T, C, M = 64, 14, 14, 2048, 13, 3001, 1024
B_MAPS = {'_Find': 1, '_Transform': 2, '_Describe': 1}


def card():
    out = {'name': torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit,clocks.max.sm',
                            '--format=csv,noheader,nounits'], capture_output=True, text=True,
                           timeout=30)
        pl, clk = [x.strip() for x in r.stdout.strip().split(',')[:2]]
        out.update({'power_limit_w': float(pl), 'max_sm_clock_mhz': float(clk)})
    except Exception as e:   # the number still stands, with the card name only
        out['power_limit_w'] = 'not read (%s)' % type(e).__name__
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10, help='train steps per timed window')
    ap.add_argument('--windows', type=int, default=5, help='timed windows per path')
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--out', default=None, help='also write the JSON result to this file')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('vqa_train_bench: no CUDA device')
    asm = Assembler(synth.vocab_file('vqa'))
    feat, wv = synth.make_inputs(B, H, W, D, T, seed=1)
    weights = wts.init_weights('vqa', H, W, D, C, seed=0, bias_std=0.1)
    f, w = torch.from_numpy(feat).cuda(), torch.from_numpy(wv).cuda()
    ex = LayoutExecutor('vqa', f, w, C, asm, weights=weights, max_batch=B, max_T=T)
    tr = ModuleNetTrainer(ex, weight_decay=0.0)
    rng = np.random.RandomState(3)
    pick = rng.choice(len(synth.VQA_LAYOUTS), size=B,
                      p=np.array([c for _, c in synth.VQA_LAYOUTS], float) /
                      sum(c for _, c in synth.VQA_LAYOUTS))
    layouts = [synth.VQA_LAYOUTS[i][0] for i in pick]
    tok = synth.tokens_from_layouts(asm, layouts, T)
    lab = rng.randint(0, C, size=B)
    prior = torch.from_numpy(0.1 * rng.standard_normal((B, C)).astype(np.float32)).cuda()
    lsp = torch.full((B,), -2.0, device='cuda')
    b_maps = sum(B_MAPS.get(m, 0) for l in layouts for m in l)
    wgrad_flops = 2.0 * H * W * (D + 2) * M * b_maps

    def step():
        return tr.train_step(f, w, tok, lab, log_seq_prob=lsp, score_prior=prior, sync=False)

    def set_path(mma_sync):
        if mma_sync:
            os.environ['N2NMN_WGRAD_MMA_SYNC'] = '1'
        else:
            os.environ.pop('N2NMN_WGRAD_MMA_SYNC', None)

    for mma_sync in (False, True):   # warm both paths
        set_path(mma_sync)
        for _ in range(a.warmup):
            step()
    torch.cuda.synchronize()
    times = {'wgmma': [], 'mma_sync': []}
    for _ in range(a.windows):        # alternating windows: both paths see the same machine state
        for name in ('wgmma', 'mma_sync'):
            set_path(name == 'mma_sync')
            step()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps):
                step()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / a.steps)
    kernels = {}
    for name in ('wgmma', 'mma_sync'):
        set_path(name == 'mma_sync')
        ex.set_profiling(True)
        acc, n_prof = {}, 5
        for _ in range(n_prof):
            step()
            torch.cuda.synchronize()
            for k, us in ex.launch_times():
                acc[k] = acc.get(k, 0.0) + us / n_prof
        ex.set_profiling(False)
        kernels[name] = acc
    set_path(False)
    res = {
        'workload': 'VQA train step: B=%d, %dx%dx%d(+2), T=%d, C=%d, map_dim=%d, '
                    'VQA_LAYOUTS histogram, question prior' % (B, H, W, D, T, C, M),
        'card': card(),
        'b_maps_per_step': b_maps,
        'wgrad_gflop_per_step': wgrad_flops / 1e9,
        'ms_per_step_median': {k: statistics.median(v) for k, v in times.items()},
        'ms_per_step_windows': times,
        'kernel_us': kernels,
        'wgrad_tflops': {k: (wgrad_flops / (v['feat_grad_kernel'] * 1e-6) / 1e12
                             if v.get('feat_grad_kernel') else None)
                         for k, v in kernels.items()},
        'last_avg_sample_loss': float(step()['avg_sample_loss']),
    }
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, 'w') as fh:
            fh.write(line + '\n')


if __name__ == '__main__':
    main()
