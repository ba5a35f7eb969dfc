"""Device time of the layout generator's training step at CLEVR training sizes (N=64, T_enc=45,
T_dec=10, lstm 512, 2 layers; `--vqa`: the VQA scripts' T_enc=26, T_dec=13, lstm 1000 over 17,742
words) with CUDA events: the recording forward, the backward pass and the clip + Adam step, each
timed on its own over R repetitions. `--dropout` turns on encoder and decoder dropout (uniforms
drawn on the device per forward, as in training). Prints milliseconds and launches per step, with
the card's name and power limit read in the same run."""
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, '.')
from n2nmn_b200 import synth  # noqa: E402
from n2nmn_b200.assembler import Assembler  # noqa: E402
from n2nmn_b200.seq2seq import AttentionSeq2Seq  # noqa: E402
from n2nmn_b200.trainer import LayoutGeneratorTrainer  # noqa: E402
from n2nmn_b200.weights import init_seq2seq_weights  # noqa: E402

N, T_enc, T_dec, L, layers, V_txt, E = 64, 45, 10, 512, 2, 90, 300
if '--vqa' in sys.argv:
    T_enc, T_dec, L, V_txt = 26, 13, 1000, 17742
drop = '--dropout' in sys.argv
R = 30
card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                      capture_output=True, text=True).stdout.strip().splitlines()[0]
asm = Assembler(synth.vocab_file('vqa' if '--vqa' in sys.argv else 'clevr'))
rng = np.random.RandomState(0)
w = init_seq2seq_weights(V_txt, E, asm.num_vocab_nmn, E, L, layers)
s = AttentionSeq2Seq(None, None, T_dec, V_txt, E, asm.num_vocab_nmn, E, L, layers, asm,
                     T_encoder=T_enc, max_batch=N, weights=w, device='cuda:0',
                     encoder_dropout=drop, decoder_dropout=drop,
                     precision='tf32' if '--tf32' in sys.argv else 'fp32')
tr = LayoutGeneratorTrainer(s, lr=1e-4)
seq = torch.from_numpy(rng.randint(0, V_txt, size=(T_enc, N)).astype(np.int32)).cuda()
lens = torch.from_numpy(rng.randint(5, T_enc + 1, size=N).astype(np.int32)).cuda()
gt = torch.from_numpy(synth.histogram_tokens(asm, synth.VQA_LAYOUTS, N, T_dec, seed=3) if '--vqa' in sys.argv
                      else synth.expert_mix_tokens(asm, N, T_dec)).cuda()
dlp = torch.full((N,), -1.0 / N, device='cuda')
dne = torch.full((N,), 0.005 / N, device='cuda')
dwv = torch.randn(T_dec, N, E, device='cuda') * 1e-3
gflat = torch.empty(tr.flat_size, device='cuda')


def timed(fn):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    n0 = s.launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(R):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / R, (s.launch_count() - n0) / R


fwd = lambda: s.forward(seq, lens, True, gt, record=True)  # noqa: E731
fwd_ms, fwd_n = timed(fwd)
fwd_plain_ms, fwd_plain_n = timed(lambda: s.forward(seq, lens, True, gt))
fwd()
bwd_ms, bwd_n = timed(lambda: s.backward(dlp, dne, dwv, out=gflat))
gen = s
adam = lambda: gen._L.n2nmn_seq2seq_adam_step(  # noqa: E731
    gen._h, tr.w.data_ptr(), gflat.data_ptr(), tr.m1.data_ptr(), tr.m2.data_ptr(), 1, 1e-4, 0.9,
    0.999, 1e-8, 10.0, 5e-6, gen._stream())
adam_ms, adam_n = timed(adam)
print('card: %s' % card)
print('seq2seq training step N=%d T_enc=%d T_dec=%d L=%d layers=%d, dropout %s:'
      % (N, T_enc, T_dec, L, layers, 'on' if drop else 'off'))
print('  forward, recording off: %.3f ms, %d launches' % (fwd_plain_ms, fwd_plain_n))
print('  forward, recording on : %.3f ms, %d launches' % (fwd_ms, fwd_n))
print('  backward              : %.3f ms, %d launches' % (bwd_ms, bwd_n))
print('  clip + Adam           : %.3f ms, %d launches' % (adam_ms, adam_n))
