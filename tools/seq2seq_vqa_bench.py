"""Device time of the layout generator at the VQA scripts' size (exp_vqa/train_vqa*.py: N=64,
T_enc=26, T_dec=13, a 17,742-word question vocabulary, embed 300, lstm 1000, 2 layers) with CUDA
events, each stage timed on its own over R repetitions after warm-up:
  * prepare(): the packed weights re-derived after a weight change (after every Adam step), mostly
    the [V_txt][4L] layer-0 table = embedding_mat · W_x, timed as (weight load + forward) minus the
    weight load and the forward;
  * the forward (greedy), without and with the encoder states; the recording forward (teacher
    forced, with the encoder states); the backward with all four upstreams; clip + Adam.
Prints milliseconds and launches per call, with the card's name and power limit read in the same
run."""
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

N, T_enc, T_dec, L, layers, V_txt, E = 64, 26, 13, 1000, 2, 17742, 300
R = 20
card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                      capture_output=True, text=True).stdout.strip().splitlines()[0]
asm = Assembler(synth.vocab_file('vqa'))
rng = np.random.RandomState(0)
w = init_seq2seq_weights(V_txt, E, asm.num_vocab_nmn, E, L, layers)
s = AttentionSeq2Seq(None, None, T_dec, V_txt, E, asm.num_vocab_nmn, E, L, layers, asm,
                     T_encoder=T_enc, max_batch=N, weights=w, device='cuda:0',
                     precision='tf32' if '--tf32' in sys.argv else 'fp32')
tr = LayoutGeneratorTrainer(s, lr=1e-4)
seq = torch.from_numpy(rng.randint(0, V_txt, size=(T_enc, N)).astype(np.int32)).cuda()
lens = torch.from_numpy(rng.randint(5, T_enc + 1, size=N).astype(np.int32)).cuda()
gt = torch.from_numpy(synth.histogram_tokens(asm, synth.VQA_LAYOUTS, N, T_dec)).cuda()
dlp = torch.full((N,), -1.0 / N, device='cuda')
dne = torch.full((N,), 0.005 / N, device='cuda')
dwv = torch.randn(T_dec, N, E, device='cuda') * 1e-3
dst = torch.randn(layers, 2, N, L, device='cuda') * 1e-3
gflat = torch.empty(tr.flat_size, device='cuda')
wflat = s.get_flat_weights()


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


fwd_ms, fwd_n = timed(lambda: s.forward(seq, lens))
fwd_st_ms, fwd_st_n = timed(lambda: s.forward(seq, lens, with_encoder_states=True))
load_ms, _ = timed(lambda: s.load_flat_weights(wflat))
s.forward(seq, lens)
reload_fwd_ms, reload_fwd_n = timed(lambda: (s.load_flat_weights(wflat), s.forward(seq, lens)))
rec = lambda: s.forward(seq, lens, True, gt, record=True, with_encoder_states=True)  # noqa: E731
rec_ms, rec_n = timed(rec)
rec()
bwd_ms, bwd_n = timed(lambda: s.backward(dlp, dne, dwv, out=gflat, d_encoder_states=dst))
adam = lambda: s._L.n2nmn_seq2seq_adam_step(  # noqa: E731
    s._h, tr.w.data_ptr(), gflat.data_ptr(), tr.m1.data_ptr(), tr.m2.data_ptr(), 1, 1e-4, 0.9,
    0.999, 1e-8, 10.0, 5e-6, s._stream())
adam_ms, adam_n = timed(adam)
print('card: %s' % card)
print('seq2seq at the VQA size N=%d T_enc=%d T_dec=%d V_txt=%d E=%d L=%d layers=%d:'
      % (N, T_enc, T_dec, V_txt, E, L, layers))
print('  prepare (table rebuild)        : %.3f ms, %d launches'
      % (reload_fwd_ms - load_ms - fwd_ms, reload_fwd_n - fwd_n))
print('  forward                        : %.3f ms, %d launches' % (fwd_ms, fwd_n))
print('  forward + encoder states       : %.3f ms, %d launches' % (fwd_st_ms, fwd_st_n))
print('  recording forward (+ states)   : %.3f ms, %d launches' % (rec_ms, rec_n))
print('  backward (four upstreams)      : %.3f ms, %d launches' % (bwd_ms, bwd_n))
print('  clip + Adam                    : %.3f ms, %d launches' % (adam_ms, adam_n))
