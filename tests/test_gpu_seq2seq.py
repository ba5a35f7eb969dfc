"""GPU parity of the seq2seq layout generator (SURVEY.md §8 f1) through the C ABI:
  * against the goldens produced by executing the reference's nmn3_netgen_att.py on the TF shim
    (tests/golden/golden_seq2seq.npz): greedy decoding under the validity masks and teacher
    forcing;
  * against the numpy oracle at the reference's real CLEVR sizes (exp_clevr/train_clevr_*.py:
    T_encoder 45, T_decoder 20 (here 10..20), embed 300, lstm 512, 2 layers, batch 64), ragged
    lengths including 1 and T_encoder.
Tolerance: tokens bit-exact; probabilities, entropies, attention maps and word vectors 2e-5
absolute (fp32 everywhere; only the summation order differs)."""
import os

import numpy as np
import pytest
import torch

from n2nmn_b200 import synth
from n2nmn_b200.weights import init_seq2seq_weights
from n2nmn_b200.assembler import Assembler
from oracle import seq2seq_oracle as so

pytestmark = pytest.mark.gpu
Z = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'golden_seq2seq.npz'))
ATOL = 2e-5


def golden_weights():
    return {k[2 + len('encoder_decoder/'):]: Z[k] for k in Z.files if k.startswith('w:')}


def make(asm, w, T_enc, N, T_dec, V_txt, E_txt, E_nmn, L, layers, precision='fp32'):
    from n2nmn_b200.seq2seq import AttentionSeq2Seq
    return AttentionSeq2Seq(None, None, T_dec, V_txt, E_txt, asm.num_vocab_nmn, E_nmn, L, layers,
                            asm, T_encoder=T_enc, max_batch=N, weights=w, device='cuda:0',
                            precision=precision)


def check(out, tokens, probs, nent, wv, atts, atol=ATOL):
    torch.cuda.synchronize()
    g = [o.cpu().numpy() for o in out]
    assert np.array_equal(g[0], tokens)
    np.testing.assert_allclose(g[1], probs, atol=atol)
    np.testing.assert_allclose(g[2], nent, atol=10 * atol)
    np.testing.assert_allclose(g[3], wv, atol=atol)
    np.testing.assert_allclose(g[4], atts, atol=atol)


def test_matches_reference_goldens():
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers, seed = [int(v) for v in Z['cfg']]
    asm = Assembler(synth.vocab_file('clevr'))
    s = make(asm, golden_weights(), T_enc, N, T_dec, V_txt, E_txt, E_nmn, L, layers)
    out = s.forward(Z['input_seq'], Z['seq_length'])
    check(out, Z['greedy_predicted_tokens'], Z['greedy_token_probs'], Z['greedy_neg_entropy'],
          Z['greedy_word_vecs'], Z['greedy_atts'])
    lsp = s.log_seq_prob.cpu().numpy()
    np.testing.assert_allclose(lsp, np.log(Z['greedy_token_probs']).sum(0), atol=1e-4)
    out = s.forward(Z['input_seq'], Z['seq_length'], True, Z['gt_layout'])
    check(out, Z['gt_layout'], Z['gt_token_probs'], Z['gt_neg_entropy'], Z['gt_word_vecs'],
          Z['gt_atts'])
    # the first call again: nothing of the forced run may leak into the next batch
    out = s.forward(Z['input_seq'], Z['seq_length'])
    check(out, Z['greedy_predicted_tokens'], Z['greedy_token_probs'], Z['greedy_neg_entropy'],
          Z['greedy_word_vecs'], Z['greedy_atts'])


@pytest.mark.parametrize('N,T_enc,T_dec,L,layers', [(64, 45, 20, 512, 2), (37, 26, 13, 208, 1),
                                                     (1, 5, 10, 64, 3)])
def test_matches_oracle_at_reference_sizes(N, T_enc, T_dec, L, layers):
    rng = np.random.RandomState(1000 + N)
    asm = Assembler(synth.vocab_file('clevr'))
    V_nmn = len(asm.module_names)
    V_txt, E_txt, E_nmn = 90, 300, 300
    w = init_seq2seq_weights(V_txt, E_txt, V_nmn, E_nmn, L, layers, seed=2000 + N)
    seq = rng.randint(0, V_txt, size=(T_enc, N)).astype(np.int32)
    lens = rng.randint(1, T_enc + 1, size=N).astype(np.int32)
    lens[0] = T_enc
    lens[-1] = 1
    s = make(asm, w, T_enc, N, T_dec, V_txt, E_txt, E_nmn, L, layers)
    _, dec = so.run(w, seq, lens, T_dec, layers, asm.P, asm.W, asm.b)
    out = s.forward(seq, lens)
    check(out, *dec)
    assert asm.assemble(out[0].cpu().numpy())[1].all()
    gt = dec[0][:, ::-1].copy()      # some other valid layouts as the forced ones
    _, dec = so.run(w, seq, lens, T_dec, layers, asm.P, asm.W, asm.b, use_gt_layout=True,
                    gt_layout=gt)
    out = s.forward(seq, lens, True, gt)
    check(out, *dec)


def test_sampled_decoding_matches_reference_goldens_and_oracle():
    """decoder_sampling=True (nmn3_netgen_att.py:234-256): with the golden's uniform numbers the
    tokens of the reference file (run on the shim's inverse-CDF tf.multinomial) bit-exactly; at
    the CLEVR sizes against the oracle, with draws whose distance from the nearest CDF boundary
    (> 1e-4, asserted) is far above the fp32 difference between a warp scan and a cumsum."""
    from n2nmn_b200.seq2seq import AttentionSeq2Seq
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers, seed = [int(v) for v in Z['cfg']]
    asm = Assembler(synth.vocab_file('clevr'))
    s = AttentionSeq2Seq(None, None, T_dec, V_txt, E_txt, asm.num_vocab_nmn, E_nmn, L, layers, asm,
                         T_encoder=T_enc, max_batch=N, weights=golden_weights(), device='cuda:0',
                         decoder_sampling=True)
    out = s.forward(Z['input_seq'], Z['seq_length'], sample_uniforms=Z['sample_uniforms'])
    check(out, Z['sample_predicted_tokens'], Z['sample_token_probs'], Z['sample_neg_entropy'],
          Z['sample_word_vecs'], Z['sample_atts'])
    # teacher forcing wins over sampling (:264-266); torch.rand draws give valid layouts
    out = s.forward(Z['input_seq'], Z['seq_length'], True, Z['gt_layout'],
                    sample_uniforms=Z['sample_uniforms'])
    check(out, Z['gt_layout'], Z['gt_token_probs'], Z['gt_neg_entropy'], Z['gt_word_vecs'],
          Z['gt_atts'])
    torch.manual_seed(5)
    drawn = set()
    for _ in range(4):
        tok = s.forward(Z['input_seq'], Z['seq_length'])[0].cpu().numpy()
        assert asm.assemble(tok)[1].all()
        drawn.add(tok.tobytes())
    assert len(drawn) > 1
    # a greedy generator is not disturbed by an earlier sampling one (the pointer is per context)
    g = make(asm, golden_weights(), T_enc, N, T_dec, V_txt, E_txt, E_nmn, L, layers)
    check(g.forward(Z['input_seq'], Z['seq_length']), Z['greedy_predicted_tokens'],
          Z['greedy_token_probs'], Z['greedy_neg_entropy'], Z['greedy_word_vecs'], Z['greedy_atts'])
    for (N, T_enc, T_dec, L, layers, useed) in [(64, 45, 20, 512, 2, 3065), (37, 26, 13, 208, 1, 3037)]:
        rng = np.random.RandomState(1000 + N)
        V_nmn, V_txt, E = len(asm.module_names), 90, 300
        w = init_seq2seq_weights(V_txt, E, V_nmn, E, L, layers, seed=2000 + N)
        seq = rng.randint(0, V_txt, size=(T_enc, N)).astype(np.int32)
        lens = rng.randint(1, T_enc + 1, size=N).astype(np.int32)
        lens[0], lens[-1] = T_enc, 1
        u = np.random.RandomState(useed).random_sample((T_dec, N)).astype(np.float32)
        margins = []
        _, dec = so.run(w, seq, lens, T_dec, layers, asm.P, asm.W, asm.b, sample_uniforms=u,
                        margins=margins)
        assert np.min(margins) > 1e-4
        s = AttentionSeq2Seq(None, None, T_dec, V_txt, E, V_nmn, E, L, layers, asm, T_encoder=T_enc,
                             max_batch=N, weights=w, device='cuda:0', decoder_sampling=True)
        out = s.forward(seq, lens, sample_uniforms=u)
        check(out, *dec)
        assert asm.assemble(out[0].cpu().numpy())[1].all()


def test_single_pass_tf32_option_stays_within_1e_3():
    """precision='tf32' (one TF32 pass per product): teacher-forced probabilities, attention maps
    and word vectors within 2e-3 of the fp32 oracle at the CLEVR sizes; greedy tokens agree on
    >= 97 % of the positions (a flip needs two scores within the TF32 error)."""
    N, T_enc, T_dec, L, layers = 64, 45, 20, 512, 2
    rng = np.random.RandomState(77)
    asm = Assembler(synth.vocab_file('clevr'))
    V_nmn, V_txt, E = asm.num_vocab_nmn, 90, 300
    w = init_seq2seq_weights(V_txt, E, V_nmn, E, L, layers, seed=5)
    seq = rng.randint(0, V_txt, size=(T_enc, N)).astype(np.int32)
    lens = rng.randint(3, T_enc + 1, size=N).astype(np.int32)
    s = make(asm, w, T_enc, N, T_dec, V_txt, E, E, L, layers, precision='tf32')
    _, dec = so.run(w, seq, lens, T_dec, layers, asm.P, asm.W, asm.b)
    out = s.forward(seq, lens)
    torch.cuda.synchronize()
    agree = float((out[0].cpu().numpy() == dec[0]).mean())
    assert agree >= 0.97, agree
    assert asm.assemble(out[0].cpu().numpy())[1].all()
    _, decf = so.run(w, seq, lens, T_dec, layers, asm.P, asm.W, asm.b, use_gt_layout=True,
                     gt_layout=dec[0])
    out = s.forward(seq, lens, True, dec[0])
    check(out, *decf, atol=2e-3)


def test_generators_of_different_sizes_coexist():
    """Kernel attributes belong to the process: creating and running a generator of a smaller
    lstm_dim must not lower the shared memory limit an earlier, larger one launches with (plain
    and recording forwards, backward)."""
    asm = Assembler(synth.vocab_file('clevr'))
    N, T_enc, T_dec, V_txt, E, layers = 8, 6, 5, 30, 32, 2
    rng = np.random.RandomState(4)
    seq = rng.randint(0, V_txt, size=(T_enc, N)).astype(np.int32)
    lens = rng.randint(1, T_enc + 1, size=N).astype(np.int32)
    d_lsp = torch.ones(N, device='cuda')

    def generator(L):
        w = init_seq2seq_weights(V_txt, E, asm.num_vocab_nmn, E, L, layers, seed=L)
        return make(asm, w, T_enc, N, T_dec, V_txt, E, E, L, layers)
    a = generator(1000)
    first = [o.clone() for o in a.forward(seq, lens, record=True)]
    a.backward(d_log_seq_prob=d_lsp)
    b = generator(512)
    b.forward(seq, lens, record=True)
    b.backward(d_log_seq_prob=d_lsp)
    for record in (False, True):
        again = a.forward(seq, lens, record=record)
        torch.cuda.synchronize()
        for x, y in zip(first, again):
            assert torch.equal(x, y)
    a.backward(d_log_seq_prob=d_lsp)
    torch.cuda.synchronize()


def test_errors_are_loud():
    from n2nmn_b200 import _lib
    asm = Assembler(synth.vocab_file('clevr'))
    N, T_enc, T_dec, V_txt, E_txt, E_nmn, L, layers, seed = [int(v) for v in Z['cfg']]
    s = make(asm, None, T_enc, N, T_dec, V_txt, E_txt, E_nmn, L, layers)
    with pytest.raises(_lib.N2NMNError):          # weights not set
        s.forward(Z['input_seq'], Z['seq_length'])
    s.set_weights(golden_weights())
    with pytest.raises(_lib.N2NMNError):          # over capacity
        s.forward(np.zeros((T_enc + 1, N), np.int32), Z['seq_length'])
    with pytest.raises(KeyError):
        s.set_weights({'encoder/embedding_mat': Z['w:encoder_decoder/encoder/embedding_mat']})
