#!/usr/bin/env python
"""Golden vectors for the layout generator's LSTM dropout, produced by EXECUTING the reference's
``models_clevr/nmn3_netgen_att.py`` (AttentionSeq2Seq) unmodified with
``encoder_dropout = decoder_dropout = True`` on the numpy TF shim (oracle/tf1_shim.py +
oracle/tf1_shim_rnn.py, plus the DropoutWrapper of tests/seq2seq_dropout_oracle.py). Greedy,
teacher-forced and sampled decoding at 2 and 3 layers. Needs the reference checkout (REF);
writes tests/golden/golden_seq2seq_dropout.npz with the weights, the inputs and, per case, the seed
of its uniform numbers (seq2seq_dropout_oracle.golden_uniforms regenerates them): enc
[T_enc, layers-1, N, L] and dec [T_dec, layers-1, N, L], which the shim's DropoutWrapper consumes in
call order (every encoder step, then every decoder step; layer by layer), and the sampling draws.
Re-run: python tests/golden/make_golden_seq2seq_dropout.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
REF = os.environ.get('N2NMN_REFERENCE', '/root/reference')

CFG = dict(N=6, T_enc=9, T_dec=8, V_txt=30, E_txt=20, E_nmn=12, L=32, seed=23)
GT = [['_Find', '_Count'], ['_Find', '_Transform', '_Filter', '_Describe'],
      ['_Scene', '_Exist'], ['_Find', '_Find', '_And', '_Exist'],
      ['_Find', '_FindSameProperty', '_Count'], ['_Find', '_Find', '_SameProperty']]


def make_weights(cfg, layers, V_nmn, rng):
    L, Et, En = cfg['L'], cfg['E_txt'], cfg['E_nmn']
    P = 'encoder_decoder/'
    w = {}

    def r(*shape, s=0.3):
        return (s * rng.standard_normal(shape)).astype(np.float32)
    w[P + 'encoder/embedding_mat'] = r(cfg['V_txt'], Et, s=0.5)
    for l in range(layers):
        w[P + 'encoder/lstm/multi_rnn_cell/cell_%d/basic_lstm_cell/weights' % l] = r((Et if l == 0 else L) + L, 4 * L)
        w[P + 'encoder/lstm/multi_rnn_cell/cell_%d/basic_lstm_cell/biases' % l] = r(4 * L, s=0.1)
    w[P + 'encoder/encoder_h_transform/weights'] = r(L, L)
    w[P + 'encoder/encoder_h_transform/biases'] = r(L, s=0.1)
    w[P + 'decoder/embedding_mat'] = r(V_nmn, En, s=0.5)
    w[P + 'decoder/go_embedding'] = r(1, En, s=0.5)
    w[P + 'decoder/att_prediction/v'] = r(L, s=0.5)
    w[P + 'decoder/att_prediction/weights'] = r(L, L)
    w[P + 'decoder/att_prediction/biases'] = r(L, s=0.1)
    w[P + 'decoder/token_prediction/weights'] = r(2 * L, V_nmn, s=0.6)
    w[P + 'decoder/token_prediction/biases'] = r(V_nmn, s=0.1)
    for l in range(layers):
        w[P + 'decoder/lstm/multi_rnn_cell/cell_%d/basic_lstm_cell/weights' % l] = r((En if l == 0 else L) + L, 4 * L)
        w[P + 'decoder/lstm/multi_rnn_cell/cell_%d/basic_lstm_cell/biases' % l] = r(4 * L, s=0.1)
    return w


def make_inputs(cfg, rng):
    N, T = cfg['N'], cfg['T_enc']
    lens = rng.randint(2, T + 1, size=N).astype(np.int32)
    lens[0] = T
    seq = rng.randint(1, cfg['V_txt'], size=(T, N)).astype(np.int32)
    for n in range(N):
        seq[lens[n]:, n] = 0
    return seq, lens


def main():
    from oracle import tf1_shim, tf1_shim_rnn
    from n2nmn_b200 import synth
    from tests import seq2seq_dropout_oracle as sdo
    cfg = CFG
    tf1_shim.install({})
    sys.path.insert(0, REF)
    from models_clevr.nmn3_assembler import Assembler
    asm = Assembler(synth.vocab_file('clevr'))
    V_nmn = len(asm.module_names)
    gt = np.stack([asm.module_list2tokens(l, cfg['T_dec']) for l in GT], axis=1).astype(np.int32)
    N, T, Td, L = cfg['N'], cfg['T_enc'], cfg['T_dec'], cfg['L']
    out = {'gt_layout': gt}
    for layers in (2, 3):
        rng = np.random.RandomState(cfg['seed'] + layers)
        weights = make_weights(cfg, layers, V_nmn, rng)
        seq, lens = make_inputs(cfg, rng)
        pre = 'l%d_' % layers
        out[pre + 'input_seq'], out[pre + 'seq_length'] = seq, lens
        for k, v in weights.items():
            out[pre + 'w:' + k] = v
        for ci, case in enumerate(('greedy', 'gt', 'sample')):
            useed = 100 * layers + ci
            enc_u, dec_u, samp_u = sdo.golden_uniforms(useed, T, Td, layers, N, L)
            tf = sdo.install_shim_dropout(tf1_shim_rnn.install_rnn(tf1_shim.install(weights)))
            for m in [k for k in sys.modules if k.startswith('models_clevr') or k.startswith('util')]:
                sys.modules.pop(m)
            from models_clevr.nmn3_netgen_att import AttentionSeq2Seq
            assert tf.contrib.rnn.DropoutWrapper is sdo.DropoutWrapper
            sdo.set_dropout_uniforms(list(enc_u.reshape(-1, N, L)) + list(dec_u.reshape(-1, N, L)))
            kw = {}
            if case == 'gt':
                kw = dict(use_gt_layout=np.array(True), gt_layout_batch=gt)
            if case == 'sample':
                tf1_shim_rnn.set_sampling_uniforms(samp_u)
            m = AttentionSeq2Seq(seq, lens, T_decoder=Td, num_vocab_txt=cfg['V_txt'],
                                 embed_dim_txt=cfg['E_txt'], num_vocab_nmn=V_nmn,
                                 embed_dim_nmn=cfg['E_nmn'], lstm_dim=L, num_layers=layers,
                                 assembler=asm, encoder_dropout=True, decoder_dropout=True,
                                 decoder_sampling=(case == 'sample'), **kw)
            assert sdo.pending_dropout_uniforms() == 0, 'every uniform array consumed'
            p = pre + case + '_'
            out[p + 'uniform_seed'] = np.int32(useed)
            out[p + 'predicted_tokens'] = np.asarray(m.predicted_tokens, np.int32)
            out[p + 'token_probs'] = np.asarray(m.token_probs, np.float32)
            out[p + 'neg_entropy'] = np.asarray(m.neg_entropy, np.float32)
            out[p + 'word_vecs'] = np.asarray(m.word_vecs, np.float32)
            out[p + 'atts'] = np.asarray(m.atts, np.float32)
            out[p + 'encoder_outputs'] = np.asarray(m.encoder_outputs, np.float32)
            for l in range(layers):
                out[p + 'encoder_c%d' % l] = np.asarray(m.encoder_states[l][0], np.float32)
                out[p + 'encoder_h%d' % l] = np.asarray(m.encoder_states[l][1], np.float32)
            print(layers, 'layers', case, 'tokens\n', out[p + 'predicted_tokens'].T)
    tf1_shim.uninstall()
    out['cfg'] = np.array([cfg[k] for k in ('N', 'T_enc', 'T_dec', 'V_txt', 'E_txt', 'E_nmn', 'L',
                                             'seed')], np.int32)
    np.savez_compressed(os.path.join(HERE, 'golden_seq2seq_dropout.npz'), **out)


if __name__ == '__main__':
    main()
