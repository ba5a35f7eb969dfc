"""Host-side mirror of the reference's layout generator ``AttentionSeq2Seq``
(models_clevr/nmn3_netgen_att.py:46-322; models_vqa/ and models_shapes/ carry the same file) over
the C ABI (`n2nmn_seq2seq_*`, include/n2nmn_b200.h). Forward pass: greedy decoding under the
Assembler's validity masks, `decoder_sampling=True` (one draw per step from the masked token
distribution, nmn3_netgen_att.py:234-256; the uniform numbers come from `torch.rand` on the device
or from the caller, `forward(..., sample_uniforms=)`) or teacher forcing (`use_gt_layout`).

Dropout: `encoder_dropout` / `decoder_dropout` are the training scripts' DropoutWrapper with
output_keep_prob 0.5 on every LSTM layer but the top one (nmn3_netgen_att.py:17-44). Only what a
layer hands to the layer above is dropped: an element is kept iff its uniform number u satisfies
floor(0.5 + u) = 1 in fp32 (u >= 0.5) and a kept element doubles, as tf.nn.dropout computes it. The
states, encoder outputs, attention and token scores are undropped, and with num_layers == 1 there
is nothing to drop. The flags are attributes read at every `forward`, so one instance trains with
dropout and evaluates without it (the reference builds two graphs for that).

The reference builds a TF graph whose placeholders are fed per batch; here the constructor takes
the shapes (and optionally the first batch) and ``forward`` / ``__call__`` runs a batch. The
attribute names after a forward are the reference's: ``predicted_tokens`` [T_decoder, N] int32,
``token_probs`` [T_decoder, N], ``neg_entropy`` [N], ``word_vecs`` [T_decoder, N, embed_dim_txt],
``atts`` [T_decoder, T_encoder, N, 1]; ``log_seq_prob`` as nmn3_model.py:45 computes it.
PyTorch only owns the device buffers; there is no CPU path.

Training: ``forward(..., record=True)`` keeps what ``backward(d_log_seq_prob, d_neg_entropy,
d_word_vecs)`` needs; the gradient of every variable lands in one flat buffer (``grads()`` gives
``{TF name: view}``), the layout the optimiser step of ``trainer.LayoutGeneratorTrainer`` reads.

VQA's question-prior net (models_vqa/question_prior_net.py) reads the encoder's final state:
``forward(..., with_encoder_states=True)`` sets ``encoder_states``, a tuple of per-layer ``(c, h)``
[N, lstm_dim] device views (TF's LSTMStateTuple order), and ``backward(..., d_encoder_states=)``
takes the gradient of that state back.

`precision='fp32'` (default): every matrix product with fp32 parity (error-compensated TF32 on the
tensor cores); `'tf32'`: one TF32 pass (13 % faster at batch 64, where the step is latency bound),
probabilities within ~1e-3, a token may
differ when two scores are that close.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import check


class AttentionSeq2Seq:
    def __init__(self, input_seq_batch, seq_length_batch, T_decoder, num_vocab_txt, embed_dim_txt,
                 num_vocab_nmn, embed_dim_nmn, lstm_dim, num_layers, assembler,
                 encoder_dropout=False, decoder_dropout=False, decoder_sampling=False,
                 use_gt_layout=None, gt_layout_batch=None, scope='encoder_decoder', reuse=None,
                 T_encoder=None, max_batch=None, device=None, weights=None, precision='fp32'):
        self.encoder_dropout, self.decoder_dropout = bool(encoder_dropout), bool(decoder_dropout)
        self.decoder_sampling = bool(decoder_sampling)
        self.T_decoder = int(T_decoder)
        self.encoder_num_vocab, self.encoder_embed_dim = int(num_vocab_txt), int(embed_dim_txt)
        self.decoder_num_vocab, self.decoder_embed_dim = int(num_vocab_nmn), int(embed_dim_nmn)
        self.lstm_dim, self.num_layers = int(lstm_dim), int(num_layers)
        self.EOS_token = assembler.EOS_idx
        self.scope = scope
        if input_seq_batch is not None:
            T_encoder = T_encoder or int(input_seq_batch.shape[0])
            max_batch = max_batch or int(input_seq_batch.shape[1])
            if device is None and isinstance(input_seq_batch, torch.Tensor) and input_seq_batch.is_cuda:
                device = input_seq_batch.device
        if T_encoder is None or max_batch is None:
            raise ValueError('give input_seq_batch or T_encoder and max_batch')
        self.device = torch.device(device if device is not None else 'cuda:0')
        if self.device.type != 'cuda':
            raise _lib.N2NMNError('n2nmn_b200 runs on a CUDA (sm_90) device only')
        self.T_encoder, self.max_batch = int(T_encoder), int(max_batch)
        self._L = _lib.lib()
        cfg = _lib.Seq2SeqConfig(_lib.ABI_VERSION, self.encoder_num_vocab, self.encoder_embed_dim,
                                 self.decoder_num_vocab, self.decoder_embed_dim, self.lstm_dim,
                                 self.num_layers, self.T_encoder, self.T_decoder, self.max_batch,
                                 self.device.index or 0, {'fp32': 0, 'tf32': 1}[precision])
        h = C.c_void_p()
        check(self._L.n2nmn_seq2seq_create(C.byref(cfg), C.byref(h)))
        self._h = h
        P = np.ascontiguousarray(assembler.P, np.int32)
        W = np.ascontiguousarray(assembler.W, np.int32)
        b = np.ascontiguousarray(assembler.b, np.int32)
        V = self.decoder_num_vocab
        if P.shape != (V, 3) or W.shape != (3, V, 4) or b.shape != (V, 4):
            raise ValueError('assembler tables do not match num_vocab_nmn')
        i32 = C.POINTER(C.c_int32)
        with torch.cuda.device(self.device):
            check(self._L.n2nmn_seq2seq_set_assembler(self._h, P.ctypes.data_as(i32),
                                                      W.ctypes.data_as(i32), b.ctypes.data_as(i32),
                                                      self._stream()))
        self._keep = None
        if weights is not None:
            self.set_weights(weights)
        self.use_gt_layout, self.gt_layout_batch = use_gt_layout, gt_layout_batch
        if input_seq_batch is not None and weights is not None:
            self.forward(input_seq_batch, seq_length_batch, use_gt_layout, gt_layout_batch)

    def __del__(self):
        h, self._h = getattr(self, '_h', None), None
        if h:
            self._L.n2nmn_seq2seq_destroy(h)

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def variables(self):
        """[(name relative to `<scope>/`, shape)] in creation order."""
        out = []
        for i in range(self._L.n2nmn_seq2seq_num_variables(self._h)):
            name, shape, nd = C.c_char_p(), (C.c_int64 * 4)(), C.c_int()
            check(self._L.n2nmn_seq2seq_variable_info(self._h, i, C.byref(name), shape, C.byref(nd)))
            out.append((name.value.decode(), tuple(shape[:nd.value])))
        return out

    def set_weights(self, weights):
        """weights: {TF variable name: array}; names may carry any prefix ending in
        ``<scope>/`` (e.g. ``neural_module_network/layout_generation/encoder_decoder/…``)."""
        tag = self.scope + '/'
        rel = {}
        for k, v in weights.items():
            k = k[2:] if k.startswith('w:') else k
            k = k.split(':')[0]
            if tag in k:
                rel[k[k.index(tag) + len(tag):]] = v
            else:
                rel[k] = v
        with torch.cuda.device(self.device):
            for name, shape in self.variables():
                if name not in rel:
                    raise KeyError('missing seq2seq weight %s' % name)
                t = torch.as_tensor(np.asarray(rel[name], np.float32) if not isinstance(
                    rel[name], torch.Tensor) else rel[name]).to(self.device, torch.float32).contiguous()
                if tuple(t.shape) != shape:
                    raise ValueError('shape of %s is %s, expected %s' % (name, tuple(t.shape), shape))
                shp = (C.c_int64 * len(shape))(*shape)
                check(self._L.n2nmn_seq2seq_set_weight(self._h, name.encode(), C.c_void_p(t.data_ptr()),
                                                       shp, len(shape), self._stream()))
                torch.cuda.current_stream(self.device).synchronize()   # t may be a temporary
        self._recorded_N = None

    def forward(self, input_seq_batch, seq_length_batch, use_gt_layout=None, gt_layout_batch=None,
                sample_uniforms=None, record=False, with_encoder_states=False, dropout_uniforms=None):
        """input_seq_batch [T_enc, N] int, seq_length_batch [N] int (device or host);
        gt_layout_batch [T_decoder, N] with use_gt_layout truthy = teacher forcing;
        sample_uniforms [T_decoder, N] in [0, 1): the numbers the sampled decoding consumes
        (decoder_sampling=True; default `torch.rand` on the device, i.e. torch's generator);
        record=True keeps what `backward` needs (same outputs, bit for bit);
        with_encoder_states=True also sets `self.encoder_states` = ((c, h) of layer 0, ...), each
        [N, lstm_dim]: the encoder's final state (nmn3_netgen_att.py:95-99), which VQA's
        question-prior net reads. Otherwise `self.encoder_states` is None.
        dropout_uniforms: None or an (enc, dec) pair, each None or the uniform numbers in [0, 1) of
        one side whose dropout flag is on, enc [T_enc, num_layers-1, N, lstm_dim] and dec
        [T_decoder, num_layers-1, N, lstm_dim], indexed by (step, layer below the top). A side whose
        flag is on and has no numbers given draws them with `torch.rand` on the device; numbers
        given for a side whose flag is off raise ValueError (they would silently do nothing), as do
        numbers of the wrong shape. Draw order
        of one forward: the sampling uniforms (decoder_sampling), then the encoder's dropout
        uniforms, then the decoder's, so a forward without dropout uses torch's generator as
        before; with num_layers == 1 nothing is dropped and nothing is drawn."""
        dev = self.device

        def i32(x):
            t = x if isinstance(x, torch.Tensor) else torch.as_tensor(np.asarray(x))
            return t.to(dev, torch.int32, non_blocking=True).contiguous()
        seq, lens = i32(input_seq_batch), i32(seq_length_batch)
        T, N = seq.shape
        if lens.shape != (N,):
            raise ValueError('seq_length_batch must have one entry per question')
        if T > self.T_encoder or N > self.max_batch:
            raise _lib.N2NMNError('batch exceeds the capacity the seq2seq was created for')
        gt = None
        if use_gt_layout:
            gt = i32(gt_layout_batch)
            if gt.shape != (self.T_decoder, N):
                raise ValueError('gt_layout_batch must be [T_decoder, N]')
        u = None
        if self.decoder_sampling or sample_uniforms is not None:
            if sample_uniforms is None:
                u = torch.rand((self.T_decoder, N), dtype=torch.float32, device=dev)
            else:
                u = (sample_uniforms if isinstance(sample_uniforms, torch.Tensor) else
                     torch.as_tensor(np.asarray(sample_uniforms, np.float32)))
                u = u.to(dev, torch.float32).contiguous()
                if u.shape != (self.T_decoder, N):
                    raise ValueError('sample_uniforms must be [T_decoder, N]')
        du = self._dropout_uniforms(dropout_uniforms, T, N)
        tokens = torch.empty((self.T_decoder, N), dtype=torch.int32, device=dev)
        probs = torch.empty((self.T_decoder, N), dtype=torch.float32, device=dev)
        ent = torch.empty((N,), dtype=torch.float32, device=dev)
        wv = torch.empty((self.T_decoder, N, self.encoder_embed_dim), dtype=torch.float32, device=dev)
        atts = torch.empty((self.T_decoder, T, N, 1), dtype=torch.float32, device=dev)
        states = None
        if with_encoder_states:
            states = torch.empty((self.num_layers, 2, N, self.lstm_dim), dtype=torch.float32,
                                 device=dev)
        with torch.cuda.device(dev):
            check(self._L.n2nmn_seq2seq_set_record(self._h, 1 if record else 0))
            check(self._L.n2nmn_seq2seq_set_sampling(
                self._h, C.c_void_p(u.data_ptr()) if u is not None else None))
            check(self._L.n2nmn_seq2seq_set_dropout(
                self._h, *[C.c_void_p(d.data_ptr()) if d is not None else None for d in du]))
            check(self._L.n2nmn_seq2seq_forward_ex(
                self._h, C.c_void_p(seq.data_ptr()), C.c_void_p(lens.data_ptr()), T, N,
                C.c_void_p(gt.data_ptr()) if gt is not None else None,
                C.c_void_p(tokens.data_ptr()), C.c_void_p(probs.data_ptr()),
                C.c_void_p(ent.data_ptr()), C.c_void_p(wv.data_ptr()), C.c_void_p(atts.data_ptr()),
                self._stream(), C.c_void_p(states.data_ptr()) if states is not None else None))
        self._keep = (seq, lens, gt, u, du)   # alive until the stream has consumed them
        self._recorded_N = N if record else None
        self.predicted_tokens, self.token_probs, self.neg_entropy = tokens, probs, ent
        self.word_vecs, self.atts = wv, atts
        self.encoder_states = None if states is None else tuple(
            (states[l, 0], states[l, 1]) for l in range(self.num_layers))
        self.log_seq_prob = torch.log(probs).sum(0)          # nmn3_model.py:45
        return tokens, probs, ent, wv, atts

    __call__ = forward

    def _dropout_uniforms(self, given, T, N):
        """(enc, dec) device tensors for n2nmn_seq2seq_set_dropout; None = no dropout there."""
        if given is None:
            given = (None, None)
        if not isinstance(given, (tuple, list)) or len(given) != 2:
            raise ValueError('dropout_uniforms must be an (enc, dec) pair')
        out = []
        for side, flag, steps, g in (('encoder', self.encoder_dropout, T, given[0]),
                                     ('decoder', self.decoder_dropout, self.T_decoder, given[1])):
            shape = (steps, self.num_layers - 1, N, self.lstm_dim)
            if g is not None and not flag:
                raise ValueError('dropout uniforms given for the %s, whose dropout is off' % side)
            if not flag or (g is None and self.num_layers == 1):   # one layer: nothing to drop
                out.append(None)
                continue
            if g is None:
                d = torch.rand(shape, dtype=torch.float32, device=self.device)
            else:
                d = g if isinstance(g, torch.Tensor) else torch.as_tensor(np.asarray(g, np.float32))
                if tuple(d.shape) != shape:
                    raise ValueError('%s dropout uniforms must be %s, got %s' % (side, shape, tuple(d.shape)))
                d = d.to(self.device, torch.float32).contiguous()
            out.append(d if self.num_layers > 1 else None)
        return out

    def launch_count(self):
        return int(self._L.n2nmn_seq2seq_launch_count(self._h))

    # ---- training -------------------------------------------------------------------------------
    def flat_layout(self):
        """(flat size, [(name, shape, offset, count)]) of the flat weight / gradient buffers."""
        out = []
        for i, (name, shape) in enumerate(self.variables()):
            off, cnt = C.c_int64(), C.c_int64()
            check(self._L.n2nmn_seq2seq_flat_offset(self._h, i, C.byref(off), C.byref(cnt)))
            out.append((name, shape, off.value, cnt.value))
        return int(self._L.n2nmn_seq2seq_flat_size(self._h)), out

    def _views(self, flat):
        return {name: flat[off:off + cnt].view(shape) for name, shape, off, cnt in self.flat_layout()[1]}

    def get_flat_weights(self, out=None):
        size = self.flat_layout()[0]
        if out is None:
            out = torch.zeros(size, dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            check(self._L.n2nmn_seq2seq_get_flat_weights(self._h, C.c_void_p(out.data_ptr()),
                                                         self._stream()))
        return out

    def load_flat_weights(self, wflat):
        with torch.cuda.device(self.device):
            check(self._L.n2nmn_seq2seq_load_flat_weights(self._h, C.c_void_p(wflat.data_ptr()),
                                                          self._stream()))

    def get_weights(self):
        """{name relative to `<scope>/`: tensor}: the current variables, as `set_weights` takes them."""
        return {k: v.clone() for k, v in self._views(self.get_flat_weights()).items()}

    def backward(self, d_log_seq_prob=None, d_neg_entropy=None, d_word_vecs=None, out=None,
                 d_encoder_states=None):
        """Gradient of Σ d_log_seq_prob·log_seq_prob + Σ d_neg_entropy·neg_entropy +
        Σ d_word_vecs·word_vecs + Σ d_encoder_states·encoder_states with respect to every variable,
        after a `forward(..., record=True)` of this batch (TF 1.0's gradients of
        nmn3_netgen_att.py; no gradient through the validity masks or the chosen tokens).
        Upstreams: [N], [N], [T_decoder, N, embed_dim_txt] device tensors or None (= zero);
        d_encoder_states in the shape of `encoder_states` (a tuple of per-layer (dc, dh) [N, L]) or
        one [num_layers, 2, N, L] tensor, or None. Returns the flat gradient buffer (`out`, or a
        new one); `grads()` gives it per variable."""
        N = getattr(self, '_recorded_N', None)
        if N is None:
            raise _lib.N2NMNError('backward needs a forward(..., record=True) of this batch')
        dev = self.device

        def f32(x, shape, what):
            if x is None:
                return None
            t = (x if isinstance(x, torch.Tensor) else torch.as_tensor(np.asarray(x, np.float32)))
            t = t.to(dev, torch.float32).contiguous()
            if tuple(t.shape) != shape:
                raise ValueError('%s must be %s (the recorded batch), got %s' % (what, shape, tuple(t.shape)))
            return t
        dlp = f32(d_log_seq_prob, (N,), 'd_log_seq_prob')
        dne = f32(d_neg_entropy, (N,), 'd_neg_entropy')
        dwv = f32(d_word_vecs, (self.T_decoder, N, self.encoder_embed_dim), 'd_word_vecs')
        if isinstance(d_encoder_states, (tuple, list)):
            if len(d_encoder_states) != self.num_layers:
                raise ValueError('d_encoder_states must hold one (dc, dh) pair per layer')
            d_encoder_states = torch.stack([torch.stack([f32(c, (N, self.lstm_dim), 'dc'),
                                                         f32(h, (N, self.lstm_dim), 'dh')])
                                            for c, h in d_encoder_states])
        dst = f32(d_encoder_states, (self.num_layers, 2, N, self.lstm_dim), 'd_encoder_states')
        if out is None:
            out = torch.empty(self.flat_layout()[0], dtype=torch.float32, device=dev)
        ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None  # noqa: E731
        with torch.cuda.device(dev):
            check(self._L.n2nmn_seq2seq_backward_ex(self._h, ptr(dlp), ptr(dne), ptr(dwv), ptr(out),
                                                    self._stream(), ptr(dst)))
        self._bwd_keep = (dlp, dne, dwv, dst)
        self._grad = out
        return out

    def grads(self):
        """{name relative to `<scope>/`: view of the last backward's gradient}."""
        return self._views(self._grad)
