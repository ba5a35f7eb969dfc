"""Layout executor: Part 2 ("layout_execution") of the reference's NMN3Model
(models_clevr/nmn3_model.py:49-159, models_shapes/nmn3_model.py:53-101,
models_vqa/nmn3_model.py:60-104) without TF Fold.

Reference call sequence (exp_clevr/eval_clevr.py:125-132)          here
    expr_list, valid = assembler.assemble(tokens)                   same Assembler
    feed = nmn3_model.compiler.build_feed_dict(expr_list)           model.compiler.build_feed_dict
    scores = sess.partial_run(h, nmn3_model.scores, feed)           model.run(feed)  /  model.scores

The fast path skips the Python dictionaries altogether: ``model.forward_tokens(tokens)`` hands
the ``[T, N]`` token matrix to the C++ layout compiler (n2nmn_compile_schedule) and launches the
compiled batch (n2nmn_run_schedule). Rows of invalid layouts are zeros
(models_clevr/nmn3_model.py:144-155).
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from . import config as cfgmod
from .assembler import INVALID_EXPR, Assembler
from .modules import MODULES_BY_FAMILY


class CompiledBatch:
    """A compiled layout batch (owns an n2nmn_sched). Plays the role of Fold's feed dict."""

    def __init__(self, lib, handle, validity=None):
        self._lib = lib
        self._h = handle
        self.validity = validity
        info = _lib.SchedInfo()
        _lib.check(lib.n2nmn_sched_get_info(handle, C.byref(info)))
        self.info = {f[0]: getattr(info, f[0]) for f in info._fields_
                     if not f[0].startswith('kernel_')}
        self.info['kernel_bytes'] = list(info.kernel_bytes)
        self.info['kernel_flops'] = list(info.kernel_flops)

    def nodes(self):
        """int32 [num_nodes, 6]: op, time_idx, batch_idx, depth, in0, in1 (arena slot = row)."""
        n = self.info['num_nodes']
        out = np.zeros((max(n, 1), 6), np.int32)
        _lib.check(self._lib.n2nmn_sched_get_nodes(
            self._h, out.ctypes.data_as(C.POINTER(C.c_int32)), max(n, 1)))
        return out[:n]

    def close(self):
        if self._h is not None and self._h.value:
            self._lib.n2nmn_sched_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class _Compiler:
    """Stands in for ``td.Compiler`` (models_clevr/nmn3_model.py:158)."""

    def __init__(self, model):
        self._m = model

    def build_feed_dict(self, expr_list):
        return self._m.compile_exprs(expr_list)


class LayoutExecutor:
    """The module network + executor for one family."""

    def __init__(self, family, image_feat_grid, word_vecs, num_choices, assembler, weights=None,
                 **ctx_kwargs):
        self.family = family
        self.assembler = assembler
        cls = MODULES_BY_FAMILY[family]
        if family == 'vqa':
            self.modules = cls(image_feat_grid, word_vecs, None, num_choices, weights=weights,
                               **ctx_kwargs)
        else:
            self.modules = cls(image_feat_grid, word_vecs, num_choices, weights=weights,
                               **ctx_kwargs)
        self.num_choices = self.modules.num_choices
        self._lib = self.modules._lib
        fam = cfgmod.FAMILIES[family]
        unknown = [n for n in assembler.module_names if n != '<eos>' and n not in fam.token_ops]
        if unknown:   # the reference would raise KeyError when such a token is executed
            raise ValueError('layout vocabulary names %r are not modules of the %r family'
                             % (unknown, family))
        self.vocab_ops = np.array([fam.token_ops.get(n, -1) for n in assembler.module_names],
                                  np.int32)
        self._vocab_ptr = self.vocab_ops.ctypes.data
        self.compiler = _Compiler(self)
        self.scores = None   # last result, like fetching `nmn3_model.scores`
        self._cache = {}

    # -- compile ----------------------------------------------------------------------------
    def compile_tokens(self, layout_tokens, cache=False):
        """[T, N] int tokens -> CompiledBatch (C++ layout compiler; no Python dicts)."""
        tok = np.ascontiguousarray(np.asarray(layout_tokens), dtype=np.int32)
        key = tok.tobytes() if cache else None
        if cache and key in self._cache:
            return self._cache[key]
        T, N = tok.shape
        validity = np.zeros(N, np.uint8)
        h = C.c_void_p()
        _lib.check(self._lib.n2nmn_compile_schedule(
            self.modules._h, tok.ctypes.data_as(C.POINTER(C.c_int32)), T, N,
            self.vocab_ops.ctypes.data_as(C.POINTER(C.c_int32)), len(self.vocab_ops),
            validity.ctypes.data_as(C.POINTER(C.c_uint8)), C.byref(h)))
        cb = CompiledBatch(self._lib, h, validity.astype(bool))
        if cache:
            self._cache[key] = cb
        return cb

    def compile_exprs(self, expr_list):
        """Assembler expression dicts -> CompiledBatch (compiler.build_feed_dict)."""
        fam = cfgmod.FAMILIES[self.family]
        op, t, b, in0, in1, q_ptr = [], [], [], [], [], [0]

        def walk(e):
            kids = [walk(e[k]) for k in ('input_0', 'input_1') if k in e]
            op.append(fam.token_ops[e['module']])
            t.append(int(e['time_idx']))
            b.append(int(e['batch_idx']))
            in0.append(kids[0] if len(kids) > 0 else -1)
            in1.append(kids[1] if len(kids) > 1 else -1)
            return len(op) - 1

        for e in expr_list:
            if e['module'] != INVALID_EXPR:
                walk(e)
            q_ptr.append(len(op))
        arrs = [np.asarray(a, np.int32) for a in (op, t, b, in0, in1, q_ptr)]
        ptr = [a.ctypes.data_as(C.POINTER(C.c_int32)) for a in arrs]
        h = C.c_void_p()
        _lib.check(self._lib.n2nmn_compile_nodes(self.modules._h, ptr[0], ptr[1], ptr[2], ptr[3],
                                                 ptr[4], len(op), ptr[5], len(expr_list),
                                                 C.byref(h)))
        validity = np.array([e['module'] != INVALID_EXPR for e in expr_list], bool)
        return CompiledBatch(self._lib, h, validity)

    # -- run ----------------------------------------------------------------------------------
    def run(self, compiled, return_att=False, out=None):
        """Evaluate a compiled batch against the bound inputs -> scores [N, C] (CUDA tensor).
        With return_att=True also returns the attention arena [num_nodes, H, W]."""
        m = self.modules
        nq = compiled.info['num_questions']
        scores = out if out is not None else torch.empty((nq, self.num_choices),
                                                         dtype=torch.float32, device=m.device)
        arena = None
        if return_att:
            arena = torch.zeros((max(compiled.info['num_nodes'], 1), m.H, m.W),
                                dtype=torch.float32, device=m.device)
        _lib.check(self._lib.n2nmn_run_schedule(
            m._h, compiled._h, C.c_void_p(scores.data_ptr()),
            C.c_void_p(arena.data_ptr()) if arena is not None else None, m._stream()))
        self.scores = scores
        return (scores, arena) if return_att else scores

    def forward_tokens(self, layout_tokens, cache=False):
        """tokens [T,N] -> (scores [N,C] CUDA tensor, validity bool[N])."""
        cb = self.compile_tokens(layout_tokens, cache=cache)
        return self.run(cb), cb.validity

    def forward_device(self, image_feat_grid, word_vecs, layout_tokens, out=None, stream=None):
        """One eval step with device-resident inputs: bind + C++ layout compile + launches in a
        single C call (n2nmn_forward_tokens). Inputs must be contiguous float32 CUDA tensors
        ([N,H,W,D], [T,N,Dt]); tokens a C-contiguous int32 [T,N] numpy array. Returns
        (scores [N,C] CUDA tensor, validity bool[N]). Asynchronous on `stream` (a
        torch.cuda.Stream; default: the current stream)."""
        m = self.modules
        tok = layout_tokens
        if tok.dtype != np.int32 or not tok.flags['C_CONTIGUOUS']:
            tok = np.ascontiguousarray(tok, dtype=np.int32)
        T, N = tok.shape
        if out is None:
            out = torch.empty((N, self.num_choices), dtype=torch.float32, device=m.device)
        validity = np.empty(N, np.uint8)
        assert image_feat_grid.is_cuda and image_feat_grid.is_contiguous() and \
            image_feat_grid.dtype == torch.float32 and word_vecs.is_cuda and \
            word_vecs.is_contiguous() and word_vecs.dtype == torch.float32
        m.image_feat_grid, m.word_vecs, m.N, m.T = image_feat_grid, word_vecs, N, T
        _lib.check(self._lib.n2nmn_forward_tokens(
            m._h, image_feat_grid.data_ptr(), word_vecs.data_ptr(), tok.ctypes.data, T, N,
            self._vocab_ptr, len(self.vocab_ops), out.data_ptr(), validity.ctypes.data,
            (stream or torch.cuda.current_stream(m.device)).cuda_stream))
        self.scores = out
        return out, validity.view(bool)

    def forward_group(self, feats, word_vecs, tokens, outs=None, stream=None):
        """Several INDEPENDENT batches of identical shape in one set of launches
        (n2nmn_forward_group; at most the context's max_group). feats / word_vecs: lists of
        contiguous float32 CUDA tensors [N,H,W,D] / [T,N,Dt]; tokens: list of int32 [T,N] arrays.
        Returns (list of scores [N,C], list of validity bool[N]); results equal those of separate
        forward_device calls."""
        m = self.modules
        n = len(feats)
        toks = [t if (t.dtype == np.int32 and t.flags['C_CONTIGUOUS'])
                else np.ascontiguousarray(t, dtype=np.int32) for t in tokens]
        T, N = toks[0].shape
        assert all(t.shape == (T, N) for t in toks) and len(word_vecs) == n and len(toks) == n
        if outs is None:
            outs = [torch.empty((N, self.num_choices), dtype=torch.float32, device=m.device)
                    for _ in range(n)]
        for f, w in zip(feats, word_vecs):
            assert f.is_cuda and f.is_contiguous() and f.dtype == torch.float32 and \
                w.is_cuda and w.is_contiguous() and w.dtype == torch.float32
        valid = np.empty((n, N), np.uint8)
        arr = lambda ptrs: (C.c_void_p * n)(*ptrs)
        _lib.check(self._lib.n2nmn_forward_group(
            m._h, n, arr([f.data_ptr() for f in feats]), arr([w.data_ptr() for w in word_vecs]),
            arr([t.ctypes.data for t in toks]), T, N, self._vocab_ptr, len(self.vocab_ops),
            arr([o.data_ptr() for o in outs]), arr([valid[i].ctypes.data for i in range(n)]),
            (stream or torch.cuda.current_stream(m.device)).cuda_stream))
        m.image_feat_grid, m.word_vecs, m.N, m.T = feats[0], word_vecs[0], N, T
        self._group_keep = (list(feats), list(word_vecs), toks, outs)
        self.scores = outs[0]
        return outs, [valid[i].view(bool) for i in range(n)]

    def last_step_info(self):
        info = _lib.SchedInfo()
        _lib.check(self._lib.n2nmn_last_step_info(self.modules._h, C.byref(info)))
        d = {f[0]: getattr(info, f[0]) for f in info._fields_ if not f[0].startswith('kernel_')}
        d['kernel_bytes'] = list(info.kernel_bytes)
        d['kernel_flops'] = list(info.kernel_flops)
        return d

    def forward(self, expr_list):
        return self.run(self.compile_exprs(expr_list))

    def bind(self, image_feat_grid, word_vecs):
        self.modules.bind(image_feat_grid, word_vecs)

    # -- e2e with host buffers ------------------------------------------------------------------
    def forward_host(self, feat_host, word_vecs_host, layout_tokens, scores_host=None):
        """Host numpy/pinned-tensor inputs -> host scores; H2D/D2H inside (n2nmn_forward_host)."""
        m = self.modules
        tok = np.ascontiguousarray(np.asarray(layout_tokens), dtype=np.int32)
        T, N = tok.shape
        f = feat_host if isinstance(feat_host, torch.Tensor) else torch.from_numpy(
            np.ascontiguousarray(feat_host, np.float32))
        w = word_vecs_host if isinstance(word_vecs_host, torch.Tensor) else torch.from_numpy(
            np.ascontiguousarray(word_vecs_host, np.float32))
        assert f.dtype == torch.float32 and w.dtype == torch.float32
        assert f.is_contiguous() and w.is_contiguous() and not f.is_cuda and not w.is_cuda
        if scores_host is None:
            scores_host = torch.empty((N, self.num_choices), dtype=torch.float32).pin_memory()
        validity = np.zeros(N, np.uint8)
        _lib.check(self._lib.n2nmn_forward_host(
            m._h, C.c_void_p(f.data_ptr()), C.c_void_p(w.data_ptr()),
            tok.ctypes.data_as(C.POINTER(C.c_int32)), T, N,
            self.vocab_ops.ctypes.data_as(C.POINTER(C.c_int32)), len(self.vocab_ops),
            C.c_void_p(scores_host.data_ptr()), validity.ctypes.data_as(C.POINTER(C.c_uint8)),
            m._stream()))
        return scores_host, validity.astype(bool)

    def set_tree_cluster(self, ctas_per_question):
        """CTAs per question in the executor kernel (0 = automatic). Tuning only."""
        _lib.check(self._lib.n2nmn_set_tree_cluster(self.modules._h, int(ctas_per_question)))

    def set_proj_ctas(self, max_ctas):
        """Cap of the contraction kernel's persistent grid (0 = one CTA per SM). Tuning only."""
        _lib.check(self._lib.n2nmn_set_proj_ctas(self.modules._h, int(max_ctas)))

    def set_text_ctas_per_group(self, n):
        """Retired knob of the round-1 text kernel: accepted and ignored (see the header)."""
        _lib.check(self._lib.n2nmn_set_text_ctas_per_group(self.modules._h, int(n)))

    # -- profiling ------------------------------------------------------------------------------
    def set_profiling(self, on):
        _lib.check(self._lib.n2nmn_set_profiling(self.modules._h, int(bool(on))))

    def launch_times(self):
        names = (C.c_char_p * 64)()
        us = (C.c_float * 64)()
        n = _lib.check(self._lib.n2nmn_get_launch_times(self.modules._h, names, us, 64))
        return [(names[i].decode(), float(us[i])) for i in range(n)]

    def launch_count(self):
        return int(self._lib.n2nmn_launch_count(self.modules._h))


class ExecutorPool:
    """K LayoutExecutors (one context + one CUDA stream + one native worker thread each) with
    dynamic batching of the queued work.

    A batch of 64 questions is a short chain of small kernels (~4 us of tensor work) that cannot
    fill the SMs on its own; successive batches are independent (eval). submit() only queues the
    batch; each context's C++ worker thread (csrc/pool.cpp) takes up to `max_group` queued batches
    at a time and runs them with ONE set of launches (n2nmn_forward_group), so the contraction
    kernel's persistent CTAs walk several tiles each and the kernels of different contexts overlap on
    the GPU. Each executor owns its workspaces, so there is no sharing hazard; weights are
    replicated (a few MB).

        pool.begin(); pool.submit(...) x n; pool.end()   # scores / validity valid after end()
    """

    def __init__(self, family, image_feat_grid, word_vecs, num_choices, assembler, weights=None,
                 num_streams=4, tree_cluster=None, proj_ctas=None, max_group=None, **ctx_kwargs):
        nb = int(ctx_kwargs.get('max_batch') or image_feat_grid.shape[0])
        if max_group is None:   # ~1024 questions per launch set: the contraction kernel's CTAs
            # then walk 10+ tiles each (0.49 of the TF32 peak against 0.42 at 512; 6.2 M vs 5.3 M q/s)
            max_group = 1 if num_streams == 1 else max(1, min(16, 1024 // max(nb, 1)))
        self.max_group = int(max_group)
        first = LayoutExecutor(family, image_feat_grid, word_vecs, num_choices, assembler,
                               weights=weights, max_group=self.max_group, **ctx_kwargs)
        w = first.modules.get_weights()
        self.executors = [first] + [
            LayoutExecutor(family, image_feat_grid, word_vecs, num_choices, assembler, weights=w,
                           max_group=self.max_group, **ctx_kwargs) for _ in range(num_streams - 1)]
        dev = first.modules.device
        # Several batches in flight: throughput, not the latency of one batch, is what counts. The
        # node kernels of a batch are latency chains, so the GPU does more work per second with
        # one CTA per question and many questions per launch than with a question spread over a
        # cluster (measured: DESIGN §9). The contraction kernel keeps its whole persistent grid:
        # a group gives every CTA several tiles.
        if tree_cluster is None:
            tree_cluster = 0 if num_streams == 1 else 1
        if proj_ctas is None:
            proj_ctas = 0
        self.tree_cluster, self.proj_ctas = tree_cluster, proj_ctas
        # retired knob of the round-1 text kernel (n2nmn_set_text_ctas_per_group is a no-op): the
        # value the pool used to pass is kept readable for callers of the ABI-2 Python API
        self.text_ctas_per_group = 0 if num_streams == 1 else 1
        for ex in self.executors:
            ex.set_tree_cluster(tree_cluster)
            ex.set_proj_ctas(proj_ctas)
        self.streams = [torch.cuda.Stream(device=dev) for _ in self.executors]
        self._i = 0
        self.device = dev
        self._lib = first._lib
        K = len(self.executors)
        ctxs = (C.c_void_p * K)(*[ex.modules._h for ex in self.executors])
        sts = (C.c_void_p * K)(*[st.cuda_stream for st in self.streams])
        h = C.c_void_p()
        rc = self._lib.n2nmn_pool_create(ctxs, sts, K, first._vocab_ptr, len(first.vocab_ops),
                                         C.byref(h))
        if rc < 0:
            raise _lib.N2NMNError('n2nmn_pool_create failed: %s' %
                                  (self._lib.n2nmn_pool_last_error() or b'').decode())
        self._h = h
        self._keep = []          # arrays the workers still write to (validity) or read from

    def group_stats(self):
        """(n2nmn_forward_group calls, batches) the workers have run so far."""
        g, j = C.c_int64(), C.c_int64()
        self._lib.n2nmn_pool_group_stats(self._h, C.byref(g), C.byref(j))
        return int(g.value), int(j.value)

    def __len__(self):
        return len(self.executors)

    def __del__(self):
        h = getattr(self, '_h', None)
        if h:
            self._lib.n2nmn_pool_destroy(h)
            self._h = None

    def begin(self):
        """Make the pool's streams wait for work already queued on the current stream."""
        cur = torch.cuda.current_stream(self.device)
        for st in self.streams:
            st.wait_stream(cur)

    def _submit(self, k, feat_ptr, wv_ptr, tok, scores_ptr, host_io):
        T, N = tok.shape
        validity = np.empty(N, np.uint8)
        rc = self._lib.n2nmn_pool_submit(self._h, k, feat_ptr, wv_ptr, tok.ctypes.data, T, N,
                                         scores_ptr, validity.ctypes.data, host_io)
        if rc < 0:
            raise _lib.N2NMNError('n2nmn_pool_submit failed: %s' %
                                  (self._lib.n2nmn_pool_last_error() or b'').decode())
        self._keep.append(validity)
        return validity.view(bool)

    @staticmethod
    def _tokens(layout_tokens):
        tok = layout_tokens
        if tok.dtype != np.int32 or not tok.flags['C_CONTIGUOUS']:
            tok = np.ascontiguousarray(tok, dtype=np.int32)
        return tok

    def submit(self, image_feat_grid, word_vecs, layout_tokens, out=None):
        """Queue one batch (device-resident inputs) on the next executor/stream; returns
        (scores, validity, stream). `scores` is ordered on `stream`; `validity` is filled by the
        worker thread and valid after end()."""
        k = (self._i // self.max_group) % len(self.executors)   # runs of max_group per context
        self._i += 1
        tok = self._tokens(layout_tokens)
        if out is None:   # allocate on the slot's stream so the caching allocator orders reuse
            with torch.cuda.stream(self.streams[k]):
                out = torch.empty((tok.shape[1], self.executors[k].num_choices),
                                  dtype=torch.float32, device=self.device)
        assert image_feat_grid.is_cuda and image_feat_grid.is_contiguous() and \
            image_feat_grid.dtype == torch.float32 and word_vecs.is_cuda and \
            word_vecs.is_contiguous() and word_vecs.dtype == torch.float32
        valid = self._submit(k, image_feat_grid.data_ptr(), word_vecs.data_ptr(), tok,
                             out.data_ptr(), 0)
        # the worker enqueues later, on the slot's stream: keep the buffers alive until end(),
        # which orders the caller's stream after the pool's streams (so a free after end() is
        # stream-ordered after the last use)
        self._keep.append((image_feat_grid, word_vecs, out))
        return out, valid, self.streams[k]

    def submit_host(self, feat_host, word_vecs_host, layout_tokens, scores_host):
        """End-to-end step from pinned HOST tensors: H2D of the batch's features and word
        vectors, the forward pass, and D2H of the scores, all enqueued by the slot's worker on
        the slot's stream (copy engines overlap the other slots' kernels). `scores_host` and the
        returned validity are valid after end() + a stream/device synchronise. `feat_host` may be
        a float16 tensor (a feature store kept in half precision: half the PCIe bytes; widened
        on the device, n2nmn_forward_group_host_f16_async)."""
        k = (self._i // self.max_group) % len(self.executors)
        self._i += 1
        tok = self._tokens(layout_tokens)
        for t in (feat_host, word_vecs_host, scores_host):
            assert (not t.is_cuda) and t.is_contiguous()
        assert word_vecs_host.dtype == torch.float32 and scores_host.dtype == torch.float32
        assert feat_host.dtype in (torch.float32, torch.float16)
        valid = self._submit(k, feat_host.data_ptr(), word_vecs_host.data_ptr(), tok,
                             scores_host.data_ptr(), 2 if feat_host.dtype == torch.float16 else 1)
        self._keep.append((feat_host, word_vecs_host, scores_host))
        return scores_host, valid, self.streams[k]

    def forward_many(self, feats, word_vecs, tokens, outs):
        """Queue a list of independent batches (item i -> context i % K); returns the validity
        arrays. Call begin() before and end() after, like submit()."""
        return [self.submit(f, w, t, out=o)[1] for f, w, t, o in zip(feats, word_vecs, tokens, outs)]

    def make_block(self, feats, word_vecs, tokens, outs, host_io=False):
        """Pre-marshal a list of same-shape batches for submit_block(): pointer arrays for ONE
        FFI call (n2nmn_pool_submit_many). The tensors/arrays must stay alive and unchanged for as
        long as the block is used; the block keeps references. `outs` device tensors (host_io:
        pinned host tensors; then feats / word_vecs are pinned host tensors too, and the feature
        grids may be float16 — all of them or none)."""
        toks = [self._tokens(t) for t in tokens]
        n = len(toks)
        T, N = toks[0].shape
        assert all(t.shape == (T, N) for t in toks)
        f16 = bool(host_io) and feats[0].dtype == torch.float16
        for f, w, o in zip(feats, word_vecs, outs):
            for t in (f, w, o):
                assert t.is_contiguous() and t.is_cuda != bool(host_io)
            assert w.dtype == torch.float32 and o.dtype == torch.float32
            assert f.dtype == (torch.float16 if f16 else torch.float32)
        valid = np.empty((n, N), np.uint8)
        arr = lambda ptrs: (C.c_void_p * n)(*ptrs)
        return {'n': n, 'T': T, 'N': N, 'host_io': 2 if f16 else int(bool(host_io)), 'valid': valid,
                'feat': arr([f.data_ptr() for f in feats]),
                'wv': arr([w.data_ptr() for w in word_vecs]),
                'tok': arr([t.ctypes.data for t in toks]),
                'out': arr([o.data_ptr() for o in outs]),
                'val': arr([valid[i].ctypes.data for i in range(n)]),
                'keep': (list(feats), list(word_vecs), toks, list(outs))}

    def submit_block(self, block):
        """Queue every batch of a make_block() result (one step each). Between begin() / end()."""
        rc = self._lib.n2nmn_pool_submit_many(self._h, block['n'], block['feat'], block['wv'],
                                              block['tok'], block['T'], block['N'], block['out'],
                                              block['val'], block['host_io'])
        if rc < 0:
            raise _lib.N2NMNError('n2nmn_pool_submit_many failed: %s' %
                                  (self._lib.n2nmn_pool_last_error() or b'').decode())
        return block['valid']

    def end(self):
        """Wait until the workers have enqueued everything submitted so far, then make the current
        stream wait for the pool's streams."""
        rc = self._lib.n2nmn_pool_wait(self._h)
        self._keep.clear()
        if rc < 0:
            raise _lib.N2NMNError('n2nmn_b200 error %d: %s' % (
                rc, (self._lib.n2nmn_pool_last_error() or b'').decode()))
        cur = torch.cuda.current_stream(self.device)
        for st in self.streams:
            cur.wait_stream(st)

    def launch_count(self):
        return sum(e.launch_count() for e in self.executors)
