"""Host-side mirror of the reference's ``class Modules`` for the three model families.

Same constructor and method names / argument order / kwargs as
``models_clevr/nmn3_modules.py:11-495``, ``models_shapes/nmn3_modules.py:9-150`` and
``models_vqa/nmn3_modules.py:33-240``; every method is one call into the C ABI
(``n2nmn_module_fwd``), with PyTorch CUDA tensors only as the buffer container.

  reference (TF graph op)                                   here (eager CUDA call)
  ------------------------------------------------------    -------------------------------------
  modules = Modules(image_feat_grid, word_vecs, C)          same (tensors live on the GPU)
  att = modules.FindModule(time_idx, batch_idx)             same; returns [n,H,W,1] float32 CUDA
  s   = modules.DescribeModule(att, time_idx, batch_idx)    same; returns [n,C]

``scope=`` / ``reuse=`` are accepted and ignored (variable scoping is a TF-graph concern);
``map_dim`` / ``kernel_size`` must match the context the object was built with.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from . import config as cfgmod
from .weights import init_weights, variable_shapes


def _as_host_i32(x, n=None):
    if x is None:
        return None
    if isinstance(x, torch.Tensor):
        x = x.detach().cpu().numpy()
    a = np.ascontiguousarray(np.asarray(x).reshape(-1), dtype=np.int32)
    return a


def _i32p(a):
    return a.ctypes.data_as(C.POINTER(C.c_int32)) if a is not None else None


class ModulesBase:
    """Owns one n2nmn_ctx: packed weights, bound inputs, workspaces."""
    family = None

    def __init__(self, image_feat_grid, word_vecs, num_choices, weights=None, device=None,
                 max_batch=None, max_T=None, flags=0, seed=0, max_group=1):
        self._lib = _lib.lib()
        fam = cfgmod.FAMILIES[self.family]
        if not torch.cuda.is_available():
            raise _lib.N2NMNError('n2nmn_b200 needs a CUDA (sm_90a) device; there is no CPU path')
        if device is None:
            device = image_feat_grid.device if isinstance(image_feat_grid, torch.Tensor) and \
                image_feat_grid.is_cuda else torch.device('cuda', torch.cuda.current_device())
        self.device = torch.device(device)
        self.image_feat_grid = self._to_dev(image_feat_grid)
        self.word_vecs = self._to_dev(word_vecs)
        N, H, W, D = self.image_feat_grid.shape
        T, N2, Dt = self.word_vecs.shape
        assert N2 == N, 'word_vecs is [T, N, D_txt] (time-major)'
        self.num_choices = int(num_choices)
        self.H, self.W, self.D, self.N, self.T, self.text_dim = H, W, D, N, T, Dt
        self.map_dim, self.kernel_size = fam.map_dim, fam.kernel_size
        self.att_shape = [None, H, W, 1]
        cfg = _lib.Config(abi_version=_lib.ABI_VERSION, family=_lib.FAMILY_ID[self.family], H=H,
                          W=W, D=D, text_dim=Dt, map_dim=fam.map_dim,
                          kernel_size=fam.kernel_size, num_choices=self.num_choices,
                          max_batch=int(max_batch or N), max_T=int(max_T or T),
                          device=self.device.index or 0, flags=int(flags),
                          max_group=int(max_group))
        self.max_batch, self.max_T = cfg.max_batch, cfg.max_T
        h = C.c_void_p()
        _lib.check(self._lib.n2nmn_create(C.byref(cfg), C.byref(h)))
        self._h = h
        self._weights = {}
        if weights is None:   # the reference's initialisers (xavier / zeros)
            weights = init_weights(self.family, H, W, D, self.num_choices, seed=seed,
                                   text_dim=Dt)
        self.set_weights(weights)
        self.bind(self.image_feat_grid, self.word_vecs)

    # -- plumbing ---------------------------------------------------------------------------
    def _to_dev(self, x):
        if not isinstance(x, torch.Tensor):
            x = torch.from_numpy(np.ascontiguousarray(np.asarray(x, np.float32)))
        return x.to(device=self.device, dtype=torch.float32).contiguous()

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def close(self):
        if getattr(self, '_h', None) is not None and self._h.value:
            self._lib.n2nmn_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def variable_names(self):
        return list(variable_shapes(self.family, self.H, self.W, self.D, self.num_choices,
                                    self.text_dim))

    def set_weights(self, weights):
        """weights: {TF variable name (relative to module_variables/): array or tensor}."""
        for name, val in weights.items():
            t = self._to_dev(val)
            shape = (C.c_int64 * t.dim())(*t.shape)
            _lib.check(self._lib.n2nmn_set_weight(self._h, name.encode(), C.c_void_p(t.data_ptr()),
                                                  shape, t.dim(), self._stream()))
            self._weights[name] = t   # keep the source alive until the async copy has run

    def get_weights(self):
        """Current weights by TF name. After optimiser steps (ModuleNetTrainer) these are views of
        the trainer's flat buffer, i.e. the values the context was last re-packed from."""
        src = getattr(self, '_weights_source', None)
        return dict(src()) if src is not None else dict(self._weights)

    def bind(self, image_feat_grid, word_vecs):
        """Re-point the context at a new batch (the reference re-feeds its placeholders)."""
        self.image_feat_grid = self._to_dev(image_feat_grid)
        self.word_vecs = self._to_dev(word_vecs)
        N, T = self.image_feat_grid.shape[0], self.word_vecs.shape[0]
        _lib.check(self._lib.n2nmn_bind_inputs(self._h, C.c_void_p(self.image_feat_grid.data_ptr()),
                                               C.c_void_p(self.word_vecs.data_ptr()), N, T,
                                               self._stream()))
        self.N, self.T = N, T

    def _check_dims(self, map_dim=None, kernel_size=None):
        if map_dim is not None and map_dim != self.map_dim:
            raise ValueError('map_dim=%r differs from the context (%d)' % (map_dim, self.map_dim))
        if kernel_size is not None and self.family != 'vqa' and kernel_size != self.kernel_size:
            raise ValueError('kernel_size=%r differs from the context (%d)' %
                             (kernel_size, self.kernel_size))

    def _run(self, op, inputs, time_idx, batch_idx, n=None):
        ins = [self._to_dev(a).reshape(-1, self.H, self.W, 1) for a in inputs]
        t = _as_host_i32(time_idx)
        b = _as_host_i32(batch_idx)
        if n is None:
            n = ins[0].shape[0] if ins else len(t)
        for a in ins:
            assert a.shape[0] == n, 'attention inputs and index vectors disagree on n'
        ans = cfgmod.OP_IS_ANS[op]
        out = torch.empty((n, self.num_choices) if ans else (n, self.H, self.W, 1),
                          dtype=torch.float32, device=self.device)
        if n == 0:
            return out
        p = [C.c_void_p(a.data_ptr()) for a in ins] + [None, None]
        _lib.check(self._lib.n2nmn_module_fwd(self._h, op, p[0], p[1], _i32p(t), _i32p(b), n,
                                              C.c_void_p(out.data_ptr()), self._stream()))
        return out

    # -- modules shared by several families ---------------------------------------------------
    def FindModule(self, time_idx, batch_idx, map_dim=None, scope='FindModule', reuse=True):
        self._check_dims(map_dim)
        return self._run(cfgmod.OP_FIND, [], time_idx, batch_idx)

    def AndModule(self, input_0, input_1, time_idx=None, batch_idx=None, scope='AndModule',
                  reuse=True):
        return self._run(cfgmod.OP_AND, [input_0, input_1], None, None)


class ModulesCLEVR(ModulesBase):
    """models_clevr/nmn3_modules.py"""
    family = 'clevr'

    def SceneModule(self, time_idx, batch_idx, pos_val=3, scope='SceneModule', reuse=True):
        n = len(_as_host_i32(time_idx))
        out = torch.empty((n, self.H, self.W, 1), dtype=torch.float32, device=self.device)
        if n:
            _lib.check(self._lib.n2nmn_scene_fwd(self._h, n, C.c_float(float(pos_val)),
                                                 C.c_void_p(out.data_ptr()), self._stream()))
        return out

    def FilterModule(self, input_0, time_idx, batch_idx, map_dim=250, scope='FilterModule',
                     reuse=True):
        self._check_dims(map_dim)
        return self._run(cfgmod.OP_FILTER, [input_0], time_idx, batch_idx)

    def FindSamePropertyModule(self, input_0, time_idx, batch_idx, map_dim=250,
                               scope='FindSamePropertyModule', reuse=True):
        self._check_dims(map_dim)
        return self._run(cfgmod.OP_FIND_SAME_PROPERTY, [input_0], time_idx, batch_idx)

    def TransformModule(self, input_0, time_idx, batch_idx, kernel_size=5, map_dim=250,
                        scope='TransformModule', reuse=True):
        self._check_dims(map_dim, kernel_size)
        return self._run(cfgmod.OP_TRANSFORM, [input_0], time_idx, batch_idx)

    def OrModule(self, input_0, input_1, time_idx=None, batch_idx=None, scope='OrModule',
                 reuse=True):
        return self._run(cfgmod.OP_OR, [input_0, input_1], None, None)

    def ExistModule(self, input_0, time_idx=None, batch_idx=None, scope='ExistModule',
                    reuse=True):
        return self._run(cfgmod.OP_EXIST, [input_0], None, None)

    def CountModule(self, input_0, time_idx=None, batch_idx=None, scope='CountModule',
                    reuse=True):
        return self._run(cfgmod.OP_COUNT, [input_0], None, None)

    def EqualNumModule(self, input_0, input_1, time_idx=None, batch_idx=None,
                       scope='EqualNumModule', reuse=True):
        return self._run(cfgmod.OP_EQUAL_NUM, [input_0, input_1], None, None)

    def MoreNumModule(self, input_0, input_1, time_idx=None, batch_idx=None,
                      scope='MoreNumModule', reuse=True):
        return self._run(cfgmod.OP_MORE_NUM, [input_0, input_1], None, None)

    def LessNumModule(self, input_0, input_1, time_idx=None, batch_idx=None,
                      scope='LessNumModule', reuse=True):
        return self._run(cfgmod.OP_LESS_NUM, [input_0, input_1], None, None)

    def SamePropertyModule(self, input_0, input_1, time_idx, batch_idx, map_dim=250,
                           scope='SamePropertyModule', reuse=True):
        self._check_dims(map_dim)
        return self._run(cfgmod.OP_SAME_PROPERTY, [input_0, input_1], time_idx, batch_idx)

    def DescribeModule(self, input_0, time_idx, batch_idx, map_dim=250, scope='DescribeModule',
                       reuse=True):
        self._check_dims(map_dim)
        return self._run(cfgmod.OP_DESCRIBE, [input_0], time_idx, batch_idx)


class ModulesSHAPES(ModulesBase):
    """models_shapes/nmn3_modules.py"""
    family = 'shapes'

    def FindModule(self, time_idx, batch_idx, map_dim=500, scope='FindModule', reuse=None):
        return super().FindModule(time_idx, batch_idx, map_dim)

    def TransformModule(self, input_0, time_idx, batch_idx, kernel_size=3, map_dim=500,
                        scope='TransformModule', reuse=None):
        self._check_dims(map_dim, kernel_size)
        return self._run(cfgmod.OP_TRANSFORM, [input_0], time_idx, batch_idx)

    def AnswerModule(self, input_0, time_idx=None, batch_idx=None, scope='AnswerModule',
                     reuse=None):
        return self._run(cfgmod.OP_EXIST, [input_0], None, None)


class ModulesVQA(ModulesBase):
    """models_vqa/nmn3_modules.py — note the extra ``encoder_states`` constructor argument; the
    reference model passes None (models_vqa/nmn3_model.py:61) and so must callers here."""
    family = 'vqa'

    def __init__(self, image_feat_grid, word_vecs, encoder_states, num_choices, **kw):
        if encoder_states is not None:
            raise NotImplementedError('encoder_states is None in the reference model '
                                      '(models_vqa/nmn3_model.py:61); that branch is not built')
        self.encoder_states = None
        super().__init__(image_feat_grid, word_vecs, num_choices, **kw)

    def FindModule(self, time_idx, batch_idx, map_dim=1024, scope='FindModule', reuse=True):
        return super().FindModule(time_idx, batch_idx, map_dim)

    def TransformModule(self, input_0, time_idx, batch_idx, kernel_size=5, map_dim=1024,
                        scope='TransformModule', reuse=True):
        self._check_dims(map_dim)
        return self._run(cfgmod.OP_FIND_SAME_PROPERTY, [input_0], time_idx, batch_idx)

    def DescribeModule(self, input_0, time_idx, batch_idx, map_dim=1024, scope='DescribeModule',
                       reuse=True):
        self._check_dims(map_dim)
        return self._run(cfgmod.OP_DESCRIBE, [input_0], time_idx, batch_idx)


MODULES_BY_FAMILY = {'clevr': ModulesCLEVR, 'shapes': ModulesSHAPES, 'vqa': ModulesVQA}
