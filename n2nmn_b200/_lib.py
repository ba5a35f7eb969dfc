"""ctypes binding of libn2nmn_b200.so (include/n2nmn_b200.h).

The library is the product; there is no Python/CPU fallback. If it has not been built
(`python -m n2nmn_b200.build` or `__graft_entry__.build()`), importing this module raises.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'lib', 'libn2nmn_b200.so')

ABI_VERSION = 2
FLAG_PROJ_FP32_SIMT = 1
FLAG_WAVE_EXECUTOR = 2
FAMILY_ID = {'clevr': 0, 'shapes': 1, 'vqa': 2}


class Config(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        'abi_version', 'family', 'H', 'W', 'D', 'text_dim', 'map_dim', 'kernel_size',
        'num_choices', 'max_batch', 'max_T', 'device', 'flags', 'max_group')]


class Seq2SeqConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        'abi_version', 'num_vocab_txt', 'embed_dim_txt', 'num_vocab_nmn', 'embed_dim_nmn',
        'lstm_dim', 'num_layers', 'T_encoder', 'T_decoder', 'max_batch', 'device', 'flags')]


class SchedInfo(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        'num_questions', 'num_valid', 'num_nodes', 'max_depth', 'num_text_nodes',
        'num_find_nodes', 'num_proj_tiles', 'num_launches')] + [
        ('algorithmic_bytes', C.c_int64), ('algorithmic_flops', C.c_int64),
        ('kernel_bytes', C.c_int64 * 3), ('kernel_flops', C.c_int64 * 3),
        ('bwd_gemm_flops', C.c_int64)]


# every symbol declared in include/n2nmn_b200.h: name -> (restype, argtypes)
_P = C.c_void_p
_I32P = C.POINTER(C.c_int32)
SIGNATURES = {
    'n2nmn_seq2seq_create': (C.c_int, [C.POINTER(Seq2SeqConfig), C.POINTER(_P)]),
    'n2nmn_seq2seq_destroy': (C.c_int, [_P]),
    'n2nmn_seq2seq_num_variables': (C.c_int, [_P]),
    'n2nmn_seq2seq_variable_info': (C.c_int, [_P, C.c_int, C.POINTER(C.c_char_p),
                                              C.POINTER(C.c_int64), C.POINTER(C.c_int)]),
    'n2nmn_seq2seq_set_weight': (C.c_int, [_P, C.c_char_p, _P, C.POINTER(C.c_int64), C.c_int, _P]),
    'n2nmn_seq2seq_set_assembler': (C.c_int, [_P, _I32P, _I32P, _I32P, _P]),
    'n2nmn_seq2seq_forward': (C.c_int, [_P, _P, _P, C.c_int, C.c_int, _P, _P, _P, _P, _P, _P, _P]),
    'n2nmn_seq2seq_forward_ex': (C.c_int, [_P, _P, _P, C.c_int, C.c_int, _P, _P, _P, _P, _P, _P, _P,
                                           _P]),
    'n2nmn_seq2seq_set_sampling': (C.c_int, [_P, _P]),
    'n2nmn_seq2seq_set_dropout': (C.c_int, [_P, _P, _P]),
    'n2nmn_seq2seq_launch_count': (C.c_int64, [_P]),
    'n2nmn_seq2seq_set_record': (C.c_int, [_P, C.c_int]),
    'n2nmn_seq2seq_backward': (C.c_int, [_P, _P, _P, _P, _P, _P]),
    'n2nmn_seq2seq_backward_ex': (C.c_int, [_P, _P, _P, _P, _P, _P, _P]),
    'n2nmn_seq2seq_flat_size': (C.c_int64, [_P]),
    'n2nmn_seq2seq_flat_offset': (C.c_int, [_P, C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    'n2nmn_seq2seq_load_flat_weights': (C.c_int, [_P, _P, _P]),
    'n2nmn_seq2seq_get_flat_weights': (C.c_int, [_P, _P, _P]),
    'n2nmn_seq2seq_adam_step': (C.c_int, [_P, _P, _P, _P, _P, C.c_int, C.c_float, C.c_float, C.c_float,
                                          C.c_float, C.c_float, C.c_float, _P]),
    'n2nmn_create': (C.c_int, [C.POINTER(Config), C.POINTER(_P)]),
    'n2nmn_destroy': (C.c_int, [_P]),
    'n2nmn_last_error': (C.c_char_p, []),
    'n2nmn_num_variables': (C.c_int, [_P]),
    'n2nmn_variable_info': (C.c_int, [_P, C.c_int, C.POINTER(C.c_char_p),
                                      C.POINTER(C.c_int64), C.POINTER(C.c_int)]),
    'n2nmn_set_weight': (C.c_int, [_P, C.c_char_p, _P, C.POINTER(C.c_int64), C.c_int, _P]),
    'n2nmn_bind_inputs': (C.c_int, [_P, _P, _P, C.c_int, C.c_int, _P]),
    'n2nmn_module_fwd': (C.c_int, [_P, C.c_int, _P, _P, _I32P, _I32P, C.c_int, _P, _P]),
    'n2nmn_scene_fwd': (C.c_int, [_P, C.c_int, C.c_float, _P, _P]),
    'n2nmn_compile_schedule': (C.c_int, [_P, _I32P, C.c_int, C.c_int, _I32P, C.c_int,
                                         C.POINTER(C.c_uint8), C.POINTER(_P)]),
    'n2nmn_compile_schedule_host': (C.c_int, [C.POINTER(Config), _I32P, C.c_int, C.c_int, _I32P,
                                              C.c_int, C.POINTER(C.c_uint8), C.POINTER(_P)]),
    'n2nmn_time_compile': (C.c_double, [C.POINTER(Config), _I32P, C.c_int, C.c_int, _I32P, C.c_int,
                                        C.c_int]),
    'n2nmn_compile_nodes': (C.c_int, [_P, _I32P, _I32P, _I32P, _I32P, _I32P, C.c_int, _I32P,
                                      C.c_int, C.POINTER(_P)]),
    'n2nmn_sched_destroy': (C.c_int, [_P]),
    'n2nmn_sched_get_info': (C.c_int, [_P, C.POINTER(SchedInfo)]),
    'n2nmn_sched_get_nodes': (C.c_int, [_P, _I32P, C.c_int]),
    'n2nmn_run_schedule': (C.c_int, [_P, _P, _P, _P, _P]),
    'n2nmn_forward_tokens': (C.c_int, [_P, _P, _P, _P, C.c_int, C.c_int, _P, C.c_int, _P, _P, _P]),
    'n2nmn_forward_group': (C.c_int, [_P, C.c_int, _P, _P, _P, C.c_int, C.c_int, _P, C.c_int, _P,
                                      _P, _P]),
    'n2nmn_forward_group_host_async': (C.c_int, [_P, C.c_int, _P, _P, _P, C.c_int, C.c_int, _P,
                                                 C.c_int, _P, _P, _P]),
    'n2nmn_forward_group_host_f16_async': (C.c_int, [_P, C.c_int, _P, _P, _P, C.c_int, C.c_int, _P,
                                                     C.c_int, _P, _P, _P]),
    'n2nmn_max_group': (C.c_int, [_P]),
    'n2nmn_last_step_info': (C.c_int, [_P, C.POINTER(SchedInfo)]),
    'n2nmn_forward_host': (C.c_int, [_P, _P, _P, _I32P, C.c_int, C.c_int, _I32P, C.c_int, _P,
                                     C.POINTER(C.c_uint8), _P]),
    'n2nmn_forward_host_async': (C.c_int, [_P, _P, _P, _I32P, C.c_int, C.c_int, _I32P, C.c_int, _P,
                                           C.POINTER(C.c_uint8), _P]),
    'n2nmn_pool_create': (C.c_int, [C.POINTER(_P), C.POINTER(_P), C.c_int, _P, C.c_int,
                                    C.POINTER(_P)]),
    'n2nmn_pool_destroy': (C.c_int, [_P]),
    'n2nmn_pool_size': (C.c_int, [_P]),
    'n2nmn_pool_submit': (C.c_int, [_P, C.c_int, _P, _P, _P, C.c_int, C.c_int, _P, _P, C.c_int]),
    'n2nmn_pool_submit_many': (C.c_int, [_P, C.c_int, _P, _P, _P, C.c_int, C.c_int, _P, _P,
                                         C.c_int]),
    'n2nmn_pool_wait': (C.c_int, [_P]),
    'n2nmn_pool_group_stats': (C.c_int, [_P, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    'n2nmn_pool_last_error': (C.c_char_p, []),
    'n2nmn_flat_size': (C.c_int64, [_P]),
    'n2nmn_flat_offset': (C.c_int, [_P, C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    'n2nmn_load_flat_weights': (C.c_int, [_P, _P, _P]),
    'n2nmn_train_backward': (C.c_int, [_P, _P, _P, _P, C.c_int, C.c_int, _P, C.c_int, _P,
                                       C.c_float, _P, _P, _P, _P, _P, _P]),
    'n2nmn_train_backward_ex': (C.c_int, [_P, _P, _P, _P, C.c_int, C.c_int, _P, C.c_int, _P,
                                          C.c_float, _P, _P, _P, _P, _P, _P, _P, _P]),
    'n2nmn_adam_step': (C.c_int, [_P, _P, _P, _P, _P, C.c_int, C.c_float, C.c_float, C.c_float,
                                  C.c_float, C.c_float, C.c_float, _P]),
    'n2nmn_train_finish': (C.c_int, [_P, _P, _P, _P, _P, C.c_int, C.c_float, C.c_float, C.c_float,
                                     C.c_float, C.c_float, C.c_float, _P, _P, _P, C.c_int, C.c_int,
                                     C.c_float, _P, _P, _P, _P]),
    'n2nmn_set_grad_scale': (C.c_int, [_P, C.c_float]),
    'n2nmn_set_tree_cluster': (C.c_int, [_P, C.c_int]),
    'n2nmn_set_proj_ctas': (C.c_int, [_P, C.c_int]),
    'n2nmn_set_text_ctas_per_group': (C.c_int, [_P, C.c_int]),
    'n2nmn_set_profiling': (C.c_int, [_P, C.c_int]),
    'n2nmn_get_launch_times': (C.c_int, [_P, C.POINTER(C.c_char_p), C.POINTER(C.c_float),
                                         C.c_int]),
    'n2nmn_launch_count': (C.c_int64, [_P]),
    'n2nmn_crc32c': (C.c_uint32, [_P, C.c_size_t, C.c_uint32]),
}


def load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            'n2nmn_b200: %s is missing. Build it with `python -m n2nmn_b200.build` (needs nvcc, '
            'sm_90a). There is no CPU fallback.' % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)     # AttributeError if the .so lacks a declared symbol
        fn.restype = res
        fn.argtypes = args
    return lib


class N2NMNError(RuntimeError):
    pass


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = load()
    return _lib


def check(rc):
    if rc < 0:
        msg = lib().n2nmn_last_error()
        raise N2NMNError('n2nmn_b200 error %d: %s' % (rc, (msg or b'').decode()))
    return rc
