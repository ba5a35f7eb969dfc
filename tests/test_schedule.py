"""CPU: the C++ layout compiler (n2nmn_compile_schedule_host) applies exactly the assembler's
stack discipline — checked against the Python Assembler drop-in and, through it, the goldens
produced by the reference's own nmn3_assembler.py."""
import ctypes as C
import json
import os
import re

import numpy as np
import pytest

from n2nmn_b200 import _lib, config as cfgmod, synth
from n2nmn_b200.assembler import Assembler, INVALID_EXPR
from tests.helpers import GOLDEN

SHAPES = {'clevr': dict(H=10, W=15, D=512, C=28), 'shapes': dict(H=3, W=3, D=64, C=2),
          'vqa': dict(H=14, W=14, D=64, C=37)}


def host_compile(family, tokens):
    lib = _lib.lib()
    fam = cfgmod.FAMILIES[family]
    asm = Assembler(synth.vocab_file(family))
    s = SHAPES[family]
    T, N = tokens.shape
    cfg = _lib.Config(abi_version=_lib.ABI_VERSION, family=_lib.FAMILY_ID[family], H=s['H'],
                      W=s['W'], D=s['D'], text_dim=300, map_dim=fam.map_dim,
                      kernel_size=fam.kernel_size, num_choices=s['C'], max_batch=N, max_T=T,
                      device=0, flags=0)
    vocab_ops = np.array([fam.token_ops.get(n, -1) for n in asm.module_names], np.int32)
    tok = np.ascontiguousarray(tokens, np.int32)
    validity = np.zeros(N, np.uint8)
    h = C.c_void_p()
    _lib.check(lib.n2nmn_compile_schedule_host(
        C.byref(cfg), tok.ctypes.data_as(C.POINTER(C.c_int32)), T, N,
        vocab_ops.ctypes.data_as(C.POINTER(C.c_int32)), len(vocab_ops),
        validity.ctypes.data_as(C.POINTER(C.c_uint8)), C.byref(h)))
    info = _lib.SchedInfo()
    _lib.check(lib.n2nmn_sched_get_info(h, C.byref(info)))
    nodes = np.zeros((max(info.num_nodes, 1), 6), np.int32)
    _lib.check(lib.n2nmn_sched_get_nodes(h, nodes.ctypes.data_as(C.POINTER(C.c_int32)),
                                         max(info.num_nodes, 1)))
    lib.n2nmn_sched_destroy(h)
    return validity.astype(bool), nodes[:info.num_nodes], info, asm


def flatten(expr_list, token_ops):
    """Post-order node list of the valid expressions: (op, t, b, depth, in0, in1)."""
    rows = []

    def walk(e):
        kids = [walk(e[k]) for k in ('input_0', 'input_1') if k in e]
        depth = 1 + max([rows[k][3] for k in kids], default=0)
        rows.append([token_ops[e['module']], e['time_idx'], e['batch_idx'], depth,
                     kids[0] if kids else -1, kids[1] if len(kids) > 1 else -1])
        return len(rows) - 1

    for e in expr_list:
        if e['module'] != INVALID_EXPR:
            walk(e)
    return np.array(rows, np.int32).reshape(-1, 6)


@pytest.mark.parametrize('family', ['clevr', 'shapes', 'vqa'])
def test_cpp_compiler_matches_assembler_on_reference_goldens(family):
    with open(os.path.join(GOLDEN, 'golden_assembler.json')) as f:
        g = json.load(f)[family]
    tokens = np.array(g['tokens'], np.int32)
    validity, nodes, info, asm = host_compile(family, tokens)
    assert validity.tolist() == g['validity']
    want = flatten(g['expr_list'], cfgmod.FAMILIES[family].token_ops)
    np.testing.assert_array_equal(nodes, want)
    assert info.num_valid == sum(g['validity'])


def test_cpp_compiler_random_fuzz_vs_python_assembler():
    rng = np.random.RandomState(3)
    asm = Assembler(synth.vocab_file('clevr'))
    for trial in range(20):
        T, N = int(rng.randint(2, 21)), int(rng.randint(1, 65))
        tokens = rng.randint(0, asm.num_vocab_nmn, size=(T, N)).astype(np.int32)
        # bias towards short valid-looking prefixes
        tokens[0] = rng.choice([0, 1], size=N)
        tokens[rng.randint(1, T, size=N), np.arange(N)] = asm.EOS_idx
        if trial % 2:
            tokens = np.concatenate([tokens, synth.random_valid_tokens(asm, 8, T, seed=trial)], 1) \
                if T >= 3 else tokens
        validity, nodes, info, _ = host_compile('clevr', tokens)
        exprs, pv = asm.assemble(tokens)
        assert validity.tolist() == pv.tolist()
        np.testing.assert_array_equal(nodes, flatten(exprs, cfgmod.CLEVR.token_ops))


def test_schedule_accounting_matches_survey_example():
    """[_Find,_Transform,_Filter,_Count] = 621,712 algorithmic bytes (SURVEY.md §8d)."""
    asm = Assembler(synth.vocab_file('clevr'))
    tokens = synth.tokens_from_layouts(asm, [['_Find', '_Transform', '_Filter', '_Count']], 8)
    validity, nodes, info, _ = host_compile('clevr', tokens)
    assert validity.all() and info.num_nodes == 4 and info.max_depth == 4
    assert info.algorithmic_bytes == 621712
    assert abs(info.algorithmic_flops - 79.8e6) < 0.5e6
    assert info.num_find_nodes == 2 and info.num_text_nodes == 3


def test_contraction_tiles_one_per_layer_and_pass():
    """num_proj_tiles counts the contraction's 128-row tiles: one per (rows, layer, pass of <= 8
    fused Find consumers)."""
    asm = Assembler(synth.vocab_file('clevr'))
    N = 10   # 10 images x 150 pixels = 12 tiles of 128 rows
    one = synth.tokens_from_layouts(asm, [['_Find', '_Exist']] * N, 12)
    assert host_compile('clevr', one)[2].num_proj_tiles == 12
    nine = synth.tokens_from_layouts(asm, [['_Find'] + ['_Filter'] * 8 + ['_Exist']] * N, 12)
    assert host_compile('clevr', nine)[2].num_proj_tiles == 24


def test_capi_exports_every_declared_symbol():
    """The .so loads and exports exactly what include/n2nmn_b200.h declares (no compute here)."""
    hdr = open(os.path.join(os.path.dirname(GOLDEN), '..', 'include', 'n2nmn_b200.h')).read()
    declared = set(re.findall(r'\b(n2nmn_[a-z_0-9]+)\s*\(', hdr))
    assert declared == set(_lib.SIGNATURES), declared ^ set(_lib.SIGNATURES)
    lib = _lib.load()
    for name in declared:
        assert hasattr(lib, name)
    assert lib.n2nmn_last_error() is not None
