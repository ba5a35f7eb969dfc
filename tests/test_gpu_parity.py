"""GPU parity: the CUDA path (through the C ABI) vs the goldens made from the reference's module
code and vs the numpy oracle, for all three families, both executors and both projection
kernels (wgmma TF32 default, fp32 CUDA-core verification path).

Tolerance: 1e-3 absolute on attention maps and answer logits (north_star), tightened to 2e-4
for the fp32 CUDA-core projection."""
import numpy as np
import pytest
import torch

from n2nmn_b200 import _lib, synth
from n2nmn_b200.assembler import Assembler
from tests.helpers import case_inputs, load_golden, node_inputs

pytestmark = pytest.mark.gpu
FAMILIES = ['clevr', 'shapes', 'vqa']
TOL = {0: 1e-3, _lib.FLAG_PROJ_FP32_SIMT: 2e-4}


def make_executor(family, feat, word_vecs, C, W, flags=0, **kw):
    from n2nmn_b200.executor import LayoutExecutor
    asm = Assembler(synth.vocab_file(family))
    return LayoutExecutor(family, torch.from_numpy(feat).cuda(), torch.from_numpy(word_vecs).cuda(),
                          C, asm, weights=W, flags=flags, **kw)


@pytest.mark.parametrize('flags', [_lib.FLAG_PROJ_FP32_SIMT, 0])
@pytest.mark.parametrize('family', FAMILIES)
def test_modules_match_reference_goldens(family, flags):
    z, meta = load_golden(family)
    feat, word_vecs, W = case_inputs(meta)
    ex = make_executor(family, feat, word_vecs, meta['C'], W, flags=flags, max_T=meta['T'])
    m = ex.modules
    worst = {}
    for k, (name, arity) in enumerate(meta['module_calls']):
        t, b, a0, a1 = node_inputs(meta, 5, meta['node_seed_base'] + k)
        out = getattr(m, name)(*(a0, a1)[:arity], t, b)
        torch.cuda.synchronize()
        ref = z['mod_' + name]
        assert tuple(out.shape) == ref.shape, name
        worst[name] = float(np.max(np.abs(out.cpu().numpy() - ref)))
    print(family, 'flags', flags, 'max abs err per module:', worst)
    bad = {k: v for k, v in worst.items() if not v <= TOL[flags]}
    assert not bad, bad


@pytest.mark.parametrize('flags', [_lib.FLAG_PROJ_FP32_SIMT, 0, _lib.FLAG_WAVE_EXECUTOR,
                                   _lib.FLAG_WAVE_EXECUTOR | _lib.FLAG_PROJ_FP32_SIMT])
@pytest.mark.parametrize('family', FAMILIES)
def test_executor_matches_reference_goldens(family, flags):
    z, meta = load_golden(family)
    feat, word_vecs, W = case_inputs(meta)
    ex = make_executor(family, feat, word_vecs, meta['C'], W, flags=flags, max_T=meta['T'])
    tol = TOL[flags & _lib.FLAG_PROJ_FP32_SIMT]
    cb = ex.compile_tokens(z['exec_tokens'])
    assert cb.validity.tolist() == [bool(v) for v in z['exec_validity']]
    scores, arena = ex.run(cb, return_att=True)
    torch.cuda.synchronize()
    scores, arena = scores.cpu().numpy(), arena.cpu().numpy()
    err_s = float(np.max(np.abs(scores - z['exec_scores'])))
    nodes = cb.nodes()
    err_a = 0.0
    n_att = 0
    for i, (op, t, b, depth, in0, in1) in enumerate(nodes):
        key = 'att_b%d_t%d' % (b, t)
        if key in z.files:
            err_a = max(err_a, float(np.max(np.abs(arena[i] - z[key]))))
            n_att += 1
    print(family, 'flags', flags, 'scores err', err_s, 'att err', err_a, 'att maps', n_att)
    assert n_att == sum(1 for k in z.files if k.startswith('att_b'))
    assert err_s <= tol and err_a <= tol
    for i, v in enumerate(cb.validity):
        if not v:
            assert not scores[i].any()
    # the dict route (compiler.build_feed_dict) gives the same numbers as the token route
    exprs, _ = ex.assembler.assemble(z['exec_tokens'])
    s2 = ex.run(ex.compiler.build_feed_dict(exprs)).cpu().numpy()
    np.testing.assert_array_equal(s2, scores)


def _oracle_scores(family, feat, word_vecs, C, W, tokens):
    from oracle.nmn_oracle import OracleModules, run_depth_batched
    asm = Assembler(synth.vocab_file(family))
    exprs, valid = asm.assemble(tokens)
    m = OracleModules(feat, word_vecs, C, W, family=family)
    s, att = run_depth_batched(m, exprs, return_att=True)
    return s, att, valid


@pytest.mark.parametrize('flags', [0, _lib.FLAG_WAVE_EXECUTOR])
def test_clevr_batch64_vs_oracle(flags):
    """BASELINE config 2 shape: B=64, 10x15x512, T=20, expert mix + random valid layouts."""
    from n2nmn_b200 import weights as wts
    N, H, Wd, D, T, C = 64, 10, 15, 512, 20, 28
    feat, word_vecs = synth.make_inputs(N, H, Wd, D, T, seed=1234)
    W = wts.init_weights('clevr', H, Wd, D, C, seed=0, bias_std=0.1)
    ex = make_executor('clevr', feat, word_vecs, C, W, flags=flags)
    asm = ex.assembler
    for name, tokens in [('expert', synth.expert_mix_tokens(asm, N, T)),
                         ('random', synth.random_valid_tokens(asm, N, T, seed=7)),
                         ('deep', synth.random_valid_tokens(asm, N, T, seed=9, ans_weight=0.15,
                                                            min_depth=3, max_depth=12))]:
        cb = ex.compile_tokens(tokens)
        scores, arena = ex.run(cb, return_att=True)
        torch.cuda.synchronize()
        ref_s, ref_att, valid = _oracle_scores('clevr', feat, word_vecs, C, W, tokens)
        assert cb.validity.tolist() == valid.tolist()
        err_s = float(np.max(np.abs(scores.cpu().numpy() - ref_s)))
        arena = arena.cpu().numpy()
        err_a = 0.0
        for i, (op, t, b, depth, in0, in1) in enumerate(cb.nodes()):
            if (b, t) in ref_att:
                err_a = max(err_a, float(np.max(np.abs(arena[i] - ref_att[(b, t)]))))
        print(name, 'flags', flags, 'nodes', cb.info['num_nodes'], 'depth', cb.info['max_depth'],
              'scores err', err_s, 'att err', err_a)
        assert err_s <= 1e-3 and err_a <= 1e-3


def test_many_find_nodes_per_image_and_ragged_inputs():
    """> 8 Find/Filter nodes on one image (second projection pass), invalid rows interleaved,
    a batch that is not a multiple of anything, T at the context maximum."""
    from n2nmn_b200 import weights as wts
    N, H, Wd, D, T, C = 5, 10, 15, 512, 24, 28
    feat, word_vecs = synth.make_inputs(N, H, Wd, D, T, seed=77)
    W = wts.init_weights('clevr', H, Wd, D, C, seed=3, bias_std=0.1)
    ex = make_executor('clevr', feat, word_vecs, C, W)
    asm = ex.assembler
    long_chain = ['_Find'] + ['_Filter'] * 10 + ['_Count']            # 11 find-type nodes
    many_and = ['_Find', '_Find', '_And'] + ['_Find', '_And'] * 8 + ['_Exist']   # 10 finds
    layouts = [long_chain, ['_Find', '_Transform'], many_and, ['_Scene', '_Exist'],
               ['_And', '_Count']]
    tokens = synth.tokens_from_layouts(asm, layouts, T)
    cb = ex.compile_tokens(tokens)
    assert cb.validity.tolist() == [True, False, True, True, False]
    scores = ex.run(cb).cpu().numpy()
    ref_s, _, _ = _oracle_scores('clevr', feat, word_vecs, C, W, tokens)
    assert not scores[1].any() and not scores[4].any()
    assert float(np.max(np.abs(scores - ref_s))) <= 1e-3


def test_zero_size_module_call_and_errors():
    """n == 0 (TF Fold's empty batches) is a no-op; bad arguments fail loudly, never silently."""
    from n2nmn_b200 import weights as wts
    N, H, Wd, D, T, C = 2, 10, 15, 512, 4, 28
    feat, word_vecs = synth.make_inputs(N, H, Wd, D, T, seed=5)
    ex = make_executor('clevr', feat, word_vecs, C,
                       wts.init_weights('clevr', H, Wd, D, C, seed=1))
    m = ex.modules
    out = m.FindModule(np.zeros(0, np.int32), np.zeros(0, np.int32))
    assert tuple(out.shape) == (0, H, Wd, 1)
    with pytest.raises(_lib.N2NMNError):
        m.FindModule(np.array([0], np.int32), np.array([N], np.int32))     # batch_idx out of range
    with pytest.raises(ValueError):
        m.FindModule(np.array([0], np.int32), np.array([0], np.int32), map_dim=123)
    with pytest.raises(_lib.N2NMNError):
        ex.compile_tokens(np.zeros((T + 1, N), np.int32))                   # T above capacity


def test_forward_device_single_call_matches_compiled_path():
    from n2nmn_b200 import weights as wts
    N, H, Wd, D, T, C = 64, 10, 15, 512, 20, 28
    feat, word_vecs = synth.make_inputs(N, H, Wd, D, T, seed=31)
    W = wts.init_weights('clevr', H, Wd, D, C, seed=2, bias_std=0.1)
    ex = make_executor('clevr', feat, word_vecs, C, W)
    tokens = synth.random_valid_tokens(ex.assembler, N, T, seed=11)
    tokens[:, 5] = ex.assembler.module_list2tokens(['_Find', '_Find'], T)   # an invalid column
    ref, valid = ex.forward_tokens(tokens)
    f2, w2 = synth.make_inputs(N, H, Wd, D, T, seed=32)     # rebinding to other buffers works
    other, _ = ex.forward_device(torch.from_numpy(f2).cuda(), torch.from_numpy(w2).cuda(), tokens)
    got, valid2 = ex.forward_device(torch.from_numpy(feat).cuda(),
                                    torch.from_numpy(word_vecs).cuda(), tokens)
    torch.cuda.synchronize()
    assert valid.tolist() == valid2.tolist() and not valid2[5]
    np.testing.assert_array_equal(got.cpu().numpy(), ref.cpu().numpy())
    assert not np.array_equal(other.cpu().numpy(), ref.cpu().numpy())
    assert ex.last_step_info()['num_questions'] == N


@pytest.mark.parametrize('cluster', ['1', '2', '4'])
def test_tree_cluster_sizes_agree(cluster):
    """The tree kernel gives the same scores whether a question runs on 1, 2 or 4 CTAs."""
    from n2nmn_b200 import weights as wts
    N, H, Wd, D, T, C = 24, 10, 15, 512, 20, 28
    feat, word_vecs = synth.make_inputs(N, H, Wd, D, T, seed=41)
    W = wts.init_weights('clevr', H, Wd, D, C, seed=4, bias_std=0.1)
    ex = make_executor('clevr', feat, word_vecs, C, W)
    ex.set_tree_cluster(int(cluster))
    tokens = synth.expert_mix_tokens(ex.assembler, N, T)
    scores, _ = ex.forward_tokens(tokens)
    ref_s, _, _ = _oracle_scores('clevr', feat, word_vecs, C, W, tokens)
    assert float(np.max(np.abs(scores.cpu().numpy() - ref_s))) <= 1e-3


def test_tuning_knobs_do_not_change_results():
    """n2nmn_set_tree_cluster / _proj_ctas / _text_ctas_per_group are tuning only: the contraction
    grid cap and the text kernel's column walk give bit-identical scores; cluster sizes agree to
    rounding (the split of a reduction changes its order). Bad values are rejected."""
    from n2nmn_b200 import weights as wts
    N, H, Wd, D, T, C = 40, 10, 15, 512, 20, 28
    feat, word_vecs = synth.make_inputs(N, H, Wd, D, T, seed=51)
    W = wts.init_weights('clevr', H, Wd, D, C, seed=5, bias_std=0.1)
    ex = make_executor('clevr', feat, word_vecs, C, W)
    tokens = synth.random_valid_tokens(ex.assembler, N, T, seed=52)
    f, w = torch.from_numpy(feat).cuda(), torch.from_numpy(word_vecs).cuda()
    base = ex.forward_device(f, w, tokens)[0].cpu().numpy().copy()
    for proj_ctas, text_ctas in [(7, 0), (32, 1), (1, 2), (0, 3)]:
        ex.set_proj_ctas(proj_ctas)
        ex.set_text_ctas_per_group(text_ctas)
        got = ex.forward_device(f, w, tokens)[0].cpu().numpy()
        np.testing.assert_array_equal(got, base)
    ex.set_proj_ctas(0)
    ex.set_text_ctas_per_group(0)
    for cs in (1, 2, 4, 0):
        ex.set_tree_cluster(cs)
        got = ex.forward_device(f, w, tokens)[0].cpu().numpy()
        assert float(np.max(np.abs(got - base))) <= 2e-5
    for bad in (lambda: ex.set_tree_cluster(3), lambda: ex.set_proj_ctas(-1),
                lambda: ex.set_text_ctas_per_group(-2)):
        with pytest.raises(_lib.N2NMNError):
            bad()


def test_executor_pool_threads_match_single_context():
    from n2nmn_b200 import weights as wts
    from n2nmn_b200.executor import ExecutorPool
    N, H, Wd, D, T, C = 32, 10, 15, 512, 20, 28
    W = wts.init_weights('clevr', H, Wd, D, C, seed=6, bias_std=0.1)
    asm = Assembler(synth.vocab_file('clevr'))
    items = []
    for i in range(7):
        f, w = synth.make_inputs(N, H, Wd, D, T, seed=200 + i)
        items.append((torch.from_numpy(f).cuda(), torch.from_numpy(w).cuda(),
                      synth.random_valid_tokens(asm, N, T, seed=300 + i)))
    pool = ExecutorPool('clevr', items[0][0], items[0][1], C, asm, weights=W, num_streams=3)
    outs = [torch.empty((N, C), device='cuda') for _ in items]
    pool.begin()
    pool.forward_many([x[0] for x in items], [x[1] for x in items], [x[2] for x in items], outs)
    pool.end()
    torch.cuda.synchronize()
    ex = pool.executors[0]
    for (f, w, tok), got in zip(items, outs):
        want, _ = ex.forward_device(f, w, tok)
        torch.cuda.synchronize()
        np.testing.assert_array_equal(got.cpu().numpy(), want.cpu().numpy())
    # the same batches from pinned host buffers (H2D, kernels, D2H all enqueued by the workers),
    # one of them with an invalid layout: validity comes back through the worker as well
    toks = [x[2].copy() for x in items]
    toks[3][:, 5] = asm.name2idx_dict['_Find']          # Find Find Find ... never terminates
    hf = [x[0].cpu().pin_memory() for x in items]
    hw = [x[1].cpu().pin_memory() for x in items]
    hs = [torch.empty((N, C)).pin_memory() for _ in items]
    pool.begin()
    valids = [pool.submit_host(f, w, t, o)[1] for f, w, t, o in zip(hf, hw, toks, hs)]
    pool.end()
    torch.cuda.synchronize()
    for (f, w, _), tok, got, valid in zip(items, toks, hs, valids):
        want, v = ex.forward_device(f, w, tok)
        torch.cuda.synchronize()
        np.testing.assert_array_equal(got.numpy(), want.cpu().numpy())
        assert valid.tolist() == v.tolist()
    assert not valids[3][5] and valids[3][4]
    # errors raised inside a worker surface at end()
    import pytest as _pt
    pool.begin()
    pool.submit(items[0][0], items[0][1], np.zeros((T + 50, N), np.int32))   # T beyond capacity
    with _pt.raises(Exception):
        pool.end()


def test_fp16_host_feature_store_matches_device_path_and_oracle():
    """n2nmn_forward_group_host_f16_async (pool.submit_host with float16 features): bit-identical
    to the device path fed the same fp16-rounded values as fp32 (the widening is exact), and within
    1e-3 of the oracle on the ORIGINAL fp32 features at the BASELINE batch (measured ~1e-4)."""
    from n2nmn_b200 import weights as wts
    from n2nmn_b200.executor import ExecutorPool
    N, H, Wd, D, T, C = 64, 10, 15, 512, 20, 28
    W = wts.init_weights('clevr', H, Wd, D, C, seed=0, bias_std=0.1)
    asm = Assembler(synth.vocab_file('clevr'))
    items = []
    for i in range(5):
        f, w = synth.make_inputs(N, H, Wd, D, T, seed=1234 + i)
        tok = (synth.expert_mix_tokens(asm, N, T) if i % 2 == 0 else
               synth.random_valid_tokens(asm, N, T, seed=7 + i))
        items.append((f, w, tok))
    pool = ExecutorPool('clevr', torch.from_numpy(items[0][0]).cuda(),
                        torch.from_numpy(items[0][1]).cuda(), C, asm, weights=W, num_streams=2,
                        max_group=3)
    hf = [torch.from_numpy(f).half().pin_memory() for f, _, _ in items]
    hw = [torch.from_numpy(w).pin_memory() for _, w, _ in items]
    hs = [torch.empty((N, C)).pin_memory() for _ in items]
    pool.begin()
    valids = [pool.submit_host(f, w, t[2], o)[1] for f, w, t, o in zip(hf, hw, items, hs)]
    pool.end()
    torch.cuda.synchronize()
    ex = pool.executors[0]
    for (f, w, tok), h16, got, valid in zip(items, hf, hs, valids):
        want, v = ex.forward_device(h16.float().cuda(), torch.from_numpy(w).cuda(), tok)
        torch.cuda.synchronize()
        np.testing.assert_array_equal(got.numpy(), want.cpu().numpy())
        assert valid.all() and valid.tolist() == v.tolist()
    ref_s, _, _ = _oracle_scores('clevr', items[0][0], items[0][1], C, W, items[0][2])
    err = float(np.max(np.abs(hs[0].numpy() - ref_s)))
    print('fp16 feature store vs fp32 oracle: max |d scores| = %.3g' % err)
    assert err <= 1e-3
    # the same through a pre-marshalled block (n2nmn_pool_submit_many, host_io = 2)
    hs2 = [torch.empty((N, C)).pin_memory() for _ in items]
    blk = pool.make_block(hf, hw, [x[2] for x in items], hs2, host_io=True)
    assert blk['host_io'] == 2
    pool.begin()
    pool.submit_block(blk)
    pool.end()
    torch.cuda.synchronize()
    for a, b in zip(hs, hs2):
        np.testing.assert_array_equal(a.numpy(), b.numpy())


@pytest.mark.parametrize('N', [1, 2, 5, 64])
def test_forward_group_equals_separate_batches(N):
    """n2nmn_forward_group: G independent batches in one set of launches give bit-identical scores
    to G separate calls — every group size up to the capacity, batch sizes whose tile counts are
    odd (filler half of a CTA pair) or not multiples of a tile, an invalid layout in the middle,
    and the fp32 CUDA-core contraction as a second opinion."""
    from n2nmn_b200 import weights as wts
    H, Wd, D, T, C = 10, 15, 512, 12, 28
    W = wts.init_weights('clevr', H, Wd, D, C, seed=16, bias_std=0.1)
    asm = Assembler(synth.vocab_file('clevr'))
    items = []
    for i in range(16):
        f, w = synth.make_inputs(N, H, Wd, D, T, seed=400 + i)
        tok = synth.random_valid_tokens(asm, N, T, seed=500 + i)
        items.append((torch.from_numpy(f).cuda(), torch.from_numpy(w).cuda(), tok))
    items[3][2][:, 0] = asm.name2idx_dict['_Find']      # never terminates: invalid -> zero row
    for flags in (0, _lib.FLAG_PROJ_FP32_SIMT):
        ex = make_executor('clevr', items[0][0].cpu().numpy(), items[0][1].cpu().numpy(), C, W,
                           flags=flags, max_batch=N, max_T=T, max_group=16)
        ex.set_tree_cluster(1)   # (the automatic cluster size depends on the question count, and
        single = []              #  a different split of a reduction changes its rounding)
        for f, w, tok in items:
            sc, v = ex.forward_device(f, w, tok)
            single.append((sc.cpu().numpy().copy(), v.copy()))
        assert not single[3][1][0] and not single[3][0][0].any()
        for G in (1, 2, 3, 8, 16):
            outs, valids = ex.forward_group([x[0] for x in items[:G]], [x[1] for x in items[:G]],
                                            [x[2] for x in items[:G]])
            torch.cuda.synchronize()
            for g in range(G):
                np.testing.assert_array_equal(outs[g].cpu().numpy(), single[g][0])
                assert valids[g].tolist() == single[g][1].tolist()
        with pytest.raises(_lib.N2NMNError):   # more batches than the context was created for
            ex2 = make_executor('clevr', items[0][0].cpu().numpy(), items[0][1].cpu().numpy(), C,
                                W, max_batch=N, max_T=T, max_group=2)
            ex2.forward_group([x[0] for x in items[:3]], [x[1] for x in items[:3]],
                              [x[2] for x in items[:3]])


def test_host_e2e_entry_matches_device_path():
    from n2nmn_b200 import weights as wts
    N, H, Wd, D, T, C = 16, 10, 15, 512, 10, 28
    feat, word_vecs = synth.make_inputs(N, H, Wd, D, T, seed=21)
    W = wts.init_weights('clevr', H, Wd, D, C, seed=2, bias_std=0.1)
    ex = make_executor('clevr', feat, word_vecs, C, W)
    tokens = synth.expert_mix_tokens(ex.assembler, N, T)
    dev_scores, valid = ex.forward_tokens(tokens)
    host_scores, valid2 = ex.forward_host(torch.from_numpy(feat).pin_memory(),
                                          torch.from_numpy(word_vecs).pin_memory(), tokens)
    assert valid.tolist() == valid2.tolist()
    np.testing.assert_array_equal(host_scores.numpy(), dev_scores.cpu().numpy())


# ---- the other BASELINE.json configurations at their real grid / channel / head sizes -----------
def _check_family_batch(family, N, H, Wd, D, T, C, tokens, flags=0, tol=1e-3, **kw):
    from n2nmn_b200 import weights as wts
    feat, word_vecs = synth.make_inputs(N, H, Wd, D, T, seed=900 + N)
    W = wts.init_weights(family, H, Wd, D, C, seed=9, bias_std=0.1)
    ex = make_executor(family, feat, word_vecs, C, W, flags=flags, **kw)
    cb = ex.compile_tokens(tokens)
    scores, arena = ex.run(cb, return_att=True)
    torch.cuda.synchronize()
    ref_s, ref_att, valid = _oracle_scores(family, feat, word_vecs, C, W, tokens)
    assert cb.validity.tolist() == valid.tolist()
    err_s = float(np.max(np.abs(scores.cpu().numpy() - ref_s)))
    arena = arena.cpu().numpy()
    err_a = 0.0
    for i, (op, t, b, depth, in0, in1) in enumerate(cb.nodes()):
        if (b, t) in ref_att:
            err_a = max(err_a, float(np.max(np.abs(arena[i] - ref_att[(b, t)]))))
    print(family, 'N', N, 'nodes', cb.info['num_nodes'], 'depth', cb.info['max_depth'],
          'scores err', err_s, 'att err', err_a)
    assert err_s <= tol and err_a <= tol
    return ex


def test_config1_shapes_batch32_real_layout_mix():
    """SHAPES gt-layout eval, batch 32, 3x3x64 grid, map_dim 500, kernel 3, the three real layouts."""
    asm = Assembler(synth.vocab_file('shapes'))
    tokens = synth.histogram_tokens(asm, synth.SHAPES_LAYOUTS, 32, 11, seed=3)
    for flags in (0, _lib.FLAG_WAVE_EXECUTOR):
        _check_family_batch('shapes', 32, 3, 3, 64, 11, 2, tokens, flags=flags)


def test_config4_vqa_14x14x512_map1024_3001_choices():
    """VQA gt-layout eval shapes: 14x14 grid, 512(+2 coord) channels, map_dim 1024 (4 N-tiles),
    3001 answer choices (head weights too large for smem), real layout histogram, T=13."""
    asm = Assembler(synth.vocab_file('vqa'))
    tokens = synth.histogram_tokens(asm, synth.VQA_LAYOUTS, 12, 13, seed=4)
    tokens[:, 0] = asm.module_list2tokens(['_Find', '_Transform', '_Find', '_And', '_Describe'], 13)
    _check_family_batch('vqa', 12, 14, 14, 512, 13, 3001, tokens)


@pytest.mark.parametrize('family,H,Wd,D,T,C,layouts', [
    ('shapes', 3, 3, 64, 11, 2, 'SHAPES_LAYOUTS'), ('vqa', 14, 14, 512, 13, 3001, 'VQA_LAYOUTS')])
def test_pool_narrow_mode_other_families(family, H, Wd, D, T, C, layouts):
    """The pool's narrow configuration (one CTA per question, capped contraction grid, one text
    CTA per node group, 12 worker threads) on the SHAPES and VQA shapes (Mp = 512 / 1024: several
    column blocks and N-tiles per CTA) gives the scores of a single default context."""
    from n2nmn_b200 import weights as wts
    from n2nmn_b200.executor import ExecutorPool, LayoutExecutor
    N = 10
    asm = Assembler(synth.vocab_file(family))
    W = wts.init_weights(family, H, Wd, D, C, seed=8, bias_std=0.1)
    items = []
    for i in range(5):
        f, w = synth.make_inputs(N, H, Wd, D, T, seed=700 + i)
        items.append((torch.from_numpy(f).cuda(), torch.from_numpy(w).cuda(),
                      synth.histogram_tokens(asm, getattr(synth, layouts), N, T, seed=70 + i)))
    pool = ExecutorPool(family, items[0][0], items[0][1], C, asm, weights=W, num_streams=12,
                        max_batch=N, max_T=T)
    assert (pool.tree_cluster, pool.proj_ctas, pool.text_ctas_per_group) == (1, 0, 1)
    assert pool.max_group == max(1, min(16, 1024 // N))
    pool.begin()
    outs = [pool.submit(f, w, tok)[0] for f, w, tok in items]
    pool.end()
    torch.cuda.synchronize()
    groups, jobs = pool.group_stats()
    assert jobs == len(items) and 1 <= groups <= jobs
    ref_ex = LayoutExecutor(family, items[0][0], items[0][1], C, asm, weights=W, max_batch=N, max_T=T)
    for (f, w, tok), got in zip(items, outs):
        want, _ = ref_ex.forward_device(f, w, tok)
        torch.cuda.synchronize()
        assert float(np.max(np.abs(got.cpu().numpy() - want.cpu().numpy()))) <= 2e-5


def test_config5_stress_20x20x1024_depth16():
    """Synthetic stress shapes: 20x20x1024 grid, CLEVR module set, T=40, layouts of depth up to 16
    (the deepest ones exceed the shared-memory attention stack and take the wave executor)."""
    asm = Assembler(synth.vocab_file('clevr'))
    tokens = synth.random_valid_tokens(asm, 12, 40, seed=21, ans_weight=0.08, min_depth=8,
                                       max_depth=16)
    depths = [synth.layout_depth(asm, tokens[:, i]) for i in range(12)]
    assert max(depths) >= 12
    _check_family_batch('clevr', 12, 20, 20, 1024, 40, 28, tokens)


# ---- BASELINE configs 4 and 5 at their REAL batch sizes (VERDICT r1 weak #6): several N-tiles per
#      work item (Mp = 1024), multi-tile persistent CTA pairs, the reference's 2048(+2) channels
def _real_size_case(family, N, H, Wd, D, T, C, tokens, seed, group=0):
    from n2nmn_b200 import weights as wts
    from n2nmn_b200.executor import ExecutorPool
    feat, word_vecs = synth.make_inputs(N, H, Wd, D, T, seed=seed)
    W = wts.init_weights(family, H, Wd, D, C, seed=9, bias_std=0.1)
    ex = make_executor(family, feat, word_vecs, C, W, max_batch=N, max_T=T)
    cb = ex.compile_tokens(tokens)
    scores, arena = ex.run(cb, return_att=True)
    torch.cuda.synchronize()
    ref_s, ref_att, valid = _oracle_scores(family, feat, word_vecs, C, W, tokens)
    assert cb.validity.tolist() == valid.tolist()
    scores_np, arena = scores.cpu().numpy(), arena.cpu().numpy()
    err_s = float(np.max(np.abs(scores_np - ref_s)))
    err_a = 0.0
    for i, (op, t, b, depth, in0, in1) in enumerate(cb.nodes()):
        if (b, t) in ref_att:
            err_a = max(err_a, float(np.max(np.abs(arena[i] - ref_att[(b, t)]))))
    print(family, 'N', N, 'D', D, 'nodes', cb.info['num_nodes'], 'depth', cb.info['max_depth'],
          'scores err', err_s, 'att err', err_a, 'max |score|', float(np.abs(ref_s).max()))
    assert err_s <= 1e-3 and err_a <= 1e-3
    if group:   # the same batch three times through the pool's dynamic batching: same numbers
        f, w = torch.from_numpy(feat).cuda(), torch.from_numpy(word_vecs).cuda()
        del ex
        pool = ExecutorPool(family, f, w, C, Assembler(synth.vocab_file(family)), weights=W,
                            num_streams=2, max_batch=N, max_T=T, max_group=group)
        pool.begin()
        outs = [pool.submit(f, w, tokens)[0] for _ in range(3)]
        pool.end()
        torch.cuda.synchronize()
        for o in outs:
            assert float(np.max(np.abs(o.cpu().numpy() - scores_np))) <= 2e-5


def test_config4_vqa_batch128_14x14x512():
    asm = Assembler(synth.vocab_file('vqa'))
    tokens = synth.histogram_tokens(asm, synth.VQA_LAYOUTS, 128, 13, seed=41)
    _real_size_case('vqa', 128, 14, 14, 512, 13, 3001, tokens, seed=940, group=3)


def test_config4_vqa_batch128_reference_depth_2048():
    """The reference's own VQA feature depth: res5c 2048 channels + 2 coordinate channels."""
    asm = Assembler(synth.vocab_file('vqa'))
    tokens = synth.histogram_tokens(asm, synth.VQA_LAYOUTS, 128, 13, seed=42)
    _real_size_case('vqa', 128, 14, 14, 2048, 13, 3001, tokens, seed=941)


def test_config5_stress_batch128_20x20x1024_depth16():
    asm = Assembler(synth.vocab_file('clevr'))
    base = synth.random_valid_tokens(asm, 16, 40, seed=21, ans_weight=0.08, min_depth=8,
                                     max_depth=16)
    tokens = np.ascontiguousarray(base[:, np.random.RandomState(5).randint(0, 16, size=128)])
    _real_size_case('clevr', 128, 20, 20, 1024, 40, 28, tokens, seed=942, group=2)
