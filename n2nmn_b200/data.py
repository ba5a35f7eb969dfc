"""Data path either side of the hot path (SURVEY.md §8f row 3): what produces the module network's
inputs on the host.

Reference counterparts
  * util/text_processing.py:3-35            -> tokenize / VocabDict
  * exp_clevr/data/get_ground_truth_layout.py:4-97 -> program_to_layout (CLEVR functional program
    -> Reverse-Polish expert layout)
  * util/clevr_train/data_reader.py:11-143  -> ClevrBatchLoader / DataReader (imdb .npy = pickled
    list of dicts, one feature .npy [1,H,W,D] per image, `prune_filter_module`, prefetch queue)

H100-first differences (behaviour of the produced batches is the reference's, checked against
fixtures made by running the reference files, tests/golden/make_golden_data.py):
  * feature grids are read straight into PINNED host buffers from a small ring, so a batch can be
    handed to ExecutorPool.submit_host (async H2D on the slot's stream) without a staging copy —
    the end-to-end path is PCIe-bound at ~50 GB/s per GPU (DESIGN.md §9), a pageable bounce would
    halve that;
  * several loader threads fill the prefetch queue (one thread reading 64 files per batch cannot
    feed a GPU that evaluates > 2000 batches per second);
  * batches() ends with a normal return at the end of a pass (the reference raises StopIteration
    inside a generator, a RuntimeError since Python 3.7).
"""
from __future__ import annotations

import queue
import re
import threading

import numpy as np

# ------------------------------------------------------------------------------ text processing
_SPLIT = re.compile(r'(\W+)')


def tokenize(sentence):
    """Lower-case, split on runs of non-word characters, keep the separators that are not blank
    (util/text_processing.py:3-7)."""
    parts = (p.strip() for p in _SPLIT.split(sentence.lower()))
    return [p for p in parts if p]


class VocabDict:
    """One word per line; index = line number; '<unk>' (if listed) catches unknown words
    (util/text_processing.py:15-35)."""

    def __init__(self, vocab_file):
        with open(vocab_file) as f:
            self.word_list = [ln.strip() for ln in f.readlines()]
        self.word2idx_dict = {w: i for i, w in enumerate(self.word_list)}
        self.num_vocab = len(self.word_list)
        self.UNK_idx = self.word2idx_dict.get('<unk>')

    def idx2word(self, n_w):
        return self.word_list[n_w]

    def word2idx(self, w):
        i = self.word2idx_dict.get(w, self.UNK_idx)
        if i is None:
            raise ValueError('word %s not in dictionary (while dictionary does not contain <unk>)'
                             % w)
        return i

    def tokenize_and_index(self, sentence):
        return [self.word2idx(w) for w in tokenize(sentence)]


# ------------------------------------------------------------------------------ expert layouts
_ATTR = ('color', 'material', 'shape', 'size')
FUNCTION2MODULE = dict(
    [('filter_' + a, '_Filter') for a in _ATTR] +
    [('same_' + a, '_FindSameProperty') for a in _ATTR] +
    [('equal_' + a, '_SameProperty') for a in _ATTR] +
    [('query_' + a, '_Describe') for a in _ATTR] +
    [('relate', '_Transform'), ('intersect', '_And'), ('union', '_Or'), ('count', '_Count'),
     ('exist', '_Exist'), ('equal_integer', '_EqualNum'), ('greater_than', '_MoreNum'),
     ('less_than', '_LessNum'), ('scene', '_Scene'), ('unique', None)])
_COMPARISONS = {'equal_integer', 'greater_than', 'less_than'} | {'equal_' + a for a in _ATTR}
_SPLICED = {'count'} | {'query_' + a for a in _ATTR}


def program_to_layout(program):
    """CLEVR functional program (list of {'function', 'inputs', ...}) -> list of module names in
    Reverse-Polish order (exp_clevr/data/get_ground_truth_layout.py:39-97, `linearize_program`):
    count / query_* feeding a comparison are spliced out (:46-66), the root is the one node nobody
    consumes (a stray `scene` root is ignored, :72-80), post-order traversal (:39-44), `unique`
    dropped, and `_Scene` directly followed by `_Filter` becomes `_Find` (:88-94). The input list is
    not modified (the reference edits it in place)."""
    prog = [None if f is None else dict(f, inputs=list(f['inputs'])) for f in program]
    for f in prog:
        if f is not None and f['function'] in _COMPARISONS:
            assert len(f['inputs']) == 2
            for slot in (0, 1):
                src = prog[f['inputs'][slot]]
                if src['function'] in _SPLICED:
                    assert len(src['inputs']) == 1
                    prog[f['inputs'][slot]] = None
                    f['inputs'][slot] = src['inputs'][0]
    consumed = set()
    for f in prog:
        if f is not None:
            consumed.update(f['inputs'])
    roots = [i for i, f in enumerate(prog) if f is not None and i not in consumed]
    if len(roots) != 1:
        roots = [i for i in roots if prog[i]['function'] != 'scene']
        assert len(roots) == 1
    order = []

    def visit(i):
        for j in prog[i]['inputs']:
            visit(j)
        order.append(prog[i]['function'])
    visit(roots[0])
    mods = [FUNCTION2MODULE[f] for f in order]
    out = list(mods)
    for i in range(1, len(mods)):
        if mods[i - 1] == '_Scene' and mods[i] == '_Filter':
            out[i - 1], out[i] = None, '_Find'
    return [m for m in out if m is not None]


def prune_filter_tokens(layout):
    """`prune_filter_module` of util/clevr_train/data_reader.py:65-71: a `_Filter` that directly
    follows a `_Find` or a `_Filter` is dropped (scanning from the end, so a run of filters
    collapses into its first element). Returns a new list."""
    toks = list(layout)
    for i in range(len(toks) - 1, 0, -1):
        if toks[i] == '_Filter' and toks[i - 1] in ('_Filter', '_Find'):
            toks[i] = None
    return [t for t in toks if t]


# ------------------------------------------------------------------------------ batches
def load_imdb(imdb_file):
    """imdb = .npy holding a pickled list of per-question dicts (data_reader.py:89-92; written by
    exp_clevr/data/build_clevr_imdb.py)."""
    if not imdb_file.endswith('.npy'):
        raise TypeError('unknown imdb format.')
    return np.load(imdb_file, allow_pickle=True)


class ClevrBatchLoader:
    """BatchLoaderClevr (util/clevr_train/data_reader.py:11-85). `load_one_batch(sample_ids)`
    returns the same dict (same keys, shapes, dtypes, values); image_feat_batch lives in a pinned
    buffer from a ring of `num_buffers` when torch + CUDA are available (`pinned=True`), so it
    stays valid until `num_buffers` further batches have been loaded.
    `data_params['feature_dtype'] = 'float16'` (not in the reference; default 'float32'): the batch
    carries the feature grids in half precision — per-image `.npy` files may be stored as float16
    or float32 (converted while the batch is filled) — for `ExecutorPool.submit_host`'s fp16 feed,
    which halves the PCIe bytes that bound the end-to-end rate (DESIGN.md §9)."""

    def __init__(self, imdb, data_params, pinned=False, num_buffers=12):
        self.imdb = imdb
        self.data_params = data_params
        self.vocab_dict = VocabDict(data_params['vocab_question_file'])
        self.T_encoder = data_params['T_encoder']
        first = self.imdb[0]
        self.load_answer = first.get('answer') is not None
        self.load_gt_layout = first.get('gt_layout_tokens') is not None
        if 'load_gt_layout' in data_params:
            self.load_gt_layout = data_params['load_gt_layout']
        self.answer_dict = VocabDict(data_params['vocab_answer_file'])
        if self.load_gt_layout:
            self.T_decoder = data_params['T_decoder']
            self.assembler = data_params['assembler']
            self.prune_filter_module = data_params.get('prune_filter_module', False)
        feats = np.load(first['feature_path'], mmap_mode='r')
        self.feat_H, self.feat_W, self.feat_D = feats.shape[1:]
        self._pinned = pinned
        self.feature_dtype = np.dtype(data_params.get('feature_dtype', 'float32'))
        if self.feature_dtype not in (np.dtype('float32'), np.dtype('float16')):
            raise ValueError('feature_dtype must be float32 or float16')
        self._ring, self._ring_pos, self._ring_n = {}, 0, max(1, num_buffers)
        self._lock = threading.Lock()

    def _feature_buffer(self, n):
        shape = (n, self.feat_H, self.feat_W, self.feat_D)
        if not self._pinned:
            return np.zeros(shape, self.feature_dtype), None
        import torch
        with self._lock:
            slot = self._ring_pos
            self._ring_pos = (slot + 1) % self._ring_n
        key = (slot, n)
        if key not in self._ring:
            dt = torch.float16 if self.feature_dtype == np.dtype('float16') else torch.float32
            self._ring[key] = torch.empty(shape, dtype=dt).pin_memory()
        t = self._ring[key]
        return t.numpy(), t

    def load_one_batch(self, sample_ids):
        n = len(sample_ids)
        input_seq = np.zeros((self.T_encoder, n), np.int32)
        seq_length = np.zeros(n, np.int32)
        feat, feat_tensor = self._feature_buffer(n)
        paths = [None] * n
        answers = np.zeros(n, np.int32) if self.load_answer else None
        layouts = np.zeros((self.T_decoder, n), np.int32) if self.load_gt_layout else None
        for j, sid in enumerate(sample_ids):
            info = self.imdb[sid]
            inds = [self.vocab_dict.word2idx(w) for w in info['question_tokens']]
            input_seq[:len(inds), j] = inds
            seq_length[j] = len(inds)
            feat[j:j + 1] = np.load(info['feature_path'], mmap_mode='r')
            paths[j] = info['image_path']
            if self.load_answer:
                answers[j] = self.answer_dict.word2idx(info['answer'])
            if self.load_gt_layout:
                toks = info['gt_layout_tokens']
                if self.prune_filter_module:
                    toks = prune_filter_tokens(toks)
                layouts[:, j] = self.assembler.module_list2tokens(toks, self.T_decoder)
        batch = dict(input_seq_batch=input_seq, seq_length_batch=seq_length,
                     image_feat_batch=feat, image_path_list=paths)
        if feat_tensor is not None:
            batch['image_feat_pinned'] = feat_tensor      # the same memory as a torch tensor
        if self.load_answer:
            batch['answer_label_batch'] = answers
        if self.load_gt_layout:
            batch['gt_layout_batch'] = layouts
        return batch


class DataReader:
    """DataReader (util/clevr_train/data_reader.py:87-143): `batches()` yields dicts from a bounded
    prefetch queue; order is the imdb order, or a fresh permutation per epoch with `shuffle`;
    the last batch of a pass may be short; `one_pass` ends the generator after one epoch.
    `rank` / `world` (not in the reference, which is single-device): this reader serves one rank of
    a data-parallel job — every epoch's order (the same on all ranks: a common `seed` is required
    with `shuffle`) is dealt round-robin, rank r taking questions r, r+world, … of it, so the ranks
    see disjoint questions and, up to one, equally many."""

    def __init__(self, imdb_file, shuffle=True, one_pass=False, prefetch_num=8, num_workers=4,
                 pinned=False, seed=None, rank=0, world=1, **kwargs):
        self.imdb = load_imdb(imdb_file) if isinstance(imdb_file, str) else imdb_file
        self.shuffle, self.one_pass = shuffle, one_pass
        self.data_params = kwargs
        self.batch_size = kwargs['batch_size']
        self.batch_loader = ClevrBatchLoader(self.imdb, kwargs, pinned=pinned,
                                             num_buffers=prefetch_num + num_workers + 2)
        if not 0 <= rank < world:
            raise ValueError('rank must be in [0, world)')
        if world > 1 and shuffle and seed is None:
            raise ValueError('a data-parallel reader needs a common seed (the ranks must draw the '
                             'same permutation to get disjoint shards)')
        self.rank, self.world = int(rank), int(world)
        self._rng = np.random.RandomState(seed)
        self._q = queue.Queue(maxsize=prefetch_num)
        self._workers = max(1, num_workers)
        self._thread = threading.Thread(target=self._produce, daemon=True)
        self._thread.start()

    def _epoch_order(self):
        n = len(self.imdb)
        order = self._rng.permutation(n) if self.shuffle else np.arange(n)
        return order[self.rank::self.world]

    def _produce(self):
        """Loader threads work on consecutive batches of the epoch; results enter the queue in
        batch order (a slot per in-flight batch)."""
        from concurrent.futures import ThreadPoolExecutor
        with ThreadPoolExecutor(self._workers) as pool:
            while True:
                order = self._epoch_order()
                chunks = [order[i:i + self.batch_size]
                          for i in range(0, len(order), self.batch_size)]
                pending = []
                for ch in chunks:
                    pending.append(pool.submit(self.batch_loader.load_one_batch, ch))
                    if len(pending) >= self._workers:
                        self._q.put(pending.pop(0).result())
                for fut in pending:
                    self._q.put(fut.result())
                if self.one_pass:
                    self._q.put(None)
                    return

    def batches(self):
        while True:
            batch = self._q.get()
            if batch is None:
                return
            yield batch
