"""Evaluation loop and result writers around the hot path (SURVEY.md §8f rows 2/4): what
exp_clevr/eval_clevr.py:93-163 does per split, with the module network on the GPU.

The reference predicts the layout tokens with its seq2seq and then runs the module network; with
the seq2seq off the hot path (BASELINE.json north_star) the tokens come from `layout_fn(batch)`,
by default the ground-truth layouts of the batch ("gt-layout eval", BASELINE config 2). Everything
after the tokens is the reference's loop: Assembler validity, scores, argmax, the three
accuracies, the accuracy text file and the one-answer-per-line prediction file in the exact
formats of eval_clevr.py:140-163 (VQA: the question-id JSON of exp_vqa/eval_vqa.py:163-165).
"""
from __future__ import annotations

import json

import numpy as np
import torch


def evaluate_split(pool, batches, assembler, answer_word_list, tst_image_set, save_file=None,
                   eval_output_file=None, layout_fn=None, word_vecs_fn=None, max_in_flight=8,
                   score_prior_fn=None):
    """pool: ExecutorPool (batches are queued `max_in_flight` at a time and evaluated with dynamic
    batching); batches: iterable of data_reader dicts (n2nmn_b200.data.DataReader.batches());
    word_vecs_fn(batch) -> [T,N,Dt] float32 tensor (the seq2seq's attended word vectors; the
    caller supplies them). score_prior_fn(batch) -> [N, num_choices] float32 logits (tensor or
    array) added to the module scores before the argmax: VQA's `scores_nmn + scores_qpn`
    (exp_vqa/eval_vqa.py, use_qpn=True); None = the module scores alone. Returns the dict of counts
    and accuracies that is also written out."""
    layout_fn = layout_fn or (lambda b: b['gt_layout_batch'])
    answer_correct = layout_correct = layout_valid = num_questions = 0
    output_answers = []
    pending = []

    def flush():
        nonlocal answer_correct, layout_valid, num_questions
        pool.end()
        torch.cuda.synchronize(pool.device)
        for batch, tokens, scores, valid, prior in pending:
            s = scores.cpu().numpy()
            if prior is not None:
                s = s + prior
            predictions = np.argmax(s, axis=1)
            if 'answer_label_batch' in batch:
                answer_correct += int(np.sum(predictions == batch['answer_label_batch']))
            layout_valid += int(np.sum(valid))
            num_questions += len(valid)
            output_answers.extend(answer_word_list[p] for p in predictions)
        pending.clear()
        pool.begin()

    pool.begin()
    for batch in batches:
        tokens = np.ascontiguousarray(layout_fn(batch), dtype=np.int32)
        if 'gt_layout_batch' in batch:      # eval_clevr.py:115-121
            gt = batch['gt_layout_batch']
            layout_correct += int(np.sum(np.all(np.logical_or(tokens == gt,
                                                              gt == assembler.EOS_idx), axis=0)))
        feat = batch.get('image_feat_pinned')
        feat = feat if feat is not None else torch.from_numpy(batch['image_feat_batch'])
        feat = feat.to(pool.device, non_blocking=True)
        wv = word_vecs_fn(batch).to(pool.device, non_blocking=True)
        scores, valid, _ = pool.submit(feat, wv, tokens)
        prior = None
        if score_prior_fn is not None:
            prior = score_prior_fn(batch)
            prior = (prior.detach().cpu().numpy() if isinstance(prior, torch.Tensor)
                     else np.asarray(prior)).astype(np.float32)
            if prior.shape != tuple(scores.shape):
                raise ValueError('score_prior_fn must return [N, num_choices] = %r, got %r'
                                 % (tuple(scores.shape), prior.shape))
        pending.append((batch, tokens, scores, valid, prior))
        if len(pending) >= max_in_flight:
            flush()
    flush()
    pool.end()
    res = dict(split=tst_image_set, num_questions=num_questions, answer_correct=answer_correct,
               layout_correct=layout_correct, layout_valid=layout_valid,
               answer_accuracy=answer_correct / max(num_questions, 1),
               layout_accuracy=layout_correct / max(num_questions, 1),
               layout_validity=layout_valid / max(num_questions, 1),
               output_answers=output_answers)
    if save_file:
        write_accuracy_file(save_file, res)
    if eval_output_file:
        write_prediction_file(eval_output_file, output_answers)
    return res


def merge_rank_results(results, tst_image_set=None):
    """One result from the per-rank results of a data-parallel evaluation (rank r evaluated
    questions r, r+world, … of the split: `DataReader(..., shuffle=False, rank=r, world=world)`):
    counts summed, accuracies recomputed, `output_answers` interleaved back into the split's
    order, so the prediction file is the one a single process writes."""
    world = len(results)
    n = sum(r['num_questions'] for r in results)
    answers = [None] * n
    for r, res in enumerate(results):
        if len(res['output_answers']) != len(range(r, n, world)):
            raise ValueError('rank %d evaluated %d questions, expected %d of %d dealt round-robin'
                             % (r, len(res['output_answers']), len(range(r, n, world)), n))
        answers[r::world] = res['output_answers']
    out = dict(split=tst_image_set or results[0]['split'], num_questions=n,
               output_answers=answers)
    for k in ('answer_correct', 'layout_correct', 'layout_valid'):
        out[k] = sum(r[k] for r in results)
    out['answer_accuracy'] = out['answer_correct'] / max(n, 1)
    out['layout_accuracy'] = out['layout_correct'] / max(n, 1)
    out['layout_validity'] = out['layout_valid'] / max(n, 1)
    return out


def gather_rank_results(res, group=None):
    """All ranks call this after `evaluate_split` on their shard (no collective on the data path:
    this is the optional gather of SURVEY.md §8e, a few KB per rank); every rank returns the
    merged result."""
    import torch.distributed as dist
    parts = [None] * dist.get_world_size(group)
    dist.all_gather_object(parts, res, group=group)
    return merge_rank_results(parts)


def accuracy_lines(res):
    """The four lines eval_clevr.py:140-151 prints and writes."""
    n = res['num_questions']
    return ['On split: %s' % res['split'],
            '\tanswer accuracy = %f (%d / %d)' % (res['answer_accuracy'], res['answer_correct'], n),
            '\tlayout accuracy = %f (%d / %d)' % (res['layout_accuracy'], res['layout_correct'], n),
            '\tlayout validity = %f (%d / %d)' % (res['layout_validity'], res['layout_valid'], n)]


def write_accuracy_file(save_file, res):
    with open(save_file, 'w') as f:
        for ln in accuracy_lines(res):
            print(ln, file=f)


def write_prediction_file(eval_output_file, output_answers):
    """One predicted answer word per line (eval_clevr.py:160-162), the format
    util/clevr_test/CLEVR_eval.py scores."""
    with open(eval_output_file, 'w') as f:
        f.writelines([a + '\n' for a in output_answers])


def write_vqa_prediction_file(eval_output_file, qids, output_answers):
    """[{"question_id": .., "answer": ..}] with the reference's separators
    (exp_vqa/eval_vqa.py:137-139,163-165)."""
    rows = [{'question_id': int(q), 'answer': a} for q, a in zip(qids, output_answers)]
    with open(eval_output_file, 'w') as f:
        json.dump(rows, f, separators=(',\n', ':\n'))
