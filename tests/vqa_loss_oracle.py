"""CPU oracle of the VQA training loss (exp_vqa/train_vqa_rl_gt_layout.py:101-116,
train_vqa_gt_layout.py:101-121) on top of the torch-autograd module oracle
(oracle/nmn_oracle_torch.py): scores = scores_nmn + scores_qpn with the question-prior logits
given, and the softmax cross-entropy on every row (an invalid layout's module scores are zeros,
so its loss is CE(prior, label)). With neither option it is nmn_oracle_torch.loss_and_grads."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle.nmn_oracle_torch import forward_scores


def loss_and_grads(m, expr_list, validity, labels, invalid_expr_loss=0.5, weight_decay=0.0,
                   score_prior=None, ce_every_row=False):
    """(scores, per_sample, avg, {variable: grad}, d word_vecs[, d score_prior]): the returned
    scores include the prior; the sixth element is present when a prior is given."""
    scores = forward_scores(m, expr_list)
    prior = None
    if score_prior is not None:
        prior = torch.as_tensor(np.asarray(score_prior), dtype=scores.dtype).clone()
        prior.requires_grad_(True)
        scores = scores + prior
    ce = F.cross_entropy(scores, torch.as_tensor(labels, dtype=torch.long), reduction='none')
    if ce_every_row:
        per_sample = ce
    else:
        valid = torch.as_tensor(np.asarray(validity), dtype=torch.bool)
        per_sample = torch.where(valid, ce, torch.full_like(ce, invalid_expr_loss))
    avg = per_sample.mean()
    l2 = sum(0.5 * (w * w).sum() for n, w in m.w.items() if n.endswith('/weights'))
    total = avg + weight_decay * l2
    names = list(m.w)
    wrt = [m.w[n] for n in names] + [m.word_vecs] + ([prior] if prior is not None else [])
    grads = torch.autograd.grad(total, wrt, allow_unused=True)
    nw = len(names)
    g = {n: (gi if gi is not None else torch.zeros_like(m.w[n])).detach().numpy()
         for n, gi in zip(names, grads[:nw])}
    g_wv = grads[nw].detach().numpy() if grads[nw] is not None else \
        np.zeros(tuple(m.word_vecs.shape), np.float32)
    out = (scores.detach().numpy(), per_sample.detach().numpy(), float(avg.detach()), g, g_wv)
    if prior is not None:
        out = out + (grads[nw + 1].detach().numpy(),)
    return out
