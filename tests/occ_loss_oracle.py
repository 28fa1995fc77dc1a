"""Two restatements of the occupancy loss of one supervised layer, written from the contract in include/gf_b200.h:

* ``oracle``: fp64 numpy, value and analytic gradient.  ``order`` (optional): per present class, the positions in V in
  the order to evaluate the Lovasz sum in; by default the stable descending order of its own fp64 errors.
* ``restatement``: the reference's lines (loss/occupancy_loss.py:102-149, loss/utils/lovasz_softmax.py:22-34,157-234)
  restated in PyTorch, in the dtype of ``pred``: boolean-mask gathers, a present test per class, ``torch.sort`` (unstable
  unless ``stable``) or a given ``order``.  Differentiable with autograd.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

PROB_LO, PROB_HI = float(np.float32(1e-6)), float(np.float32(1 - 1e-6))


def _pool(B, N, labels, occ_mask, empty_label):
    y = np.asarray(labels).reshape(-1).astype(np.int64)
    m = np.ones(B * N, bool) if occ_mask is None else np.asarray(occ_mask).reshape(-1).astype(bool)
    if empty_label is not None:
        m &= y != empty_label
    return np.nonzero(m)[0], y


def oracle(pred, labels, occ_mask, class_weights, *, use_softmax, lovasz_ignore, ignore_index=255, empty_label=None,
           ce_weight=1.0, lovasz_weight=1.0, order=None):
    """pred [B, C, N] (any float), labels [B, N], occ_mask [B, N] or None, class_weights [C].  Returns a dict: loss, ce,
    lovasz, grad [B, C, N] (fp64), V (flat voxel index b * N + n of every position in V), present (list of classes),
    order ({class: positions in V in evaluation order}), errors ({class: fp64 errors in V order})."""
    x = np.asarray(pred, np.float64)
    B, C, N = x.shape
    w = np.asarray(class_weights, np.float64)
    S, y = _pool(B, N, labels, occ_mask, empty_label)
    X = x.transpose(0, 2, 1).reshape(B * N, C)[S]
    Y = y[S]
    if use_softmax:
        mx = X.max(axis=1, keepdims=True)
        ex = np.exp(X - mx)
        se = ex.sum(axis=1, keepdims=True)
        P = ex / se
        lse = (mx + np.log(se))[:, 0]
    else:
        P = X
    g = np.zeros_like(X)
    # cross-entropy over the s in S with a class label other than ignore_index
    ok = (Y != ignore_index) & (Y >= 0) & (Y < C)
    rows = np.nonzero(ok)[0]
    yk = Y[ok]
    wy = w[yk]
    den = wy.sum()
    if use_softmax:
        nll = lse[ok] - X[rows, yk]
    else:
        q = np.clip(X[rows, yk].astype(np.float32), np.float32(PROB_LO), np.float32(PROB_HI)).astype(np.float64)
        nll = -np.log(q)
    with np.errstate(invalid="ignore", divide="ignore"):
        ce = (wy * nll).sum() / den
        if use_softmax:
            onehot = np.zeros((len(rows), C))
            onehot[np.arange(len(rows)), yk] = 1.0
            g[rows] += ce_weight * wy[:, None] * (P[rows] - onehot) / den
        else:
            xy = X[rows, yk]
            passes = (xy >= PROB_LO) & (xy <= PROB_HI)
            np.add.at(g, (rows, yk), np.where(passes, -ce_weight * wy / q / den, 0.0))
    # Lovasz-softmax over V = S without lovasz_ignore
    vrows = np.nonzero(Y != lovasz_ignore)[0]
    R, YV = P[vrows], Y[vrows]
    present = [c for c in range(C) if (YV == c).any()]
    gR = np.zeros_like(R)
    losses, orders, errors = [], {}, {}
    for c in present:
        fg = (YV == c).astype(np.float64)
        d = fg - R[:, c]
        e = np.abs(d)
        perm = np.asarray(order[c]) if order is not None else np.argsort(-e, kind="stable")
        fs = fg[perm]
        G = fs.sum()
        J = 1.0 - (G - np.cumsum(fs)) / (G + np.cumsum(1.0 - fs))
        delta = J.copy()
        delta[1:] -= J[:-1]
        losses.append(float((e[perm] * delta).sum()))
        gR[perm, c] = -np.sign(d[perm]) * delta
        orders[c], errors[c] = perm, e
    lov = float(np.mean(losses)) if losses else 0.0
    if present:
        gR *= lovasz_weight / len(present)
        if use_softmax:
            g[vrows] += R * (gR - (gR * R).sum(axis=1, keepdims=True))
        else:
            g[vrows] += gR
    full = np.zeros((B * N, C))
    full[S] = g
    return dict(loss=ce_weight * ce + lovasz_weight * lov, ce=ce, lovasz=lov,
                grad=full.reshape(B, N, C).transpose(0, 2, 1), V=S[vrows], present=present, order=orders,
                errors=errors)


def _lovasz_grad(gt_sorted):
    gts = gt_sorted.sum()
    intersection = gts - gt_sorted.cumsum(0)
    union = gts + (1 - gt_sorted).cumsum(0)
    jaccard = 1.0 - intersection / union
    if len(gt_sorted) > 1:
        jaccard[1:] = jaccard[1:] - jaccard[:-1]
    return jaccard


def restatement(pred, labels, occ_mask, class_weights, *, use_softmax, lovasz_ignore, ignore_index=255,
                empty_label=None, ce_weight=1.0, lovasz_weight=1.0, stable=False, order=None):
    """The reference's arithmetic in ``pred``'s dtype (pred [B, C, N] torch tensor, may require grad).  Returns
    (loss, ce, lovasz) tensors."""
    labels = labels.long()
    w = class_weights.to(pred.dtype)
    if empty_label is not None:
        empty_mask = labels != empty_label
        occ_mask = empty_mask if occ_mask is None else empty_mask & occ_mask.flatten(1)
    sem = pred
    if occ_mask is not None:
        occ_mask = occ_mask.flatten(1)
        labels = labels[occ_mask][None]
        sem = pred.transpose(1, 2)[occ_mask][None].transpose(1, 2)
    if use_softmax:
        ce = F.cross_entropy(sem, labels, weight=w, ignore_index=ignore_index)
    else:
        # the bounds as an fp32 tensor holds them (the same clamp in fp32; an fp64 restatement of the fp32 original)
        ce = F.nll_loss(torch.log(torch.clamp(sem, PROB_LO, PROB_HI)), labels, w, ignore_index=ignore_index)
    probas = (torch.softmax(sem, dim=1) if use_softmax else sem).transpose(1, 2).flatten(0, 1)
    lab = labels.flatten()
    valid = lab != lovasz_ignore
    vprobas = probas[valid.nonzero().squeeze(1)]
    vlabels = lab[valid]
    losses = []
    for c in range(probas.shape[1]):
        fg = (vlabels == c).to(pred.dtype)
        if fg.sum() == 0:
            continue
        errors = (fg - vprobas[:, c]).abs()
        if order is not None:
            perm = torch.as_tensor(np.asarray(order[c]), device=pred.device)
            errors_sorted = errors[perm]
        else:
            errors_sorted, perm = (torch.sort(errors, dim=0, descending=True, stable=True) if stable else
                                   torch.sort(errors, 0, descending=True))
        losses.append(torch.dot(errors_sorted, _lovasz_grad(fg[perm])))
    lov = torch.stack(losses).mean() if losses else torch.zeros((), dtype=pred.dtype, device=pred.device)
    return ce_weight * ce + lovasz_weight * lov, ce, lov
