"""Federated evaluation (DESIGN.md §13): every client scores its deployed model on its own test scans, and only the
CKKS-summed counts leave it.

One client's count vector holds, for C classes and ``nbins`` score bins, V = C·C + C·C·nbins + 1 values:

* ``conf[t][pred]`` at ``t·C + pred``: the confusion matrix (pred = arg-max of the logits, lowest index on ties);
* ``hist[t][c][b]`` at ``C·C + (t·C + c)·nbins + b``: how many scans of true class t had p_c in bin b, with
  p = softmax(logits) in fp32 and b = min(nbins - 1, floor(p_c · nbins)) in fp32;
* the cross-entropy sum at ``V - 1``.

The vectors are summed over the federation; ``metrics_from_counts`` turns the sum into accuracy, weighted precision /
recall / F1 (exactly ``classification_metrics`` of the pooled predictions), the mean loss, and the per-class
one-vs-rest binned ROC AUC.
"""
from __future__ import annotations

from fractions import Fraction
from typing import Dict, List, Optional, Sequence

import torch
import torch.nn.functional as F

MAX_CLASSES = 32          # score_stats keeps one row's logits in registers


def count_len(num_classes: int, nbins: int) -> int:
    """V: the length of one client's count vector."""
    return num_classes * num_classes * (nbins + 1) + 1


def check_fedeval_options(cfg, num_classes: Optional[int] = None, capacity: Optional[int] = None,
                          test_sets: Optional[Sequence] = None, train_classes: Optional[Dict[str, int]] = None) -> None:
    """Reject federated-evaluation settings the round cannot honour (they arrive from flags and environment variables).
    ``capacity``: values the transport's ciphertext buffer holds; ``test_sets``: the clients' test datasets;
    ``train_classes``: the training folder's ``class_indices``, when it has them."""
    every, nb = cfg.fed_eval_every, cfg.fed_eval_bins
    if not (isinstance(every, int) and every >= 0):
        raise ValueError(f"fed_eval_every must be an integer >= 0 (0 = on request only), got {every!r}")
    if not (isinstance(nb, int) and 2 <= nb <= 1024):
        raise ValueError(f"fed_eval_bins must be an integer in 2..1024, got {nb!r}")
    if num_classes is None:
        return
    if num_classes > MAX_CLASSES:
        raise ValueError(f"federated evaluation handles up to {MAX_CLASSES} classes, the model has {num_classes}")
    if cfg.compat_sequential_clients:
        raise ValueError("federated evaluation scores the global model of a round: it does not combine with "
                         "compat_sequential_clients")
    v = count_len(num_classes, nb)
    if capacity is not None and v > capacity:
        raise ValueError(f"the count vector of {num_classes} classes x {nb} bins ({v} values) does not fit the "
                         f"{capacity} values of the ciphertext buffer: lower fed_eval_bins")
    for i, ds in enumerate(test_sets or ()):
        if ds is None or len(ds) == 0:
            continue
        if int(ds.labels.max()) >= num_classes or int(ds.labels.min()) < 0:
            raise ValueError(f"test set {i}: labels must be in 0..{num_classes - 1}, got "
                             f"{int(ds.labels.min())}..{int(ds.labels.max())}")
        ci = getattr(ds, "class_indices", None)
        if train_classes is not None and ci is not None and ci != train_classes:
            raise ValueError(f"test set {i}: class names {sorted(ci)} differ from the training folder's "
                             f"{sorted(train_classes)}")


def score_counts_torch(logits: torch.Tensor, labels: torch.Tensor, nbins: int,
                       probs: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The count vector (float64 [V], on the logits' device) of a batch, in PyTorch: the reference the kernels are
    tested against and the path of the autograd backends. ``probs``: the fp32 softmax to bin (default: computed here
    from ``logits``)."""
    logits = logits.float()
    B, C = logits.shape
    labels = labels.long().to(logits.device)
    p = torch.softmax(logits, dim=1) if probs is None else probs.float()
    pred = logits.argmax(1)
    bins = (p * float(nbins)).floor().clamp(0, nbins - 1).long()
    conf = torch.bincount(labels * C + pred, minlength=C * C)
    cls = torch.arange(C, device=logits.device)
    hist = torch.bincount(((labels[:, None] * C + cls) * nbins + bins).flatten(), minlength=C * C * nbins)
    loss = F.cross_entropy(logits.double(), labels, reduction="sum") if B else torch.zeros((), dtype=torch.float64)
    return torch.cat([conf.double(), hist.double(), loss.reshape(1).to(conf.device)])


def binned_auc(pos: Sequence[int], neg: Sequence[int]) -> Optional[float]:
    """One-vs-rest ROC AUC from the binned scores of the positives and the negatives: the Mann–Whitney statistic, a
    positive above a negative counts 1 and a tie inside a bin ½. None without positives or without negatives."""
    P, N = sum(pos), sum(neg)
    if P == 0 or N == 0:
        return None
    below, num2 = 0, 0
    for p, n in zip(pos, neg):
        num2 += 2 * p * below + p * n
        below += n
    return float(Fraction(num2, 2 * P * N))


def metrics_from_confusion(conf: Sequence[Sequence[int]], n: int) -> Dict[str, float]:
    """Support-weighted precision / recall / F1 (zero where undefined, sklearn's ``average='weighted',
    zero_division=0``) and accuracy of confusion matrix ``conf[true][pred]`` over ``n`` >= 1 samples."""
    C = len(conf)
    p_w = r_w = f_w = 0.0
    for c in range(C):
        tp = float(conf[c][c])
        fp = float(sum(conf[t][c] for t in range(C)) - conf[c][c])
        fn = float(sum(conf[c]) - conf[c][c])
        prec = tp / (tp + fp) if tp + fp > 0 else 0.0
        rec = tp / (tp + fn) if tp + fn > 0 else 0.0
        f1 = 2 * prec * rec / (prec + rec) if prec + rec > 0 else 0.0
        w = (tp + fn) / n
        p_w, r_w, f_w = p_w + w * prec, r_w + w * rec, f_w + w * f1
    return {"precision": p_w, "recall": r_w, "f1": f_w, "accuracy": float(sum(conf[c][c] for c in range(C))) / n}


def metrics_from_counts(counts, num_classes: int, nbins: int) -> Dict:
    """The federation's result from a summed count vector (integer counts, then the loss sum): n, accuracy, weighted
    precision / recall / F1, the mean loss, per-class binned ROC AUC (None where undefined), their mean over the
    defined ones, and the confusion matrix."""
    vals = counts.tolist() if isinstance(counts, torch.Tensor) else list(counts)
    C = num_classes
    if len(vals) != count_len(C, nbins):
        raise ValueError(f"count vector of {len(vals)} values, expected {count_len(C, nbins)} for {C} classes and "
                         f"{nbins} bins")
    ints = [int(round(v)) for v in vals[:-1]]
    conf = [ints[t * C:(t + 1) * C] for t in range(C)]
    hist = ints[C * C:]
    n = sum(sum(r) for r in conf)
    out = {"n": n, **metrics_from_confusion(conf, max(1, n)), "loss": vals[-1] / n if n else None}

    def h(t, c):
        return hist[(t * C + c) * nbins:(t * C + c + 1) * nbins]

    aucs: List[Optional[float]] = []
    for c in range(C):
        neg = [sum(col) for col in zip(*[h(t, c) for t in range(C) if t != c])] if C > 1 else [0] * nbins
        aucs.append(binned_auc(h(c, c), neg))
    defined = [a for a in aucs if a is not None]
    out.update({"auc": aucs, "macro_auc": sum(defined) / len(defined) if defined else None, "confusion": conf})
    return out
