"""NumPy restatement of the implicit-feedback scorers of spotlight/evaluation.py
(mrr_score :9-56, sequence_mrr_score :59-102, sequence_precision_recall_score :105-151,
precision_recall_score :154-220) in the form the device implementation computes them:
score rows, exclusions and targets -> average ranks and stable positions -> the metrics.

For a target t of a score row with s = row[t]:
  average rank    = 1 + #(row > s) + 0.5 * (#(row == s) - 1)     (rankdata of -row)
  stable position = #(row > s) + #(row == s and item < t)         (index in argsort(-row, stable))
and t is a hit at k iff its stable position is < k.
"""

import numpy as np

FLOAT_MAX = np.finfo(np.float32).max


def exclude(row, items):
    """The reference's ``predictions[items] = FLOAT_MAX`` on the negated row."""
    row = np.array(row, dtype=np.float32)
    row[np.asarray(items, dtype=np.int64)] = -FLOAT_MAX
    return row


def average_rank(row, t):
    s = row[t]
    return 1.0 + np.sum(row > s) + 0.5 * (np.sum(row == s) - 1)


def stable_position(row, t):
    s = row[t]
    return int(np.sum(row > s) + np.sum((row == s) & (np.arange(len(row)) < t)))


def mrr(rows, targets, excluded=None):
    """Mean over each row's targets of 1 / average rank; ``targets[r]`` and ``excluded[r]`` are
    item lists of row r."""
    out = []
    for r, row in enumerate(rows):
        if excluded is not None:
            row = exclude(row, excluded[r])
        out.append(np.mean([1.0 / average_rank(row, t) for t in targets[r]]))
    return np.array(out)


def precision_recall(rows, targets, ks, excluded=None, recall_denominator=None):
    """(precision, recall), each (n_rows, len(ks)): hits = distinct targets with stable
    position < k, precision = hits / min(k, n_items), recall = hits / len(set(targets))
    unless ``recall_denominator`` (the sequence scorer divides by k) is given."""
    ks = np.atleast_1d(ks)
    precision = np.zeros((len(rows), len(ks)))
    recall = np.zeros((len(rows), len(ks)))
    for r, row in enumerate(rows):
        if excluded is not None:
            row = exclude(row, excluded[r])
        uniq = np.unique(np.asarray(targets[r], dtype=np.int64))
        pos = np.array([stable_position(row, t) for t in uniq])
        for j, k in enumerate(ks):
            hits = float(np.sum(pos < k))
            precision[r, j] = hits / min(k, len(row))
            recall[r, j] = hits / (recall_denominator or len(uniq))
    return precision, recall
