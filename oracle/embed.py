"""The generic route's kernels, restated in NumPy (oracle).

TEST INFRASTRUCTURE ONLY.  Restates what the kernels behind ``ops.embedding``,
``ops.embedding_backward``, ``ops.bloom_rows`` (csrc/embed.cu), ``ops.mf_scores`` /
``ops.mf_scores_backward`` (csrc/mf.cu) and ``ops.pairwise_loss`` / ``ops.rating_loss``
(csrc/loss.cu) compute:

* lookup: plain (``H = 0``: the id is the row) or Bloom (the sum of the H rows of
  ``oracle.murmur.bloom_rows``, the padding id ``pad`` mapping to row 0 for every hash);
* backward: the dense table gradient.  Term t = b * fan + k (fan = max(H, 1)) names row
  ``rows[b, k]`` and adds ``dout[t // fan]``; the frozen row (``pad``, the padding row of a plain
  table and the frozen row of a Bloom one; -1 = none) gets no gradient;
* scores: <Wu[u], Wi[i]> + bu[u] + bi[i], with one user broadcast over all items when
  ``users`` has one entry and ``items`` more; the backward scatters g * Wi[i], g * Wu[u], g, g;
* losses: the pairwise losses of ``oracle.mf.loss_and_score_grads`` and the rating losses of
  ``oracle.explicit.loss_and_score_grad`` (the standalone poisson loss takes the exponentiated
  prediction p, so its gradient is the score gradient divided by p).

The lookup and its backward come in two forms: float64, and *ordered float32*, the exact order
of the kernels' float32 additions (the forward starts at 0.f and adds the hashed rows in hash
order; the backward adds each row's ``dout`` rows in ascending term order), so that a kernel
result can be compared bit for bit.  The library is built without fast-math, so those adds
round to nearest; cases draw |x| in [2^-4, 2^4], so no partial sum is subnormal.

``mutate`` (a tuple of names) restates plausible kernel mistakes, so that
tests/test_embed_oracle_cpu.py can show the GPU checks catch each of them:

``pad_hashed``        the padding id hashed like any other id
``freeze_row0``       row 0 frozen instead of row ``pad``
``train_frozen``      the frozen row trained
``dup_row_once``      a row hit by two hashes of one id credited once
``fan_mod``           the backward's source row taken as t % n instead of t // fan
``tail_zero``         the elements of the last partial lane chunk left at 0
``long_drop_last``    a segment longer than ``seg_sort_cap(G)`` loses its largest term
``order_desc``        the backward adds in descending term order (only the bit check sees it)
``bcast_user_once``   a broadcast user credited with the first item's term only
``last_tie``          the adaptive hinge credits the last tied maximum
``mask_mean_over_n``  the masked mean divided by n instead of the mask's sum
"""

import numpy as np

from oracle import explicit as oe
from oracle.mf import loss_and_score_grads
from oracle.murmur import bloom_rows

MUTATIONS = ('pad_hashed', 'freeze_row0', 'train_frozen', 'dup_row_once', 'fan_mod', 'tail_zero',
             'long_drop_last', 'order_desc', 'bcast_user_once', 'last_tie', 'mask_mean_over_n')

_NO_ID = -(1 << 62)          # a padding id no real id equals


def pow2_lanes(D):
    """Lanes per row of emb_fwd_kernel / emb_bwd_kernel: a power of two, at most 32, covering
    D / 4 float4 pieces (D % 4 == 0) or D floats."""
    n = D // 4 if D % 4 == 0 else D
    p = 1
    while p < n and p < 32:
        p <<= 1
    return p


def vec4(D):
    return D % 4 == 0


def seg_sort_cap(G):
    """Longest member list seg_visit_sorted sorts in shared memory (segindex.cuh); longer lists
    take the min-selection path."""
    return 128 if G >= 8 else (64 if G >= 4 else 16 * G)


def frozen_row(pad, mutate=()):
    if pad < 0 or 'train_frozen' in mutate:
        return -1
    return 0 if 'freeze_row0' in mutate else pad


def term_rows(ids, H, M, pad, mutate=()):
    """(n, max(H, 1)) rows of the terms of ``ids`` in a table of M rows."""
    ids = np.asarray(ids, dtype=np.int64).reshape(-1)
    if H == 0:
        return ids[:, None]
    return bloom_rows(ids, H, M, _NO_ID if 'pad_hashed' in mutate else pad)


def _first_hit(rows):
    """Mask of the hash columns of each id that name a row for the first time."""
    keep = np.ones(rows.shape, dtype=bool)
    for k in range(1, rows.shape[1]):
        keep[:, k] = (rows[:, :k] != rows[:, k:k + 1]).all(axis=1)
    return keep


def _tail(out, D, mutate):
    if 'tail_zero' in mutate:
        chunk = pow2_lanes(D) * (4 if vec4(D) else 1)
        out[..., (D // chunk) * chunk:] = 0
    return out


def lookup(W, ids, H, pad, ordered=False, mutate=()):
    """out[b] = sum_k W[rows[b, k]]: float64, or (``ordered``) float32 added in hash order."""
    M, D = W.shape
    rows = term_rows(ids, H, M, pad, mutate)
    keep = _first_hit(rows) if 'dup_row_once' in mutate else np.ones(rows.shape, dtype=bool)
    dt = np.float32 if ordered else np.float64
    Wd = W.astype(dt)
    out = np.zeros((rows.shape[0], D), dtype=dt)
    for k in range(rows.shape[1]):
        out = out + np.where(keep[:, k:k + 1], Wd[rows[:, k]], dt(0))
    return _tail(out, D, mutate)


def lookup_backward(dout, ids, H, M, pad, ordered=False, mutate=()):
    """Dense (M, D) gradient of the lookup: float64, or (``ordered``) float32 with each row's
    terms added in ascending term order (the segmented scatter's order)."""
    dout = np.asarray(dout)
    n, D = dout.shape
    rows = term_rows(ids, H, M, pad, mutate)
    fan = rows.shape[1]
    keep = _first_hit(rows) if 'dup_row_once' in mutate else np.ones(rows.shape, dtype=bool)
    r = rows.reshape(-1)
    t = np.arange(r.size, dtype=np.int64)
    src = t % max(n, 1) if 'fan_mod' in mutate else t // fan
    fr = frozen_row(pad, mutate)
    live = keep.reshape(-1) & (r != fr)
    r, t, src = r[live], t[live], src[live]
    # segments: terms sorted stably by (row, t), or (row, -t) for order_desc
    order = np.lexsort((-t if 'order_desc' in mutate else t, r))
    r, t, src = r[order], t[order], src[order]
    starts = np.flatnonzero(np.r_[True, r[1:] != r[:-1]]) if r.size else np.zeros(0, dtype=np.int64)
    lens = np.diff(np.r_[starts, r.size])
    pos = np.arange(r.size) - np.repeat(starts, lens)
    if 'long_drop_last' in mutate:
        cap = seg_sort_cap(pow2_lanes(D))
        seglen = np.repeat(lens, lens)
        # the largest term of a long segment: the last in ascending order
        drop = (seglen > cap) & (t == np.repeat(np.maximum.reduceat(t, starts) if r.size else t, lens))
        r, src, pos = r[~drop], src[~drop], pos[~drop]
    dt = np.float32 if ordered else np.float64
    dW = np.zeros((M, D), dtype=dt)
    if not ordered:
        np.add.at(dW, r, dout[src].astype(np.float64))
        return _tail(dW, D, mutate)
    # one position at a time across all segments: within one position a row appears once
    by_pos = np.argsort(pos, kind='stable')
    bounds = np.searchsorted(pos[by_pos], np.arange(pos.max() + 2 if pos.size else 1))
    dsrc = dout.astype(np.float32)
    for p in range(len(bounds) - 1):
        sel = by_pos[bounds[p]:bounds[p + 1]]
        dW[r[sel]] = dW[r[sel]] + dsrc[src[sel]]
    return _tail(dW, D, mutate)


def term_counts(ids, H, M, pad):
    """Members per row as the backward's segment index counts them (frozen row excluded)."""
    r = term_rows(ids, H, M, pad).reshape(-1)
    c = np.bincount(r, minlength=M)
    if pad >= 0:
        c[pad] = 0
    return c


# ------------------------------------------------------------------ BilinearNet scores

def _score_users(users, n):
    users = np.asarray(users, dtype=np.int64).reshape(-1)
    return np.full(n, users[0], dtype=np.int64) if users.size == 1 and n != 1 else users


def scores(Wu, Wi, bu, bi, users, items):
    items = np.asarray(items, dtype=np.int64).reshape(-1)
    u = _score_users(users, items.size)
    Wu, Wi = Wu.astype(np.float64), Wi.astype(np.float64)
    return (Wu[u] * Wi[items]).sum(axis=1) + bu.astype(np.float64).reshape(-1)[u] + \
        bi.astype(np.float64).reshape(-1)[items]


def scores_backward(g, Wu, Wi, users, items, mutate=()):
    """(dWu, dWi, dbu, dbi) in float64; the biases shaped (rows, 1)."""
    items = np.asarray(items, dtype=np.int64).reshape(-1)
    u = _score_users(users, items.size)
    g = np.asarray(g, dtype=np.float64).copy()
    Wu, Wi = Wu.astype(np.float64), Wi.astype(np.float64)
    dWu, dWi = np.zeros(Wu.shape), np.zeros(Wi.shape)
    dbu, dbi = np.zeros(Wu.shape[0]), np.zeros(Wi.shape[0])
    gu = g
    if 'bcast_user_once' in mutate and np.asarray(users).size == 1 and items.size > 1:
        gu = np.where(np.arange(g.size) == 0, g, 0.0)
    np.add.at(dWu, u, gu[:, None] * Wi[items])
    np.add.at(dbu, u, gu)
    np.add.at(dWi, items, g[:, None] * Wu[u])
    np.add.at(dbi, items, g)
    return dWu, dWi, dbu.reshape(-1, 1), dbi.reshape(-1, 1)


# ------------------------------------------------------------------ standalone losses

def pairwise_loss(kind, pos, neg, mask=None, mutate=()):
    """(loss, d loss / d pos, d loss / d neg) in float64; ``neg`` is (n_neg, n) for the adaptive
    hinge."""
    pos = np.asarray(pos, dtype=np.float64)
    neg = np.asarray(neg, dtype=np.float64)
    m = None if mask is None else np.asarray(mask).astype(np.float64)
    if 'mask_mean_over_n' in mutate and m is not None:
        f = m.sum() / pos.size                  # sum(loss * m) / n = (masked mean) * sum(m) / n
        l, gp, gn = loss_and_score_grads(kind, pos, neg, m, np.float64)
        return float(l) * f, gp * f, gn * f
    if kind == 'adaptive_hinge' and 'last_tie' in mutate:
        n_neg = neg.shape[0]
        kstar = n_neg - 1 - np.argmax(neg[::-1], axis=0)
        top = neg[kstar, np.arange(pos.size)]
        l, gp, gtop = loss_and_score_grads('hinge', pos, top, m, np.float64)
        gn = np.zeros_like(neg)
        gn[kstar, np.arange(pos.size)] = gtop
        return float(l), gp, gn
    l, gp, gn = loss_and_score_grads(kind, pos, neg, m, np.float64)
    return float(l), gp, gn


def rating_loss(kind, pred, ratings):
    """(mean loss, d loss / d pred) in float64 of the standalone rating loss; poisson's ``pred`` is
    the exponentiated prediction."""
    pred = np.asarray(pred, dtype=np.float64)
    if kind == 'poisson':
        l, g = oe.loss_and_score_grad(kind, np.log(pred), ratings)
        return float(l), g / pred
    l, g = oe.loss_and_score_grad(kind, pred, ratings)
    return float(l), g
