"""BilinearNet with hashed (Bloom) embedding tables: one training step in float64 (oracle).

TEST INFRASTRUCTURE ONLY.  Restates what ``slb_mf_bloom_train_step`` (csrc/mf.cu) computes for
a ``BilinearNet`` whose user and / or item layer is a ``BloomEmbedding`` (spotlight/layers.py:
132-244), on top of ``oracle.murmur.bloom_rows``:

* each side is plain (``H = 0``: the id is the row) or hashed (``1 <= H <= 24``, seeds
  ``SEEDS[:H]``): the entity's vector is the sum of its H rows, the padding id ``pad`` maps to row
  0 for every hash, and row ``pad`` of the compressed table is frozen (no gradient, no decay;
  ``pad = -1``: none).  The biases stay indexed by the raw id (representations.py:58-59);
* pos = u . q + bu[u] + bi[i]; the losses and the adaptive-hinge pairing (the flat negative f
  scored with ``users[f // n]``, viewed ``(n, B)``, the first maximum credited) are
  ``oracle.mf``'s; the loss is divided by ``norm`` (default B);
* every (side, hashed user row, hashed item row) term of an interaction side with score gradient
  g adds g * (item row) to its user row and g * (user row) to its item row, per hash and not per
  distinct row, all from the tables as they were before the step; the id-space biases take
  dbu[u] += gp, dbu[u'] += gn, dbi[i] += gp, dbi[j] += gn;
* fused mode applies SGD / Adagrad row-wise with ``g + wd * w`` to touched entries only: a table
  row when a term with g != 0 names it and it is not frozen, an id-space bias when its id is the
  scored user or item of an interaction side with g != 0 (the MF rule: even when the bias's
  summed gradient is exactly 0).  Everything else stays bit-identical.

``mutate`` (a tuple of names) restates plausible kernel mistakes, so that
tests/test_mf_bloom_oracle_cpu.py can show the GPU tolerances catch each of them:

``pad_hashed``           the padding id hashed like any other id
``freeze_row0``          row 0 frozen instead of row ``pad``
``train_frozen``         the frozen row trained
``item_first_hash``      the item vector taken as its first hashed row only
``item_mean``            the item vector taken as the mean of its rows
``dup_row_once``         a row hit by two hashes of one id credited once
``adaptive_user_b``      the adaptive negative f = k B + b scored with ``users[b]``
``last_tie``             the last of tied maximal negatives credited
``stash_post_update``    item gradients taken from the updated user rows
``user_bias_no_gn``      the user-bias pair loses gn when the credited negative's user differs
``user_bias_zero_pair``  a user bias whose pairs sum to exactly 0 is not touched (no decay)
``decay_all_rows``       every row and bias the batch names is decayed, active or not
``adagrad_div_before_add`` Adagrad divides by the state before adding g^2
``bucket_merge``         distinct bias ids in one hash bucket merged into the smallest
``drop_last_pair``       each bias id's last non-zero (id, g) pair dropped
"""

import numpy as np

from oracle.explicit import apply_rowwise
from oracle.mf import loss_and_score_grads, negative_pairs
from oracle.murmur import bloom_rows

MUTATIONS = ('pad_hashed', 'freeze_row0', 'train_frozen', 'item_first_hash', 'item_mean', 'dup_row_once',
             'adaptive_user_b', 'last_tie', 'stash_post_update', 'user_bias_no_gn', 'user_bias_zero_pair',
             'decay_all_rows', 'adagrad_div_before_add', 'bucket_merge', 'drop_last_pair')

_NO_ID = -(1 << 62)          # a padding id no real id equals


def table_rows(ids, H, M, pad, mutate=()):
    """Rows of ``ids`` in a table of M rows: ``ids[..., None]`` when plain, else the H hashed rows."""
    ids = np.asarray(ids, dtype=np.int64)
    if H == 0:
        return ids[..., None]
    return bloom_rows(ids, H, M, _NO_ID if 'pad_hashed' in mutate else pad)


def frozen_row(H, pad, mutate=()):
    """The row of a table that receives neither gradient nor decay (-1 = none)."""
    if H == 0 or pad < 0 or 'train_frozen' in mutate:
        return -1
    return 0 if 'freeze_row0' in mutate else pad


def bias_buckets(B):
    """Hash-bucket count of the id-space bias update: the smallest power of two >= max(4096, 2 * 2B)."""
    nb = 4096
    while nb < 4 * B:
        nb <<= 1
    return nb


def _vectors(W, rows, item, mutate):
    if item and 'item_first_hash' in mutate:
        return W[rows[:, 0]]
    if item and 'item_mean' in mutate:
        return W[rows].mean(axis=1)
    return W[rows].sum(axis=1)


def _distinct(rows):
    """Mask of the hash columns of each id that name a row for the first time."""
    keep = np.ones(rows.shape, dtype=bool)
    for k in range(1, rows.shape[1]):
        keep[:, k] = (rows[:, :k] != rows[:, k:k + 1]).all(axis=1)
    return keep


def _row_grads(shape, rows, g, vec, mutate):
    """sum over terms: each hash column k of ``rows`` adds g * vec to row rows[:, k]."""
    out = np.zeros(shape)
    keep = _distinct(rows) if 'dup_row_once' in mutate else np.ones(rows.shape, dtype=bool)
    for k in range(rows.shape[1]):
        m = keep[:, k]
        np.add.at(out, rows[m, k], g[m, None] * vec[m])
    return out


def _bias_pairs(ids, g, n, B, mutate):
    """Sum the (id, g) pairs per id, restating the mistakes of the hash-bucket bias update."""
    ids, g = ids.copy(), g.copy()
    if 'drop_last_pair' in mutate:
        nz = np.flatnonzero(g != 0)
        last = {}
        for k in nz:
            last[ids[k]] = k
        counts = np.bincount(ids[nz], minlength=n)
        drop = [k for i, k in last.items() if counts[i] > 1]
        g[drop] = 0.0
    if 'bucket_merge' in mutate:
        nb = bias_buckets(B)
        used = np.unique(ids[g != 0])
        first = {}
        for i in used:
            first.setdefault(i & (nb - 1), i)
        ids = np.array([first.get(i & (nb - 1), i) if gk != 0 else i for i, gk in zip(ids, g)], dtype=np.int64)
    out = np.zeros(n)
    np.add.at(out, ids, g)
    return out


def step(params, users, items, negs, loss, Hu=0, Hi=0, pad_u=0, pad_i=0, n_neg=1, opt=None, lr=0.0,
         weight_decay=0.0, eps=1e-10, states=None, norm=None, mutate=()):
    """One float64 step.  ``params`` = [Wu, Wi, bu, bi] (Wu / Wi the plain or compressed tables,
    bu / bi of shape (num_users, 1) / (num_items, 1)).  ``negs`` has B * n_neg entries.

    ``opt=None`` is the dense mode: nothing is updated.  ``opt`` in ('sgd', 'adagrad') is the
    fused mode: ``params`` (and the Adagrad ``states``) are updated in place.  Returns
    dict(loss, pos, neg, gp, gn, dWu, dWi, dbu, dbi, touched=(Wu, Wi, bu, bi) masks)."""
    Wu, Wi, bu, bi = params
    users, items, negs = (np.asarray(x, dtype=np.int64).reshape(-1) for x in (users, items, negs))
    B = len(users)
    NU, NI = bu.shape[0], bi.shape[0]
    norm = B if norm is None else norm
    adaptive = loss == 'adaptive_hinge'
    n = n_neg if adaptive else 1
    Mu, Mi = Wu.shape[0], Wi.shape[0]
    W0u = Wu.copy()

    def user_rows(ids):
        return table_rows(ids, Hu, Mu, pad_u, mutate)

    def item_rows(ids):
        return table_rows(ids, Hi, Mi, pad_i, mutate)

    def score(u, i, Wu_):
        ru, ri = user_rows(u), item_rows(i)
        uv, iv = _vectors(Wu_, ru, False, mutate), _vectors(Wi, ri, True, mutate)
        return (uv * iv).sum(axis=1) + bu.reshape(-1)[u] + bi.reshape(-1)[i]

    pos = score(users, items, Wu)
    nu, ni = negative_pairs(users, negs, n, adaptive)
    if adaptive and 'adaptive_user_b' in mutate:
        nu = users[np.arange(B * n) % B]
    neg = score(nu, ni, Wu)
    if adaptive:
        negv = neg.reshape(n, B)
        if 'last_tie' in mutate:
            kstar = n - 1 - np.argmax(negv[::-1], axis=0)
        else:
            kstar = np.argmax(negv, axis=0)
        top = negv[kstar, np.arange(B)]
        lval, gp, gn = loss_and_score_grads('hinge', pos, top, None, np.float64)
        f = kstar * B + np.arange(B)
        u2, j = nu[f], ni[f]
    else:
        lval, gp, gn = loss_and_score_grads(loss, pos, neg, None, np.float64)
        u2, j = users, negs
    gp, gn = gp * (B / norm), gn * (B / norm)

    # the two sides of every interaction: (user ids, item ids, score gradient)
    sides = ((users, items, gp), (u2, j, gn))
    fu, fi = frozen_row(Hu, pad_u, mutate), frozen_row(Hi, pad_i, mutate)

    def user_grads(Wsrc):
        d = np.zeros(Wu.shape)
        for u, i, g in sides:
            d += _row_grads(Wu.shape, user_rows(u), g, _vectors(Wi, item_rows(i), True, mutate), mutate)
        if fu >= 0:
            d[fu] = 0.0
        return d

    def item_grads(Wsrc):
        d = np.zeros(Wi.shape)
        for u, i, g in sides:
            ri = item_rows(i)
            if 'item_first_hash' in mutate:
                ri = ri[:, :1]
            gi = g / ri.shape[1] if 'item_mean' in mutate else g
            d += _row_grads(Wi.shape, ri, gi, _vectors(Wsrc, user_rows(u), False, mutate), mutate)
        if fi >= 0:
            d[fi] = 0.0
        return d

    # an interaction whose negative is scored with its own user gives that user's bias one pair,
    # gp + gn (an exact 0 for bpr / hinge)
    same = u2 == users
    bu_ids = np.concatenate([users, u2])
    bu_g = np.concatenate([np.where(same, gp + gn, gp), np.where(same, 0.0, gn)])
    if 'user_bias_no_gn' in mutate:
        bu_g[B:] = np.where(u2 != users, 0.0, gn)
    bi_ids = np.concatenate([items, j])
    bi_g = np.concatenate([gp, gn])
    dbu = _bias_pairs(bu_ids, bu_g, NU, B, mutate).reshape(bu.shape)
    dbi = _bias_pairs(bi_ids, bi_g, NI, B, mutate).reshape(bi.shape)

    def touched_rows(M, rows_of, ids_g, frozen):
        t = np.zeros(M, dtype=bool)
        for ids, g in ids_g:
            act = np.ones(len(ids), dtype=bool) if 'decay_all_rows' in mutate else g != 0
            t[rows_of(ids[act]).reshape(-1)] = True
        if frozen >= 0:
            t[frozen] = False
        return t

    tWu = touched_rows(Mu, user_rows, ((users, gp), (u2, gn)), fu)
    tWi = touched_rows(Mi, item_rows, ((items, gp), (j, gn)), fi)
    tbu = touched_rows(NU, lambda x: x, ((users, gp), (u2, gn)), -1)
    tbi = touched_rows(NI, lambda x: x, ((items, gp), (j, gn)), -1)
    if 'user_bias_zero_pair' in mutate:
        # the merged pair (gp + gn of one user) is dropped when it is exactly 0
        same = u2 == users
        pair_ids = np.concatenate([users, u2[~same]])
        pair_g = np.concatenate([np.where(same, gp + gn, gp), gn[~same]])
        tbu = np.zeros(NU, dtype=bool)
        tbu[pair_ids[pair_g != 0]] = True

    out = dict(loss=float(lval) * B / norm, pos=pos, neg=neg, gp=gp, gn=gn, kstar_user=u2, kstar_item=j,
               touched=(tWu, tWi, tbu, tbi), dbu=dbu, dbi=dbi)
    if opt is None:
        out.update(dWu=user_grads(Wu), dWi=item_grads(Wu))
        return out
    wds = (weight_decay,) * 2
    st = (lambda a, b: None) if states is None else (lambda a, b: (states[a], states[b]))
    if 'stash_post_update' in mutate:
        dWu = user_grads(Wu)
        apply_rowwise((Wu, bu), (dWu, dbu), (tWu, tbu), opt, lr, wds, eps, st(0, 2), mutate)
        dWi = item_grads(Wu)
    else:
        dWi = item_grads(W0u)
        dWu = user_grads(Wu)
        apply_rowwise((Wu, bu), (dWu, dbu), (tWu, tbu), opt, lr, wds, eps, st(0, 2), mutate)
    apply_rowwise((Wi, bi), (dWi, dbi), (tWi, tbi), opt, lr, wds, eps, st(1, 3), mutate)
    out.update(dWu=dWu, dWi=dWi)
    return out


def fit(params, users, items, num_items, loss, batch_size, n_iter, random_state, opt, lr, Hu=0, Hi=0,
        pad_u=0, pad_i=0, n_neg=1, weight_decay=0.0, eps=1e-10, states=None, mutate=()):
    """The reference's fit loop (spotlight/factorization/implicit.py:184-252) on the hashed step,
    in float64: per epoch one ``shuffle(arange(n))``, then per minibatch one
    ``randint(0, num_items, len(batch) * n)`` and a fused ``step``.  Parameters and states are
    updated in place; returns the epoch losses (mean of the minibatch losses)."""
    n = len(users)
    nn = n_neg if loss == 'adaptive_hinge' else 1
    losses = []
    for _ in range(n_iter):
        order = np.arange(n)
        random_state.shuffle(order)
        u, i = np.asarray(users)[order].astype(np.int64), np.asarray(items)[order].astype(np.int64)
        ep = []
        for lo in range(0, n, batch_size):
            bu_, bi_ = u[lo:lo + batch_size], i[lo:lo + batch_size]
            negs = random_state.randint(0, num_items, len(bu_) * nn, dtype=np.int64)
            ep.append(step(params, bu_, bi_, negs, loss, Hu, Hi, pad_u, pad_i, nn, opt, lr, weight_decay, eps,
                           states, mutate=mutate)['loss'])
        losses.append(float(np.mean(ep)))
    return losses
