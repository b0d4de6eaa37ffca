"""BilinearNet + implicit losses, closed-form forward/backward (oracle).

TEST INFRASTRUCTURE ONLY.  Restates, in NumPy:

* ``BilinearNet.forward``      spotlight/factorization/representations.py:80-91
* ``pointwise/bpr/hinge/adaptive_hinge`` losses   spotlight/losses.py:40-50,
  82-90, 115-124, 164-166 (masked mean: ``sum(loss*mask)/mask.sum()``)
* the autograd result of ``loss.backward()`` in
  spotlight/factorization/implicit.py:229-243, including the adaptive-hinge
  user/negative misalignment of ``_get_multiple_negative_predictions``
  (implicit.py:266-275: users are repeated ``[u0]*n,[u1]*n,...`` but the flat
  prediction vector is *viewed* as ``(n, B)``).

``dtype`` selects the arithmetic (float32 mimics the reference, float64 gives
a tighter arbiter).  tests/test_oracle_mf.py pins it against golden vectors
produced by the live reference (tests/golden/make_golden.py).

``fused_step`` / ``fit`` restate, in float64, the planned step with its fused row-wise SGD /
Adagrad (csrc/mf_v2.cuh) and the reference's fit loop around it.  ``mutate`` (a tuple of
names, empty by default) restates plausible kernel mistakes, so that
tests/test_mf_planned_oracle_cpu.py can show that the GPU tolerances catch each of them:

``stash_post_update``     the item side reads the user rows after the user-side update
``neg_to_pos_row``        the negative's item term credited to the positive's row
``user_bias_no_gn``       the user-bias gradient without the negative's term
``hinge_strict``          hinge active at z > 0 instead of z >= 0
``decay_all_rows``        weight decay on every row of the batch, not only rows with a non-zero term
``no_decay_user_rows``    weight decay skipped on the user embedding rows
``no_decay_biases``       weight decay skipped on both bias tables
``adagrad_div_before_add`` Adagrad divides by the state before adding g^2
``item_first4``           item lists of 5..cap terms sum only their first 4 terms
``hot_drop_last``         the last member of each hot list (longer than ``cap``) dropped
``local_norm``            the gradient normalised by the local batch instead of ``norm``
"""

import numpy as np

from oracle.explicit import apply_rowwise

LOSSES = ('pointwise', 'bpr', 'hinge', 'adaptive_hinge')


def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def bilinear_scores(Wu, Wi, bu, bi, users, items, dtype=np.float32):
    """representations.py:80-91: (U[u]*Q[i]).sum(1) + bu[u] + bi[i]."""
    u = Wu[users].astype(dtype)
    q = Wi[items].astype(dtype)
    dot = (u * q).sum(axis=-1, dtype=dtype)
    return dot + bu[users].reshape(dot.shape).astype(dtype) + bi[items].reshape(dot.shape).astype(dtype)


def loss_and_score_grads(kind, pos, neg, mask=None, dtype=np.float32):
    """Loss value and d loss / d pos, d loss / d neg.

    ``neg`` has the shape of ``pos`` except for adaptive_hinge, where it is
    ``(n,) + pos.shape`` and the gradient is routed to the first arg-max over
    axis 0 (torch.max CPU tie-break; losses.py:164).
    """
    pos = pos.astype(dtype)
    neg = neg.astype(dtype)
    if mask is None:
        w = np.full(pos.shape, 1.0 / pos.size, dtype=dtype)
    else:
        m = mask.astype(dtype)
        w = m / m.sum(dtype=dtype)

    if kind == 'adaptive_hinge':
        kstar = np.argmax(neg, axis=0)
        top = np.take_along_axis(neg, kstar[None], axis=0)[0]
        l, gp, gtop = loss_and_score_grads('hinge', pos, top, mask, dtype)
        gn = np.zeros_like(neg)
        np.put_along_axis(gn, kstar[None], gtop[None], axis=0)
        return l, gp, gn

    if kind == 'bpr':
        s = _sigmoid(pos - neg)
        per = 1.0 - s
        gp = -s * (1.0 - s) * w
        gn = -gp
    elif kind == 'hinge':
        z = neg - pos + 1.0
        per = np.maximum(z, 0.0)
        act = (z >= 0.0).astype(dtype)     # clamp backward passes at 0
        gp = -act * w
        gn = act * w
    elif kind == 'pointwise':
        sp = _sigmoid(pos)
        sn = _sigmoid(neg)
        per = (1.0 - sp) + sn
        gp = -sp * (1.0 - sp) * w
        gn = sn * (1.0 - sn) * w
    else:
        raise ValueError(kind)
    if mask is None:
        loss = per.mean(dtype=dtype)
    else:
        loss = (per * m).sum(dtype=dtype) / m.sum(dtype=dtype)
    return dtype(loss), gp.astype(dtype), gn.astype(dtype)


def negative_pairs(users, negs, n_neg, adaptive):
    """(user, item) id pairs the negative predictions are scored with.

    Non-adaptive: pair b = (users[b], negs[b]).  Adaptive (implicit.py:266-275):
    flat index f in [0, B*n) pairs users[f // n] with negs[f]; the (n, B) view
    puts f = k*B + b at [k, b].
    """
    if not adaptive:
        return users, negs
    f = np.arange(users.shape[0] * n_neg)
    return users[f // n_neg], negs.reshape(-1)


def mf_step(Wu, Wi, bu, bi, users, items, negs, loss='bpr', n_neg=1,
            dtype=np.float32):
    """One minibatch: predictions, loss and dense parameter gradients.

    ``negs``: int64 ``[B]`` (or ``[B*n]`` flat for adaptive_hinge, exactly what
    ``sample_items(num_items, B*n)`` returned).
    Returns a dict with pos, neg, loss, dWu, dWi, dbu, dbi (dense, like the
    reference's ``.grad`` with sparse=False).
    """
    adaptive = loss == 'adaptive_hinge'
    B = users.shape[0]
    nu, ni = negative_pairs(users, negs, n_neg, adaptive)
    pos = bilinear_scores(Wu, Wi, bu, bi, users, items, dtype)
    negp = bilinear_scores(Wu, Wi, bu, bi, nu, ni, dtype)
    if adaptive:
        negp = negp.reshape(n_neg, B)
    l, gp, gn = loss_and_score_grads(loss, pos, negp, None, dtype)
    gn_flat = gn.reshape(-1)

    acc = np.float64 if dtype == np.float64 else np.float32
    dWu = np.zeros(Wu.shape, dtype=acc)
    dWi = np.zeros(Wi.shape, dtype=acc)
    dbu = np.zeros(bu.shape, dtype=acc)
    dbi = np.zeros(bi.shape, dtype=acc)
    # index_add in batch order == np.add.at
    np.add.at(dWu, users, gp[:, None] * Wi[items].astype(dtype))
    np.add.at(dWi, items, gp[:, None] * Wu[users].astype(dtype))
    np.add.at(dWu, nu, gn_flat[:, None] * Wi[ni].astype(dtype))
    np.add.at(dWi, ni, gn_flat[:, None] * Wu[nu].astype(dtype))
    np.add.at(dbu.reshape(-1), users, gp)
    np.add.at(dbi.reshape(-1), items, gp)
    np.add.at(dbu.reshape(-1), nu, gn_flat)
    np.add.at(dbi.reshape(-1), ni, gn_flat)
    return dict(pos=pos, neg=negp, loss=l, gp=gp, gn=gn,
                dWu=dWu, dWi=dWi, dbu=dbu, dbi=dbi)


def bloom_embed(W, rows):
    """layers.py:240-241: sum of the H hashed rows.  rows: (..., H)."""
    return W[rows].sum(axis=-2)


def mf_bloom_step(Wu, Wi, bu, bi, users, items, negs, loss, num_hash, pad=0, dtype=np.float64):
    """One minibatch of BilinearNet with a BloomEmbedding ITEM layer (plain user table):
    the item vector is the sum of the H hashed rows (layers.py:206-244), the biases stay
    indexed by the raw ids (representations.py:58-59).  ``Wi`` is the (M, D) hashed table.
    Returns loss and dense gradients dWu, dWi (M rows, padding row 0 frozen), dbu, dbi.
    Non-adaptive losses only (the sharded hashed path, BASELINE config 4, uses hinge)."""
    from oracle.murmur import bloom_rows
    M = Wi.shape[0]
    ri = bloom_rows(np.asarray(items), num_hash, M, pad)
    rj = bloom_rows(np.asarray(negs), num_hash, M, pad)
    Wu_, Wi_ = Wu.astype(dtype), Wi.astype(dtype)
    u = Wu_[users]
    qi, qj = Wi_[ri].sum(1), Wi_[rj].sum(1)
    pos = (u * qi).sum(1) + bu.reshape(-1)[users] + bi.reshape(-1)[items]
    neg = (u * qj).sum(1) + bu.reshape(-1)[users] + bi.reshape(-1)[negs]
    l, gp, gn = loss_and_score_grads(loss, pos.astype(dtype), neg.astype(dtype), None, dtype)
    dWu = np.zeros(Wu.shape, dtype=np.float64)
    dWi = np.zeros(Wi.shape, dtype=np.float64)
    dbu = np.zeros(bu.shape, dtype=np.float64)
    dbi = np.zeros(bi.shape, dtype=np.float64)
    np.add.at(dWu, users, gp[:, None] * qi + gn[:, None] * qj)
    for k in range(num_hash):
        np.add.at(dWi, ri[:, k], gp[:, None] * u)
        np.add.at(dWi, rj[:, k], gn[:, None] * u)
    dWi[0] = 0                                   # the padding row of the compressed table is frozen
    np.add.at(dbu.reshape(-1), users, gp + gn)
    np.add.at(dbi.reshape(-1), items, gp)
    np.add.at(dbi.reshape(-1), negs, gn)
    return dict(loss=l, pos=pos, neg=neg, dWu=dWu, dWi=dWi, dbu=dbu, dbi=dbi)



def _rank_in_list(rows):
    """Position of every member in its row's member list (members in ascending term order)
    and that list's length."""
    order = np.argsort(rows, kind='stable')
    sr = rows[order]
    rank = np.empty(len(rows), dtype=np.int64)
    rank[order] = np.arange(len(rows)) - np.searchsorted(sr, sr, side='left')
    return rank, np.bincount(rows)[rows]


def _row_sums(shape, rows, vals):
    """Dense (shape) array of the sums of ``vals`` per row id (np.add.at, by sorting)."""
    out = np.zeros(shape)
    if len(rows) == 0:
        return out
    order = np.argsort(rows, kind='stable')
    r = rows[order]
    starts = np.flatnonzero(np.r_[True, r[1:] != r[:-1]])
    out.reshape(shape[0], -1)[r[starts]] = np.add.reduceat(vals[order].reshape(len(rows), -1), starts, axis=0)
    return out


def touched(n, rows, g):
    """Rows (of a table of ``n``) that carry a gradient term with g != 0: the rows the compact
    segment list holds (mf_fill_kernel places a term only when its score gradient is non-zero).
    ``rows`` / ``g``: the terms' row ids and score gradients."""
    out = np.zeros(n, dtype=bool)
    out[np.asarray(rows)[np.asarray(g) != 0]] = True
    return out


def fused_step(params, users, items, negs, loss, opt, lr, weight_decay=0.0, eps=1e-10, states=None,
               norm=None, mutate=(), cap=128):
    """One in-place float64 step of the planned route (pointwise / bpr / hinge) with the fused
    row-wise optimizer.  ``params`` = (Wu, Wi, bu, bi) and Adagrad ``states`` are float64 arrays,
    updated in place.  ``norm`` is the batch the loss is averaged over (default len(users); the
    global batch in gradient-out mode).  A user row is touched when one of its interactions has
    gp != 0 or gn != 0, an item row when one of its terms (positive or negative) has g != 0;
    touched rows take ``g + weight_decay * w``, the others stay bit-identical.

    Returns dict(loss, pos, neg, gp, gn, dWu, dWi, dbu, dbi, touched_u, touched_i), the gradients and the
    loss already divided by ``norm``."""
    Wu, Wi, bu, bi = params
    users, items, negs = (np.asarray(x, dtype=np.int64) for x in (users, items, negs))
    B = len(users)
    norm = B if (norm is None or 'local_norm' in mutate) else norm
    # mf_step's scores and score gradients; the row sums below are mf_step's, per term
    pos = bilinear_scores(Wu, Wi, bu, bi, users, items, np.float64)
    neg = bilinear_scores(Wu, Wi, bu, bi, users, negs, np.float64)
    lval, gp, gn = loss_and_score_grads(loss, pos, neg, None, np.float64)
    gp, gn = gp * (B / norm), gn * (B / norm)
    if 'hinge_strict' in mutate and loss == 'hinge':
        act = (neg - pos + 1.0) > 0.0
        gp, gn = np.where(act, gp, 0.0), np.where(act, gn, 0.0)

    keep_u = np.ones(B, dtype=bool)
    t_row = np.stack([items, negs], axis=1).reshape(-1)          # term 2b: positive, 2b + 1: negative
    if 'neg_to_pos_row' in mutate:
        t_row = np.repeat(items, 2)
    t_g = np.stack([gp, gn], axis=1).reshape(-1)
    t_user = np.repeat(users, 2)
    keep_i = np.ones(2 * B, dtype=bool)
    if 'item_first4' in mutate:
        rank, length = _rank_in_list(t_row)
        keep_i &= (rank < 4) | (length > cap)
    if 'hot_drop_last' in mutate:
        for keep, rows in ((keep_u, users), (keep_i, t_row)):
            rank, length = _rank_in_list(rows)
            keep &= ~((length > cap) & (rank == length - 1))

    wds = [weight_decay] * 4
    if 'no_decay_user_rows' in mutate:
        wds[0] = 0.0
    if 'no_decay_biases' in mutate:
        wds[2] = wds[3] = 0.0

    # user side: forward against the old item rows, then the user rows' update
    Wu_old = Wu.copy()
    ku = np.nonzero(keep_u)[0]
    dWu = _row_sums(Wu.shape, users[ku], gp[ku, None] * Wi[items[ku]] + gn[ku, None] * Wi[negs[ku]])
    gbu = gp if 'user_bias_no_gn' in mutate else gp + gn
    dbu = _row_sums(bu.shape, users[ku], gbu[ku])
    tu = touched(Wu.shape[0], t_user, np.where(np.repeat(keep_u, 2), t_g, 0.0))
    if 'decay_all_rows' in mutate:
        tu[users] = True
    apply_rowwise((Wu, bu), (dWu, dbu), (tu, tu), opt, lr, (wds[0], wds[2]), eps,
                  None if states is None else (states[0], states[2]), mutate)

    # item side: the stash holds the pre-update user rows
    src = Wu if 'stash_post_update' in mutate else Wu_old
    ki = np.nonzero(keep_i)[0]
    dWi = _row_sums(Wi.shape, t_row[ki], t_g[ki, None] * src[t_user[ki]])
    dbi = _row_sums(bi.shape, t_row[ki], t_g[ki])
    ti = touched(Wi.shape[0], t_row, np.where(keep_i, t_g, 0.0))
    if 'decay_all_rows' in mutate:
        ti[t_row] = True
    apply_rowwise((Wi, bi), (dWi, dbi), (ti, ti), opt, lr, (wds[1], wds[3]), eps,
                  None if states is None else (states[1], states[3]), mutate)
    return dict(loss=float(lval) * B / norm, pos=pos, neg=neg, gp=gp, gn=gn, dWu=dWu, dWi=dWi, dbu=dbu, dbi=dbi,
                touched_u=tu, touched_i=ti)


def fit(params, users, items, num_items, loss, batch_size, n_iter, random_state, opt, lr,
        weight_decay=0.0, eps=1e-10, states=None, mutate=()):
    """The reference's fit loop (spotlight/factorization/implicit.py:184-252) on the planned
    route, in float64: per epoch one ``shuffle(arange(n))``, then per minibatch one
    ``randint(0, num_items, len(batch))`` for the negatives and a ``fused_step``.
    ``random_state`` stands where the model's constructor left it.  Parameters and states are
    updated in place; returns the epoch losses (mean of the minibatch losses)."""
    n = len(users)
    losses = []
    for _ in range(n_iter):
        order = np.arange(n)
        random_state.shuffle(order)
        u, i = np.asarray(users)[order].astype(np.int64), np.asarray(items)[order].astype(np.int64)
        ep = []
        for lo in range(0, n, batch_size):
            bu_, bi_ = u[lo:lo + batch_size], i[lo:lo + batch_size]
            negs = random_state.randint(0, num_items, len(bu_), dtype=np.int64)
            ep.append(fused_step(params, bu_, bi_, negs, loss, opt, lr, weight_decay, eps, states,
                                 mutate=mutate)['loss'])
        losses.append(float(np.mean(ep)))
    return losses
