"""BilinearNet with hashed (Bloom) embedding tables under a rating loss: one training step and
the fit loop in float64 (oracle).

TEST INFRASTRUCTURE ONLY.  Restates what ``slb_mf_bloom_train_step`` (csrc/mf.cu) computes with
a rating loss (regression / poisson / logistic) -- the loop body of
``ExplicitFactorizationModel.fit`` (spotlight/factorization/explicit.py:223-234) on a
``BilinearNet`` whose user and / or item layer is a ``BloomEmbedding``.  It combines the two
oracles that already exist:

* the tables, hashes, padding and frozen rows, and the per-hash gradient terms of
  ``oracle.bloom`` (each side plain or hashed; the entity's vector is the sum of its rows; every
  (hashed user row, hashed item row) term with score gradient g adds g * (item vector) to its user
  row and g * (user vector) to its item row, from the tables as they were before the step);
* the rating losses and the row-wise optimizer of ``oracle.explicit``: the score is
  ``u . q + bu[u] + bi[i]``, the loss and d loss / d score are ``loss_and_score_grad``'s, the
  id-space biases take dbu[u] += g, dbi[i] += g, and in fused mode an entry is touched (updated and
  decayed) when its interaction has g != 0, the frozen row excepted.

``mutate`` takes ``oracle.bloom``'s table mutations (``pad_hashed``, ``freeze_row0``,
``train_frozen``, ``item_first_hash``, ``item_mean``, ``dup_row_once``, ``stash_post_update``,
``decay_all_rows``), ``oracle.explicit``'s loss and optimizer mutations, and in ``fit``
``full_batch_norm``; tests/test_explicit_bloom_oracle_cpu.py shows the GPU tolerances catch them.
"""

import numpy as np

from oracle.bloom import _bias_pairs, _row_grads, _vectors, frozen_row, table_rows
from oracle.explicit import apply_rowwise, loss_and_score_grad


def step(params, users, items, ratings, loss, Hu=0, Hi=0, pad_u=0, pad_i=0, opt=None, lr=0.0,
         weight_decay=0.0, eps=1e-10, states=None, norm=None, mutate=()):
    """One float64 step.  ``params`` = [Wu, Wi, bu, bi] (Wu / Wi the plain or compressed tables,
    bu / bi of shape (num_users, 1) / (num_items, 1)); the loss is divided by ``norm`` (default B).

    ``opt=None`` is the dense mode: nothing is updated.  ``opt`` in ('sgd', 'adagrad') is the
    fused mode: ``params`` (and the Adagrad ``states``) are updated in place.  Returns
    dict(loss, pos, gs, dWu, dWi, dbu, dbi, touched=(Wu, Wi, bu, bi) masks)."""
    Wu, Wi, bu, bi = params
    users, items = (np.asarray(x, dtype=np.int64).reshape(-1) for x in (users, items))
    B = len(users)
    norm = B if norm is None else norm
    Mu, Mi = Wu.shape[0], Wi.shape[0]
    W0u = Wu.copy()
    ru, ri = table_rows(users, Hu, Mu, pad_u, mutate), table_rows(items, Hi, Mi, pad_i, mutate)
    iv = _vectors(Wi, ri, True, mutate)
    pos = (_vectors(Wu, ru, False, mutate) * iv).sum(axis=1) + bu.reshape(-1)[users] + bi.reshape(-1)[items]
    lval, g = loss_and_score_grad(loss, pos, ratings, norm, mutate)
    fu, fi = frozen_row(Hu, pad_u, mutate), frozen_row(Hi, pad_i, mutate)

    def user_grads():
        d = _row_grads(Wu.shape, ru, g, iv, mutate)
        if fu >= 0:
            d[fu] = 0.0
        return d

    def item_grads(Wsrc):
        rows = ri[:, :1] if 'item_first_hash' in mutate else ri
        gi = g / rows.shape[1] if 'item_mean' in mutate else g
        d = _row_grads(Wi.shape, rows, gi, _vectors(Wsrc, ru, False, mutate), mutate)
        if fi >= 0:
            d[fi] = 0.0
        return d

    def touched(M, rows, frozen):
        act = np.ones(B, dtype=bool) if 'decay_all_rows' in mutate else g != 0
        t = np.zeros(M, dtype=bool)
        t[rows[act].reshape(-1)] = True
        if frozen >= 0:
            t[frozen] = False
        return t

    tWu, tWi = touched(Mu, ru, fu), touched(Mi, ri, fi)
    tbu, tbi = touched(bu.shape[0], users[:, None], -1), touched(bi.shape[0], items[:, None], -1)
    dbu = _bias_pairs(users, g, bu.shape[0], B, mutate).reshape(bu.shape)
    dbi = _bias_pairs(items, g, bi.shape[0], B, mutate).reshape(bi.shape)
    out = dict(loss=float(lval) * B / norm, pos=pos, gs=g, touched=(tWu, tWi, tbu, tbi), dbu=dbu, dbi=dbi)
    if opt is None:
        out.update(dWu=user_grads(), dWi=item_grads(Wu))
        return out
    wds = (weight_decay,) * 2
    st = (lambda a, b: None) if states is None else (lambda a, b: (states[a], states[b]))
    if 'stash_post_update' in mutate:
        dWu = user_grads()
        apply_rowwise((Wu, bu), (dWu, dbu), (tWu, tbu), opt, lr, wds, eps, st(0, 2), mutate)
        dWi = item_grads(Wu)
    else:
        dWi = item_grads(W0u)
        dWu = user_grads()
        apply_rowwise((Wu, bu), (dWu, dbu), (tWu, tbu), opt, lr, wds, eps, st(0, 2), mutate)
    apply_rowwise((Wi, bi), (dWi, dbi), (tWi, tbi), opt, lr, wds, eps, st(1, 3), mutate)
    out.update(dWu=dWu, dWi=dWi)
    return out


def fit(params, users, items, ratings, loss, batch_size, n_iter, random_state, opt, lr, Hu=0, Hi=0,
        pad_u=0, pad_i=0, weight_decay=0.0, eps=1e-10, states=None, mutate=()):
    """The reference's explicit fit loop (spotlight/factorization/explicit.py:199-243) on the
    hashed step, in float64: per epoch one ``shuffle(arange(n))`` (the only use of the
    ``RandomState``), then a fused ``step`` per minibatch (``full_batch_norm`` in ``mutate``: a
    short last batch normalised by ``batch_size``).  Parameters and states are updated in place;
    returns the epoch losses (mean of the minibatch losses)."""
    n = len(users)
    losses = []
    for _ in range(n_iter):
        order = np.arange(n)
        random_state.shuffle(order)
        u, i = np.asarray(users)[order].astype(np.int64), np.asarray(items)[order].astype(np.int64)
        r = np.asarray(ratings)[order]
        norm = batch_size if 'full_batch_norm' in mutate else None
        ep = [step(params, u[lo:lo + batch_size], i[lo:lo + batch_size], r[lo:lo + batch_size], loss, Hu, Hi,
                   pad_u, pad_i, opt, lr, weight_decay, eps, states, norm, mutate)['loss']
              for lo in range(0, n, batch_size)]
        losses.append(float(np.mean(ep)))
    return losses
