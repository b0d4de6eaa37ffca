"""BilinearNet + explicit-feedback (rating) losses, closed-form forward/backward (oracle).

TEST INFRASTRUCTURE ONLY.  Restates, in NumPy:

* ``regression_loss`` / ``poisson_loss`` / ``logistic_loss``   spotlight/losses.py:169-244
  (plain mean; logistic clamps the targets to [0, 1]; poisson sees ``exp(score)``, which
  ``fit`` applies first, spotlight/factorization/explicit.py:225-226)
* the autograd result of ``loss.backward()`` for one minibatch of
  ``ExplicitFactorizationModel.fit`` (explicit.py:215-234)
* SGD / Adagrad steps (torch.optim, lr_decay 0, initial accumulator 0) and the ``fit`` loop,
  whose only use of the ``RandomState`` is one ``shuffle(arange(n))`` per epoch.

``mutate`` (a tuple of names, empty by default) restates plausible kernel mistakes, so that
tests/test_explicit_oracle_cpu.py can show the GPU tolerance catches each of them:

``regression_no_factor2``   d/ds (r - s)^2 taken as (s - r)
``poisson_grad_r_minus_p``  poisson gradient with the wrong sign, r - p
``poisson_grad_on_s``       poisson gradient taken against s instead of p = exp(s): s - r
``logistic_no_clamp``       -1 ratings kept as the target
``full_batch_norm``         a short last batch normalised by the full batch size
``no_user_bias_grad``       the user-bias gradient dropped
``no_decay_items``          weight decay skipped on updated item rows
"""

import numpy as np

LOSSES = ('regression', 'poisson', 'logistic')


def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def transform(kind, s):
    """What ``predict`` returns for raw scores ``s`` (explicit.py:277-282)."""
    if kind == 'poisson':
        return np.exp(s)
    if kind == 'logistic':
        return _sigmoid(s)
    return s


def loss_and_score_grad(kind, s, r, norm=None, mutate=()):
    """Mean loss over ``len(s)`` and d loss / d s, scaled by 1 / ``norm`` (default len(s))."""
    s = np.asarray(s, dtype=np.float64)
    r = np.asarray(r, dtype=np.float64)
    n = s.size
    norm = n if norm is None else norm
    if kind == 'regression':
        per = (r - s) ** 2
        g = (s - r) if 'regression_no_factor2' in mutate else 2.0 * (s - r)
    elif kind == 'poisson':
        p = np.exp(s)
        per = p - r * s
        if 'poisson_grad_r_minus_p' in mutate:
            g = r - p
        elif 'poisson_grad_on_s' in mutate:
            g = s - r
        else:
            g = p - r
    elif kind == 'logistic':
        t = r if 'logistic_no_clamp' in mutate else np.clip(r, 0.0, 1.0)
        per = np.maximum(s, 0.0) - s * t + np.log1p(np.exp(-np.abs(s)))
        g = _sigmoid(s) - t
    else:
        raise ValueError(kind)
    return per.sum() / n, g / norm


def explicit_step(Wu, Wi, bu, bi, users, items, ratings, loss, norm=None, mutate=()):
    """One minibatch: dict(loss, scores, pred, gs, dWu, dWi, dbu, dbi) in float64."""
    Wu, Wi = Wu.astype(np.float64), Wi.astype(np.float64)
    bu, bi = bu.astype(np.float64).reshape(-1), bi.astype(np.float64).reshape(-1)
    u, q = Wu[users], Wi[items]
    s = (u * q).sum(axis=1) + bu[users] + bi[items]
    l, g = loss_and_score_grad(loss, s, ratings, norm, mutate)
    dWu, dWi = np.zeros_like(Wu), np.zeros_like(Wi)
    dbu, dbi = np.zeros_like(bu), np.zeros_like(bi)
    np.add.at(dWu, users, g[:, None] * q)
    np.add.at(dWi, items, g[:, None] * u)
    if 'no_user_bias_grad' not in mutate:
        np.add.at(dbu, users, g)
    np.add.at(dbi, items, g)
    return dict(loss=l, scores=s, pred=transform(loss, s), gs=g, dWu=dWu, dWi=dWi,
                dbu=dbu.reshape(-1, 1), dbi=dbi.reshape(-1, 1))


def apply_rowwise(params, grads, touched, opt, lr, weight_decay=0.0, eps=1e-10, states=None,
                  mutate=()):
    """The fused row-wise optimizer (spotlight_b200.optim.FusedSGD / FusedAdagrad): the rows in
    ``touched`` (a boolean mask per table; rows with a non-zero score-gradient term) take
    torch.optim's SGD / Adagrad step with ``g + weight_decay * w``; other rows stay.  ``params``,
    ``grads``, ``touched``, ``states`` and a per-table ``weight_decay`` tuple are (Wu, Wi, bu,
    bi)-ordered; updated in place.  The mutation ``adagrad_div_before_add`` divides by the state
    before adding ``g^2`` to it."""
    wds = tuple(weight_decay) if np.ndim(weight_decay) else (weight_decay,) * 4
    for k, (w, g, rows) in enumerate(zip(params, grads, touched)):
        wd = 0.0 if ('no_decay_items' in mutate and k in (1, 3)) else wds[k]
        gg = g[rows] + wd * w[rows]
        if opt == 'sgd':
            w[rows] -= lr * gg
        elif 'adagrad_div_before_add' in mutate:
            st = states[k]
            w[rows] -= lr * gg / (np.sqrt(st[rows]) + eps)
            st[rows] += gg * gg
        else:
            st = states[k]
            st[rows] += gg * gg
            w[rows] -= lr * gg / (np.sqrt(st[rows]) + eps)


def touched_rows(shapes, users, items, gs):
    nz = gs != 0
    tu = np.zeros(shapes[0], dtype=bool)
    ti = np.zeros(shapes[1], dtype=bool)
    tu[users[nz]] = True
    ti[items[nz]] = True
    return tu, ti, tu, ti


def fused_step(params, users, items, ratings, loss, opt, lr, weight_decay=0.0, eps=1e-10,
               states=None, norm=None, mutate=()):
    """One in-place step of the fused route; returns the step's loss dict."""
    Wu, Wi, bu, bi = params
    out = explicit_step(Wu, Wi, bu, bi, users, items, ratings, loss, norm, mutate)
    tu, ti, _, _ = touched_rows((Wu.shape[0], Wi.shape[0]), users, items, out['gs'])
    apply_rowwise(params, (out['dWu'], out['dWi'], out['dbu'], out['dbi']), (tu, ti, tu, ti), opt, lr,
                  weight_decay, eps, states, mutate)
    return out


def fit(params, users, items, ratings, loss, batch_size, n_iter, random_state, opt, lr,
        weight_decay=0.0, eps=1e-10, states=None, mutate=()):
    """The reference's fit loop (explicit.py:199-243) with SGD or Adagrad, in float64; the
    parameters (and Adagrad ``states``) are updated in place.  Returns the epoch losses."""
    n = len(users)
    losses = []
    for _ in range(n_iter):
        order = np.arange(n)
        random_state.shuffle(order)
        u, i, r = users[order], items[order], ratings[order]
        total, nb = 0.0, 0
        for lo in range(0, n, batch_size):
            hi = min(n, lo + batch_size)
            norm = batch_size if 'full_batch_norm' in mutate else None
            out = fused_step(params, u[lo:hi], i[lo:hi], r[lo:hi], loss, opt, lr, weight_decay, eps,
                             states, norm, mutate)
            total += out['loss']
            nb += 1
        losses.append(total / nb)
    return losses
