"""PoolNet / CNNNet sequence step, closed-form forward/backward (oracle).

TEST INFRASTRUCTURE ONLY.  Restates, in NumPy:

* ``PoolNet.user_representation`` / ``forward``
  spotlight/sequence/representations.py:91-114, 136-144
* ``CNNNet.user_representation`` / ``forward``
  spotlight/sequence/representations.py:385-422, 444-453
* the training step of spotlight/sequence/implicit.py:230-255 (mask =
  ``seq != PADDING_IDX``; adaptive negatives via ``repeat`` :278-286)

and the gradients autograd produces for them (padding rows of the item
embedding and item bias receive zero gradient: ``padding_idx=PADDING_IDX`` at
representations.py:68-72, 349-353).  Pinned against golden vectors from the
live reference in tests/test_oracle_seq.py.

``mutate`` (a tuple of names, empty by default) restates plausible kernel
mistakes for tests/test_seq_oracle_cpu.py, which shows that the GPU
tolerances catch each of them:

* ``'count_per_row'``  PoolNet divides by a per-row count of non-padding items
  instead of the per-element count of non-zero entries;
* ``'pad0_rf_minus_1'`` CNNNet pads layer 0 by rf - 1 instead of rf;
* ``'residual_shift'``  CNNNet adds e_t instead of e_{t-1} on layer 0's residual.
"""

import numpy as np

from oracle.mf import loss_and_score_grads

PADDING_IDX = 0


def pool_representation(E, seq, dtype=np.float32, mutate=()):
    """All S+1 prefix representations, shape (B, S+1, D).

    r_t = sum_{s<t} e_s / (sum_{s<t} [e_s != 0] + 1), element-wise count
    (representations.py:104-112).
    """
    e = E[seq].astype(dtype)                                  # (B,S,D)
    B, S, D = e.shape
    P = np.zeros((B, S + 1, D), dtype=dtype)
    C = np.zeros((B, S + 1, D), dtype=dtype)
    P[:, 1:] = np.cumsum(e, axis=1, dtype=dtype)
    nz = e != 0.0
    if 'count_per_row' in mutate:
        nz = np.broadcast_to((seq != PADDING_IDX)[..., None], e.shape)
    C[:, 1:] = np.cumsum(nz.astype(dtype), axis=1, dtype=dtype)
    return P / (C + 1.0), C


def _scores(r, E, bias, tgt, dtype):
    """representations.py:136-144 : <r_t, E[tgt_t]> + bias[tgt_t]."""
    te = E[tgt].astype(dtype)
    return (r * te).sum(axis=-1, dtype=dtype) + bias[tgt].reshape(tgt.shape).astype(dtype)


def _targets_backward(E, bias, r, seq, negs, gp, gn, dE, dbias, dtype):
    """Target-role grads + d loss / d r.  negs/gn: (n,B,S)."""
    D = E.shape[1]
    np.add.at(dE, seq.reshape(-1), (gp[..., None] * r).reshape(-1, D))
    np.add.at(dbias.reshape(-1), seq.reshape(-1), gp.reshape(-1))
    dr = gp[..., None] * E[seq].astype(dtype)
    for k in range(negs.shape[0]):
        np.add.at(dE, negs[k].reshape(-1), (gn[k][..., None] * r).reshape(-1, D))
        np.add.at(dbias.reshape(-1), negs[k].reshape(-1), gn[k].reshape(-1))
        dr = dr + gn[k][..., None] * E[negs[k]].astype(dtype)
    return dr


def _prep_negs(negs, B, S, loss, n_neg):
    if loss == 'adaptive_hinge':
        return negs.reshape(n_neg, B, S)       # rows k*B+b  (implicit.py:281-286)
    return negs.reshape(1, B, S)


def pool_step(E, bias, seq, negs, loss='pointwise', n_neg=1, dtype=np.float32, mutate=()):
    """One PoolNet minibatch.  negs: (B,S), or (n*B,S) for adaptive_hinge.

    Also returns the score gradients gp (B,S) and gn ((n,B,S) for adaptive_hinge, else (B,S)).
    """
    B, S = seq.shape
    D = E.shape[1]
    rall, C = pool_representation(E, seq, dtype, mutate)
    r = rall[:, :S]
    negs3 = _prep_negs(negs, B, S, loss, n_neg)
    pos = _scores(r, E, bias, seq, dtype)
    neg = np.stack([_scores(r, E, bias, negs3[k], dtype) for k in range(negs3.shape[0])])
    mask = seq != PADDING_IDX
    if loss == 'adaptive_hinge':
        lval, gp, gn = loss_and_score_grads(loss, pos, neg, mask, dtype)
    else:
        lval, gp, gn0 = loss_and_score_grads(loss, pos, neg[0], mask, dtype)
        gn = gn0[None]
    dE = np.zeros(E.shape, dtype=dtype)
    dbias = np.zeros(bias.shape, dtype=dtype)
    dr = _targets_backward(E, bias, r, seq, negs3, gp, gn, dE, dbias, dtype)
    dP = dr / (C[:, :S] + 1.0)
    # input role: e_s feeds every P_t with t > s  -> exclusive suffix sum
    suffix = np.cumsum(dP[:, ::-1], axis=1, dtype=dtype)[:, ::-1]
    dinp = np.zeros_like(dP)
    dinp[:, :-1] = suffix[:, 1:]
    np.add.at(dE, seq.reshape(-1), dinp.reshape(-1, D))
    dE[PADDING_IDX] = 0
    dbias[PADDING_IDX] = 0
    return dict(pos=pos, neg=neg if loss == 'adaptive_hinge' else neg[0], loss=lval,
                dE=dE, dbias=dbias, final=rall[:, S], gp=gp, gn=gn if loss == 'adaptive_hinge' else gn[0])


def _act(x, kind):
    return np.tanh(x) if kind == 'tanh' else np.maximum(x, 0.0)


def _dact(a, kind):
    return 1.0 - a * a if kind == 'tanh' else (a > 0.0).astype(a.dtype)


def cnn_representation(E, convs, seq, kernel_width, dilation, nonlinearity='tanh',
                       residual=True, dtype=np.float32, mutate=()):
    """CNNNet.user_representation.  convs: list of (W (D,D,k,1), b (D,)).

    Returns (y (B,S+1,D), saved) where y[:, t] only sees items < t.
    """
    e = E[seq].astype(dtype)
    B, S, D = e.shape
    saved = []
    x = None
    for l, (W, b) in enumerate(convs):
        k, d = kernel_width[l], dilation[l]
        rf = k + (k - 1) * (d - 1)
        if l == 0:
            xin = np.zeros((B, S + rf, D), dtype=dtype)      # left pad rf (not rf-1)
            pad0 = rf - 1 if 'pad0_rf_minus_1' in mutate else rf
            xin[:, pad0:pad0 + S] = e
        else:
            xin = np.zeros((B, S + 1 + rf - 1, D), dtype=dtype)
            xin[:, rf - 1:] = x
        z = np.zeros((B, S + 1, D), dtype=dtype) + b.astype(dtype)
        for j in range(k):
            tap = xin[:, j * d: j * d + S + 1]               # (B,S+1,Din)
            z = z + np.einsum('bti,oi->bto', tap, W[:, :, j, 0].astype(dtype))
        a = _act(z, nonlinearity).astype(dtype)
        if residual:
            if l == 0:
                res = np.zeros((B, S + 1, D), dtype=dtype)
                if 'residual_shift' in mutate:
                    res[:, :S] = e
                else:
                    res[:, 1:] = e
            else:
                res = x
            y = a + res
        else:
            y = a
        saved.append((xin, a))
        x = y
    return x, saved


def cnn_step(E, bias, convs, seq, negs, kernel_width, dilation, loss='pointwise',
             n_neg=1, nonlinearity='tanh', residual=True, dtype=np.float32, mutate=()):
    """One CNNNet minibatch: loss and grads for E, bias and every conv (and gp / gn as in
    pool_step)."""
    B, S = seq.shape
    D = E.shape[1]
    y, saved = cnn_representation(E, convs, seq, kernel_width, dilation,
                                  nonlinearity, residual, dtype, mutate)
    r = y[:, :S]
    negs3 = _prep_negs(negs, B, S, loss, n_neg)
    pos = _scores(r, E, bias, seq, dtype)
    neg = np.stack([_scores(r, E, bias, negs3[k], dtype) for k in range(negs3.shape[0])])
    mask = seq != PADDING_IDX
    if loss == 'adaptive_hinge':
        lval, gp, gn = loss_and_score_grads(loss, pos, neg, mask, dtype)
    else:
        lval, gp, gn0 = loss_and_score_grads(loss, pos, neg[0], mask, dtype)
        gn = gn0[None]
    dE = np.zeros(E.shape, dtype=dtype)
    dbias = np.zeros(bias.shape, dtype=dtype)
    dr = _targets_backward(E, bias, r, seq, negs3, gp, gn, dE, dbias, dtype)
    dy = np.zeros((B, S + 1, D), dtype=dtype)
    dy[:, :S] = dr
    dconvs = []
    de = np.zeros((B, S, D), dtype=dtype)
    for l in range(len(convs) - 1, -1, -1):
        W, b = convs[l]
        k, d = kernel_width[l], dilation[l]
        rf = k + (k - 1) * (d - 1)
        xin, a = saved[l]
        dz = dy * _dact(a, nonlinearity)
        dW = np.zeros(W.shape, dtype=dtype)
        dxin = np.zeros_like(xin)
        for j in range(k):
            tap = xin[:, j * d: j * d + S + 1]
            dW[:, :, j, 0] = np.einsum('bto,bti->oi', dz, tap)
            dxin[:, j * d: j * d + S + 1] += np.einsum('bto,oi->bti', dz, W[:, :, j, 0].astype(dtype))
        db = dz.sum(axis=(0, 1), dtype=dtype)
        dconvs.append((dW, db))
        if l == 0:
            pad0 = rf - 1 if 'pad0_rf_minus_1' in mutate else rf
            de += dxin[:, pad0:pad0 + S]
            if residual:
                de += dy[:, :S] if 'residual_shift' in mutate else dy[:, 1:]
        else:
            dprev = dxin[:, rf - 1:]
            if residual:
                dprev = dprev + dy
            dy = dprev
    dconvs.reverse()
    np.add.at(dE, seq.reshape(-1), de.reshape(-1, D))
    dE[PADDING_IDX] = 0
    dbias[PADDING_IDX] = 0
    return dict(pos=pos, neg=neg if loss == 'adaptive_hinge' else neg[0], loss=lval,
                dE=dE, dbias=dbias, dconvs=dconvs, final=y[:, S],
                gp=gp, gn=gn if loss == 'adaptive_hinge' else gn[0])
