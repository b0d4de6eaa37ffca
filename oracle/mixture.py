"""MixtureLSTMNet sequence step, closed-form forward / backward (oracle).

TEST INFRASTRUCTURE ONLY.  Restates, in NumPy:

* ``MixtureLSTMNet.user_representation`` / ``forward``
  spotlight/sequence/representations.py:517-596: the LSTM of ``oracle.lstm`` over x_0 = 0,
  x_t = E[seq_{t-1}], then ``nn.Conv1d(D, 2MD, 1)``; output channel j*D + d is row d of block j,
  blocks 0..M-1 the taste components c_m, blocks M..2M-1 the mixture vectors v_m.  An item e
  with bias beta scores  s = beta + sum_m softmax_m(v_m . e) (c_m . e).
* the training step of spotlight/sequence/implicit.py:230-255, with the masked losses and the
  adaptive-hinge credit of ``oracle.mf.loss_and_score_grads``

and the gradients autograd produces for them (the padding rows of the item embedding and bias
receive zero gradient).  Pinned against golden vectors from the live reference in
tests/test_mixture_oracle_cpu.py.

``mutate`` (a tuple of names, empty by default) restates plausible mistakes of the head and the
projection for tests/test_mixture_oracle_cpu.py, which shows that the GPU tolerances catch each
of them:

* ``'swap_cv'``         components and mixture vectors swapped (blocks M..2M-1 read as c);
* ``'softmax_over_d'``  the softmax taken over D instead of M (``F.softmax(v * e, 2).sum(2)``:
  every mixture weight is 1 and carries no gradient);
* ``'dv_no_sbar'``      the s_bar term dropped from dv;
* ``'de_no_v'``         de missing its v term;
* ``'no_proj_bias'``    the projection bias omitted;
* ``'proj_hprev'``      the projection fed h_{t-1} instead of h_t.
"""

import numpy as np

from oracle import lstm as olstm
from oracle.mf import loss_and_score_grads
from oracle.seq import PADDING_IDX, _prep_negs


def _proj_input(h, mutate):
    if 'proj_hprev' not in mutate:
        return h
    hin = np.zeros_like(h)
    hin[:, 1:] = h[:, :-1]
    return hin


def mixture_representation(E, lstm, proj, seq, num_mixtures, dtype=np.float32, mutate=()):
    """(P (B, S+1, 2MD), saved): the projection output, time-major; P[:, t] has seen items < t.

    lstm: the ``nn.LSTM`` parameters as in ``oracle.lstm``; proj: dict(w (2MD, D, 1) or (2MD, D),
    b (2MD,)), the ``nn.Conv1d`` parameters.
    """
    h, sv = olstm.lstm_representation(E, lstm, seq, dtype)
    D = E.shape[1]
    w = proj['w'].reshape(2 * num_mixtures * D, D).astype(dtype)
    hin = _proj_input(h, mutate)
    P = hin @ w.T
    if 'no_proj_bias' not in mutate:
        P = P + proj['b'].astype(dtype)
    return P, dict(h=h, hin=hin, lstm=sv, w=w)


def _split(P, M, D, S, mutate):
    """(components, mixture vectors), each (B, S, M, D), of the trained positions t < S."""
    B = P.shape[0]
    Pb = P[:, :S].reshape(B, S, 2 * M, D)
    c, v = Pb[:, :, :M], Pb[:, :, M:]
    return (v, c) if 'swap_cv' in mutate else (c, v)


def head(c, v, e, beta, mutate=()):
    """Scores (B, S) of item rows e (B, S, D) with biases beta (B, S), and what the backward needs."""
    a = (v * e[:, :, None]).sum(-1)                                  # (B, S, M)
    if 'softmax_over_d' in mutate:
        w = np.ones_like(a)
    else:
        w = np.exp(a - a.max(-1, keepdims=True))
        w = w / w.sum(-1, keepdims=True)
    z = (c * e[:, :, None]).sum(-1)
    sbar = (w * z).sum(-1)
    return beta + sbar, dict(w=w, z=z, sbar=sbar, e=e)


def head_backward(g, c, v, hc, mutate=()):
    """(dc, dv, de) of the head for score gradients g (B, S)."""
    w, z, sbar, e = hc['w'], hc['z'], hc['sbar'], hc['e']
    gw = g[..., None] * w                                            # (B, S, M)
    dz = z - (0.0 if 'dv_no_sbar' in mutate else sbar[..., None])
    dc = gw[..., None] * e[:, :, None]
    if 'softmax_over_d' in mutate:
        dv = np.zeros_like(v)
        u = np.zeros_like(gw)
    else:
        dv = (gw * dz)[..., None] * e[:, :, None]
        u = gw * (z - sbar[..., None])
    de = (gw[..., None] * c).sum(2)
    if 'de_no_v' not in mutate:
        de = de + (u[..., None] * v).sum(2)
    return dc, dv, de


def _lstm_backward(sv, h, dH, dtype):
    """Backpropagation through time of oracle.lstm's recurrence from d loss / d h (B, T, D):
    (dict(w_ih, w_hh, b_ih, b_hh), d x (B, T, D))."""
    x, c, gates, w_ih, w_hh = sv['x'], sv['c'], sv['gates'], sv['w_ih'], sv['w_hh']
    B, T, D = h.shape
    dW_ih = np.zeros(w_ih.shape, dtype=dtype)
    dW_hh = np.zeros(w_hh.shape, dtype=dtype)
    db = np.zeros(4 * D, dtype=dtype)
    dx = np.zeros((B, T, D), dtype=dtype)
    zero = np.zeros((B, D), dtype=dtype)
    dh_next, dc_next = zero, zero
    for t in range(T - 1, -1, -1):
        dh = dH[:, t] + dh_next
        i, f, g, o = (gates[:, t, k] for k in range(4))
        tc = np.tanh(c[:, t])
        cprev = c[:, t - 1] if t > 0 else zero
        hprev = h[:, t - 1] if t > 0 else zero
        dc = dh * o * (1.0 - tc * tc) + dc_next
        da = np.concatenate([dc * g * i * (1.0 - i), dc * cprev * f * (1.0 - f),
                             dc * i * (1.0 - g * g), dh * tc * o * (1.0 - o)], axis=1)
        dW_ih += da.T @ x[:, t]
        dW_hh += da.T @ hprev
        db += da.sum(axis=0)
        dx[:, t] = da @ w_ih
        dh_next = da @ w_hh
        dc_next = dc * f
    return dict(w_ih=dW_ih, w_hh=dW_hh, b_ih=db, b_hh=db.copy()), dx


def mixture_step(E, bias, lstm, proj, seq, negs, num_mixtures, loss='pointwise', n_neg=1, dtype=np.float32,
                 mutate=()):
    """One MixtureLSTMNet minibatch: loss, scores, grads for E, bias, the LSTM (``dlstm``) and the
    projection (``dmix`` = dict(w (2MD, D, 1), b)), the score gradients gp / gn as
    oracle.seq.pool_step, the target's mixture weights ``w_pos`` (B, S, M) and the final
    representation ``final`` (B, 2MD)."""
    B, S = seq.shape
    D = E.shape[1]
    M = num_mixtures
    T = S + 1
    P, sv = mixture_representation(E, lstm, proj, seq, M, dtype, mutate)
    c, v = _split(P, M, D, S, mutate)
    negs3 = _prep_negs(negs, B, S, loss, n_neg)
    bias1 = bias.reshape(-1).astype(dtype)
    pos, hp = head(c, v, E[seq].astype(dtype), bias1[seq], mutate)
    nh = [head(c, v, E[negs3[k]].astype(dtype), bias1[negs3[k]], mutate) for k in range(negs3.shape[0])]
    neg = np.stack([s for s, _ in nh])
    mask = seq != PADDING_IDX
    if loss == 'adaptive_hinge':
        lval, gp, gn = loss_and_score_grads(loss, pos, neg, mask, dtype)
    else:
        lval, gp, gn0 = loss_and_score_grads(loss, pos, neg[0], mask, dtype)
        gn = gn0[None]
    dE = np.zeros(E.shape, dtype=dtype)
    dbias = np.zeros(bias.shape, dtype=dtype)
    db1 = dbias.reshape(-1)
    dc, dv, de = head_backward(gp, c, v, hp, mutate)
    np.add.at(dE, seq.reshape(-1), de.reshape(-1, D))
    np.add.at(db1, seq.reshape(-1), gp.reshape(-1))
    for k in range(negs3.shape[0]):
        dck, dvk, dek = head_backward(gn[k], c, v, nh[k][1], mutate)
        dc, dv = dc + dck, dv + dvk
        np.add.at(dE, negs3[k].reshape(-1), dek.reshape(-1, D))
        np.add.at(db1, negs3[k].reshape(-1), gn[k].reshape(-1))
    if 'swap_cv' in mutate:
        dc, dv = dv, dc
    dP = np.zeros((B, T, 2 * M * D), dtype=dtype)
    dP[:, :S] = np.concatenate([dc, dv], axis=2).reshape(B, S, 2 * M * D)
    hin, w = sv['hin'], sv['w']
    dW = np.einsum('btj,btd->jd', dP, hin)
    dbp = dP.sum(axis=(0, 1))
    dhin = dP @ w
    if 'proj_hprev' in mutate:
        dH = np.zeros_like(dhin)
        dH[:, :-1] = dhin[:, 1:]
    else:
        dH = dhin
    dlstm, dx = _lstm_backward(sv['lstm'], sv['h'], dH, dtype)
    np.add.at(dE, seq.reshape(-1), dx[:, 1:].reshape(-1, D))
    dE[PADDING_IDX] = 0
    dbias[PADDING_IDX] = 0
    return dict(pos=pos, neg=neg if loss == 'adaptive_hinge' else neg[0], loss=lval,
                dE=dE, dbias=dbias, dlstm=dlstm, dmix=dict(w=dW.reshape(2 * M * D, D, 1), b=dbp),
                final=P[:, S], w_pos=hp['w'], gp=gp, gn=gn if loss == 'adaptive_hinge' else gn[0])
