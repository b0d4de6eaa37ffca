"""LSTMNet sequence step, closed-form forward / backward through time (oracle).

TEST INFRASTRUCTURE ONLY.  Restates, in NumPy:

* ``LSTMNet.user_representation`` / ``forward``
  spotlight/sequence/representations.py:213-258: one ``nn.LSTM`` layer (gate order
  i, f, g, o) over x_0 = 0, x_t = E[seq_{t-1}]; padding is not masked
* the training step of spotlight/sequence/implicit.py:230-255, scored and
  differentiated exactly as in ``oracle.seq`` (whose ``_scores``,
  ``_targets_backward`` and ``_prep_negs`` it uses)

and the gradients autograd produces for them (the padding rows of the item
embedding and bias receive zero gradient).  Pinned against golden vectors from
the live reference in tests/test_lstm_oracle_cpu.py.

``mutate`` (a tuple of names, empty by default) restates plausible recurrence
mistakes for tests/test_lstm_oracle_cpu.py, which shows that the GPU tolerances
catch each of them:

* ``'swap_if'``       gate rows i and f swapped;
* ``'no_zero_step'``  the leading zero step dropped: the state starts at zero on
  the first item instead of being advanced through the biases;
* ``'no_b_hh'``       b_hh omitted;
* ``'dc_no_f'``       BPTT does not carry dc through the forget gate;
* ``'dwhh_ht'``       dW_hh taken against h_t instead of h_{t-1};
* ``'skip_padding'``  the state held over padded inputs instead of advanced.
"""

import numpy as np

from oracle.mf import loss_and_score_grads
from oracle.seq import PADDING_IDX, _prep_negs, _scores, _targets_backward


def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def _swap_if(D):
    return np.r_[D:2 * D, 0:D, 2 * D:4 * D]


def lstm_representation(E, lstm, seq, dtype=np.float32, mutate=()):
    """All S+1 hidden states, (h (B, S+1, D), saved); h[:, t] has seen items < t.

    lstm: dict(w_ih, w_hh (4D, D), b_ih, b_hh (4D,)), the ``nn.LSTM`` parameters.
    """
    e = E[seq].astype(dtype)
    B, S, D = e.shape
    T = S + 1
    w_ih, w_hh = lstm['w_ih'].astype(dtype), lstm['w_hh'].astype(dtype)
    b = lstm['b_ih'].astype(dtype) + (0.0 if 'no_b_hh' in mutate else lstm['b_hh'].astype(dtype))
    if 'swap_if' in mutate:
        w_ih, w_hh, b = w_ih[_swap_if(D)], w_hh[_swap_if(D)], b[_swap_if(D)]
    x = np.zeros((B, T, D), dtype=dtype)
    x[:, 1:] = e
    adv = np.ones((B, T), dtype=bool)            # the step advances the state
    if 'no_zero_step' in mutate:
        adv[:, 0] = False
    if 'skip_padding' in mutate:
        adv[:, 1:] = seq != PADDING_IDX
    h = np.zeros((B, T, D), dtype=dtype)
    c = np.zeros((B, T, D), dtype=dtype)
    gates = np.zeros((B, T, 4, D), dtype=dtype)
    hp = np.zeros((B, D), dtype=dtype)
    cp = np.zeros((B, D), dtype=dtype)
    for t in range(T):
        a = x[:, t] @ w_ih.T + hp @ w_hh.T + b
        i, f = _sigmoid(a[:, :D]), _sigmoid(a[:, D:2 * D])
        g, o = np.tanh(a[:, 2 * D:3 * D]), _sigmoid(a[:, 3 * D:])
        cn = f * cp + i * g
        m = adv[:, t][:, None]
        c[:, t] = np.where(m, cn, cp)
        h[:, t] = np.where(m, o * np.tanh(cn), hp)
        gates[:, t] = np.stack([i, f, g, o], axis=1)
        hp, cp = h[:, t], c[:, t]
    return h, dict(x=x, c=c, gates=gates, adv=adv, w_ih=w_ih, w_hh=w_hh)


def lstm_step(E, bias, lstm, seq, negs, loss='pointwise', n_neg=1, dtype=np.float32, mutate=()):
    """One LSTMNet minibatch: loss, grads for E, bias and the LSTM parameters (``dlstm`` =
    dict(w_ih, w_hh, b_ih, b_hh)), and the score gradients gp / gn as oracle.seq.pool_step."""
    B, S = seq.shape
    D = E.shape[1]
    T = S + 1
    h, sv = lstm_representation(E, lstm, seq, dtype, mutate)
    r = h[:, :S]
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
    dH = np.zeros((B, T, D), dtype=dtype)
    dH[:, :S] = dr
    x, c, gates, adv, w_ih, w_hh = sv['x'], sv['c'], sv['gates'], sv['adv'], sv['w_ih'], sv['w_hh']
    dW_ih = np.zeros(w_ih.shape, dtype=dtype)
    dW_hh = np.zeros(w_hh.shape, dtype=dtype)
    db = np.zeros(4 * D, dtype=dtype)
    dx = np.zeros((B, T, D), dtype=dtype)
    zero = np.zeros((B, D), dtype=dtype)
    dh_next = zero                               # d loss / d h_t through later steps
    dc_next = zero                               # d loss / d c_t through later steps
    for t in range(T - 1, -1, -1):
        dh = dH[:, t] + dh_next
        i, f, g, o = (gates[:, t, k] for k in range(4))
        tc = np.tanh(c[:, t])
        cprev = c[:, t - 1] if t > 0 else zero
        hprev = h[:, t - 1] if t > 0 else zero
        dc = dh * o * (1.0 - tc * tc) + dc_next
        m = adv[:, t][:, None]
        da = np.where(m, np.concatenate([dc * g * i * (1.0 - i), dc * cprev * f * (1.0 - f),
                                         dc * i * (1.0 - g * g), dh * tc * o * (1.0 - o)], axis=1), 0.0)
        dW_ih += da.T @ x[:, t]
        dW_hh += da.T @ (h[:, t] if 'dwhh_ht' in mutate else hprev)
        db += da.sum(axis=0)
        dx[:, t] = da @ w_ih
        # a held step (mutations only) passes its state's gradients straight through
        dh_next = np.where(m, da @ w_hh, dh)
        dc_next = np.where(m, 0.0 if 'dc_no_f' in mutate else dc * f, dc_next)
    if 'swap_if' in mutate:
        dW_ih, dW_hh, db = dW_ih[_swap_if(D)], dW_hh[_swap_if(D)], db[_swap_if(D)]
    np.add.at(dE, seq.reshape(-1), dx[:, 1:].reshape(-1, D))
    dE[PADDING_IDX] = 0
    dbias[PADDING_IDX] = 0
    dlstm = dict(w_ih=dW_ih, w_hh=dW_hh, b_ih=db, b_hh=np.zeros_like(db) if 'no_b_hh' in mutate else db.copy())
    return dict(pos=pos, neg=neg if loss == 'adaptive_hinge' else neg[0], loss=lval,
                dE=dE, dbias=dbias, dlstm=dlstm, final=h[:, S],
                gp=gp, gn=gn if loss == 'adaptive_hinge' else gn[0])
