"""Lazy-exact row-wise Adam, restated on the CPU (TEST INFRASTRUCTURE ONLY).

The reference's default optimizer is dense ``torch.optim.Adam(params, weight_decay=l2, lr)``
(spotlight/factorization/implicit.py:143-148): every row moves at every step, also rows without
a gradient (their first moment decays).  The product (spotlight_b200/csrc/mf_adam.cuh) applies it
row-wise and lazily; this module states the same scheme in NumPy float64 so that the *scheme*
-- catch-up of every referenced row BEFORE the forward pass, real step on the touched rows,
flush at the end -- can be pinned on the CPU against the reference's recorded default-Adam
trajectory (tests/golden/fit_pointwise_adam.npz) and against torch.optim.Adam.

Per element and step t (torch/optim/adam.py, _single_tensor_adam):
    g += wd * w;  m += (g - m) * (1 - b1);  v = v * b2 + (1 - b2) * g * g
    w -= lr / (1 - b1^t) * m / (sqrt(v) / sqrt(1 - b2^t) + eps)
"""

import numpy as np


class LazyAdamTable(object):
    """One (rows, D) table with its Adam state and the step each row is current for."""

    def __init__(self, w, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0):
        self.w = np.array(w, dtype=np.float64)
        self.m = np.zeros_like(self.w)
        self.v = np.zeros_like(self.w)
        self.last = np.zeros(self.w.shape[0], dtype=np.int64)
        self.lr, (self.b1, self.b2), self.eps, self.wd = lr, betas, eps, weight_decay

    def _step(self, rows, t, g):
        g = g + self.wd * self.w[rows]
        self.m[rows] += (g - self.m[rows]) * (1.0 - self.b1)
        self.v[rows] = self.v[rows] * self.b2 + (1.0 - self.b2) * g * g
        ss, bc = self.lr / (1.0 - self.b1 ** t), np.sqrt(1.0 - self.b2 ** t)
        self.w[rows] -= ss * (self.m[rows] / (np.sqrt(self.v[rows]) / bc + self.eps))

    def catch_up(self, rows, upto):
        """Replay the gradient-free steps (last, upto] of ``rows`` (mf_adam_prepass_kernel): for
        each step s, every row still behind s takes it together.  Element for element the same
        float64 operations as ``catch_up_loop``, which it is pinned to."""
        rows = np.unique(np.asarray(rows, dtype=np.int64))
        rows = rows[self.last[rows] < upto]
        if len(rows) == 0:
            return
        last = self.last[rows]
        for t in range(int(last.min()) + 1, upto + 1):
            self._step(rows[last < t], t, 0.0)
        self.last[rows] = upto

    def catch_up_loop(self, rows, upto):
        """``catch_up`` one row and one step at a time (the plain statement of it)."""
        rows = np.unique(np.asarray(rows))
        for r in rows:
            for t in range(int(self.last[r]) + 1, upto + 1):
                self._step(np.array([r]), t, 0.0)
            self.last[r] = max(int(self.last[r]), upto)

    def apply(self, rows, grads, t):
        """The real step t on the touched rows (mf_adam_apply_kernel); rows must be current for t-1."""
        rows = np.asarray(rows)
        assert (self.last[rows] == t - 1).all()
        self._step(rows, t, grads)
        self.last[rows] = t

    def flush(self, t):
        """Every row current for step t (adam_flush_kernel)."""
        self.catch_up(np.arange(self.w.shape[0]), t)


# ---- the first-generation MF step under lazy-exact Adam (csrc/mf.cu launch_step, SLB_OPT_ADAM) -----
#
# Four tables (Wu, Wi, bu, bi); each bias shares its embedding's `last` (both LazyAdamTables of a pair
# keep equal `last` arrays).  Step t:
#   1. mf_adam_prepass_kernel: every referenced row -- the users; the items and all B * n_neg
#      negatives (rating losses: the items) -- with its bias is caught up through t - 1;
#   2. the forward and backward on those tables (oracle.mf.mf_step / oracle.explicit.explicit_step);
#   3. mf_adam_apply_kernel: step t on the rows with a non-zero score-gradient term only
#      (oracle.mf.touched), so rows referenced but not touched end at last = t - 1.
#
# ``mutate`` restates plausible kernel mistakes (tests/test_mf_adam_oracle_cpu.py shows that the GPU
# tolerances catch each):
#
# ``prepass_no_negs``       the negatives are not caught up before the forward
# ``bias_own_last``         the bias reads its own copy of `last`, which the prepass already advanced:
#                           it never replays its missed steps
# ``catch_up_through_t``    the prepass replays (last, t] instead of (last, t - 1]
# ``apply_all_referenced``  step t applied to every referenced row, touched or not
# ``no_decay_replay``       the replayed steps leave out weight decay

MF_MUTATIONS = ('prepass_no_negs', 'bias_own_last', 'catch_up_through_t', 'apply_all_referenced', 'no_decay_replay')


def _catch_up_pair(emb, bias, rows, upto, mutate):
    wd = emb.wd, bias.wd
    if 'no_decay_replay' in mutate:
        emb.wd = bias.wd = 0.0
    if 'bias_own_last' in mutate:
        r = np.unique(np.asarray(rows, dtype=np.int64))
        bias.last[r] = np.maximum(bias.last[r], upto)
    else:
        bias.catch_up(rows, upto)
    emb.catch_up(rows, upto)
    emb.wd, bias.wd = wd


def mf_terms(P, users, items, negs, loss, n_neg=1, ratings=None):
    """Forward and backward of one step in float64 on the tables P = [Wu, Wi, bu, bi]: the oracle's
    dict plus ``terms`` = (user rows, item rows, score gradients) of every gradient term (positive
    terms, then the B * n_neg negative terms, most of them 0 under adaptive hinge)."""
    from oracle import explicit as oex
    from oracle import mf as omf
    if loss in oex.LOSSES:
        ref = oex.explicit_step(*P, users, items, ratings, loss)
        ref['terms'] = (users, items, ref['gs'])
        return ref
    ref = omf.mf_step(*P, users, items, negs, loss, n_neg, np.float64)
    nu, ni = omf.negative_pairs(users, negs, n_neg, loss == 'adaptive_hinge')
    ref['terms'] = (np.r_[users, nu], np.r_[items, ni], np.r_[ref['gp'], ref['gn'].reshape(-1)])
    return ref


def lazy_mf_step(tabs, users, items, negs, loss, t, n_neg=1, ratings=None, mutate=()):
    """One step t on the four LazyAdamTables ``tabs`` (modified in place); ``negs`` is None for the
    rating losses, which take ``ratings``.  Returns mf_terms's dict plus touched_u / touched_i."""
    from oracle import mf as omf
    Wu, Wi, bu, bi = tabs
    users, items = (np.asarray(x, dtype=np.int64).reshape(-1) for x in (users, items))
    negs = None if negs is None else np.asarray(negs, dtype=np.int64).reshape(-1)
    iref = items if negs is None or 'prepass_no_negs' in mutate else np.r_[items, negs]
    upto = t if 'catch_up_through_t' in mutate else t - 1
    _catch_up_pair(Wu, bu, users, upto, mutate)
    _catch_up_pair(Wi, bi, iref, upto, mutate)
    ref = mf_terms([tab.w for tab in tabs], users, items, negs, loss, n_neg, ratings)
    tu_rows, ti_rows, g = ref['terms']
    tu, ti = omf.touched(Wu.w.shape[0], tu_rows, g), omf.touched(Wi.w.shape[0], ti_rows, g)
    if 'apply_all_referenced' in mutate:
        tu[users] = True
        ti[items if negs is None else np.r_[items, negs]] = True
    for emb, bias, mask, g, gb in ((Wu, bu, tu, ref['dWu'], ref['dbu']), (Wi, bi, ti, ref['dWi'], ref['dbi'])):
        rows = np.flatnonzero(mask)
        # the apply kernel replays from the row's `last` itself (a no-op after a correct prepass)
        _catch_up_pair(emb, bias, rows, t - 1, mutate)
        for tab, grad in ((emb, g), (bias, gb.reshape(-1, 1))):
            if 'catch_up_through_t' in mutate:       # rows already at t take step t once more
                tab._step(rows, t, grad[rows])
                tab.last[rows] = t
            else:
                tab.apply(rows, grad[rows], t)
    ref['touched_u'], ref['touched_i'] = tu, ti
    return ref
