"""Cases for the first-generation MF step under lazy-exact Adam (csrc/mf.cu launch_step with
csrc/mf_adam.cuh).

TEST INFRASTRUCTURE ONLY (tests/test_mf_adam_oracle_gpu.py, tests/test_mf_adam_oracle_cpu.py).

The minibatches come from oracle.mf_cases.make_case with the first-generation lane groups, so every
member-list length class runs, up to cap + 1 and the very hot lists mf_bwd_long_kernel<L, 0> takes.
On top of that:

* adaptive hinge draws B * n_neg negatives; interactions whose chosen negative is within 1e-4 of
  the runner-up or whose hinge argument is within 1e-3 of 0 draw theirs again;
* rating losses take ratings (regression 1..5, Poisson counts, logistic +-1) and no negatives;
* ``seed_state`` gives the Adam state a start step t0: at t0 = 1 it is zero; at t0 > 1 exp_avg and
  exp_avg_sq are of the size the case's gradients give, and the rows fall in four groups by
  ``last``: current (t0 - 1), one step behind, far behind (up to t0 - 2 steps) and never touched
  (last = 0, exp_avg = exp_avg_sq = 0).
"""

import numpy as np

from oracle import explicit as oex
from oracle import mf_cases as mc
from oracle.adam import LazyAdamTable, mf_terms

TABLES = ('Wu', 'Wi', 'bu', 'bi')
IMPLICIT = ('pointwise', 'bpr', 'hinge', 'adaptive_hinge')
EXPLICIT = oex.LOSSES


def fwd_small_limit(sms):
    """mf_fwd_tile_kernel takes its 8-interaction tiles while B < this."""
    return sms * 36 * 32


def bwd_small_limit(sms):
    """mf_bwd_tile_kernel takes its 8-segment tiles while 2B < this."""
    return sms * 24 * 32


def make_case(D, B, loss, n_neg=1, seed=0, sms=132):
    """make_case's dict with ``loss``, ``n_neg`` and, for a rating loss, ``ratings`` (negs None)."""
    base = {'adaptive_hinge': 'hinge'}.get(loss, loss if loss in mc.LOSSES else 'pointwise')
    case = mc.make_case(D, B, base, seed, sms=sms, first_gen=True)
    case['loss'], case['n_neg'] = loss, (n_neg if loss == 'adaptive_hinge' else 1)
    rs = np.random.RandomState(seed + 1)
    if loss in EXPLICIT:
        B = len(case['users'])
        case['ratings'] = {'regression': lambda: rs.randint(1, 6, B),
                           'poisson': lambda: rs.poisson(1.5, B),
                           'logistic': lambda: rs.choice([-1.0, 1.0], B)}[loss]().astype(np.float32)
        case['negs'] = None
    elif loss == 'adaptive_hinge':
        B = len(case['users'])
        case['negs'] = np.r_[case['negs'], rs.randint(0, case['I'], B * (n_neg - 1))].astype(np.int64)
        _separate_adaptive(case, rs)
    return case


def _separate_adaptive(case, rs):
    B, n = len(case['users']), case['n_neg']
    P = mc.tables64(case)
    for _ in range(100):
        ref = mf_terms(P, case['users'], case['items'], case['negs'], 'adaptive_hinge', n)
        neg = np.sort(ref['neg'], axis=0)
        z = neg[-1] - ref['pos'] + 1.0
        bad = np.abs(z) < 1e-3
        if n > 1:
            bad |= neg[-1] - neg[-2] < 1e-4
        if not bad.any():
            return
        for b in np.flatnonzero(bad):
            case['negs'][np.arange(n) * B + b] = rs.randint(0, case['I'], n)
    raise ValueError('could not separate the adaptive hinge scores')


def tables(case, lr, wd, state=None):
    """[Wu, Wi, bu, bi] float64 LazyAdamTables of the case, with ``seed_state``'s state."""
    tabs = [LazyAdamTable(case[k].astype(np.float64), lr=lr, weight_decay=wd) for k in TABLES]
    if state is not None:
        for k, tab in enumerate(tabs):
            m, v, last = state[k]
            tab.m, tab.v, tab.last = m.astype(np.float64), v.astype(np.float64), last.astype(np.int64)
    return tabs


def seed_state(case, t0, seed=0):
    """Four (exp_avg, exp_avg_sq, last) float32 / int32 triples for a state at step t0 - 1 (see the
    module docstring); a bias has its embedding's ``last``.  The rows of the case's fixed
    interactions (the hinge tie) are current, so that step t0 reads them as built."""
    rs = np.random.RandomState(seed)
    P = mc.tables64(case)
    out = []
    if t0 == 1:
        for p in P:
            out.append((np.zeros(p.shape, np.float32), np.zeros(p.shape, np.float32), np.zeros(p.shape[0], np.int32)))
        return out
    ref = mf_terms(P, case['users'], case['items'], case['negs'], case['loss'], case['n_neg'], case.get('ratings'))
    grads = (ref['dWu'], ref['dWi'], ref['dbu'], ref['dbi'])
    fixed = np.flatnonzero(case['fixed'])
    keep = (case['users'][fixed], np.r_[case['items'][fixed]] if case['negs'] is None
            else np.r_[case['items'][fixed], case['negs'][fixed]])
    lasts = []
    for side in range(2):
        n = P[side].shape[0]
        group = rs.randint(0, 4, n)
        group[keep[side]] = 0
        last = np.select([group == 0, group == 1, group == 2],
                         [t0 - 1, max(t0 - 2, 0), rs.randint(1, max(t0 - 2, 2), n)], 0)
        lasts.append((last.astype(np.int32), group == 3))
    for k, (p, g) in enumerate(zip(P, grads)):
        last, never = lasts[k % 2]
        gs = np.abs(g).max()
        m = rs.randn(*p.shape) * 0.5 * gs
        v = gs * gs * rs.uniform(0.25, 1.0, p.shape)
        m[never], v[never] = 0.0, 0.0
        out.append((m.astype(np.float32), v.astype(np.float32), last.copy()))
    return out


def batches(case, steps, seed=0):
    """``steps`` minibatches (users, items, negs or None, ratings or None): the first is the whole
    case; each later one a random quarter of its interactions (not the fixed ones), so that rows
    miss steps between touches."""
    B, n = len(case['users']), case['n_neg']
    rs = np.random.RandomState(seed)
    out = [(case['users'], case['items'], case['negs'], case.get('ratings'))]
    free = np.flatnonzero(~case['fixed'])
    for _ in range(steps - 1):
        idx = np.sort(rs.choice(free, max(1, B // 4), replace=False))
        negs = None if case['negs'] is None else case['negs'].reshape(n, B)[:, idx].reshape(-1)
        ratings = None if case.get('ratings') is None else case['ratings'][idx]
        out.append((case['users'][idx], case['items'][idx], negs, ratings))
    return out


# ---- the GPU test's matrix (tests/test_mf_adam_oracle_gpu.py), shared with the CPU mutation test -----
DIMS = (4, 8, 12, 16, 24, 32, 64, 100, 128, 256, 260)
LOSS_N = (('pointwise', 1), ('bpr', 1), ('hinge', 1), ('adaptive_hinge', 2), ('adaptive_hinge', 5),
          ('regression', 1), ('poisson', 1), ('logistic', 1))
# every D twice with small batches, the losses cycling; weight decay and t0 alternate: (D, loss, n_neg, wd, t0)
SMALL = [(D, ) + LOSS_N[(2 * k + s) % len(LOSS_N)] + ((0.0, 0.1)[(k + s) % 2], (1, 1000)[(k // 2 + s) % 2])
         for k, D in enumerate(DIMS) for s in (0, 1)]
# 2B above the backward-tile threshold
LARGE = [(4, 'hinge', 1, 0.1, 1000), (12, 'adaptive_hinge', 5, 0.0, 1000), (24, 'regression', 1, 0.1, 1000),
         (64, 'bpr', 1, 0.0, 1), (100, 'logistic', 1, 0.1, 1), (260, 'pointwise', 1, 0.1, 1)]


def small_case(D, loss, n, sms=132):
    return make_case(D, 3001 + D, loss, n, seed=D + 17 * n + len(loss), sms=sms)


def large_case(D, loss, n, sms=132):
    return make_case(D, bwd_small_limit(sms) // 2 + 1001, loss, n, seed=D + 5, sms=sms)
