"""Planned-step test cases (csrc/mf_v2.cuh) with controlled member-list lengths.

TEST INFRASTRUCTURE ONLY (tests/test_mf_planned_oracle_gpu.py, tests/test_mf_planned_oracle_cpu.py).

Each member-list length class of the planned step is a separate code path, so ``make_case``
builds the minibatch from prescribed list lengths instead of hoping random ids hit them:

* user lists (interactions of one user) of length 1, 2, 3..16, 17..cap, exactly cap, cap + 1 and
  one very hot list whose length is not a multiple of the long kernels' lane groups;
* item lists (positive and negative terms on one item row) of length 1..4 (held in registers),
  5..8, 9 (a chunk of 8 and a remainder), 10..16, 17..cap, cap, cap + 1 and one very hot list;
* an interaction whose positive and negative are the same item, and the ids 0, U - 1 and I - 1.

The rest of the batch is filler: users and items drawn uniformly from pools sized for short
lists (most users have one or two interactions, as in a uniform batch).  Scores stay within
+-8 for the sigmoid losses; hinge cases have 20-80 % of the interactions active with |z| >= 1e-3,
one interaction exactly at z = 0 (a zero user row and dyadic biases) and one user whose
interactions are all inactive, on item rows nothing else touches.  ``check_properties``
verifies all of this on the oracle's result.
"""

import numpy as np

from oracle import mf as omf


def lpr_for_dim(D):
    """Lanes per row of the first-generation kernels (mf.cu lpr_for_dim)."""
    l, p = D // 4, 1
    if l >= 32:
        return 32
    while p < l:
        p <<= 1
    return p


def seg_sort_cap(D):
    """Longest member list the tile kernels handle; longer lists are hot (segindex.cuh)."""
    G = lpr_for_dim(D)
    return 128 if G >= 8 else (64 if G >= 4 else 16 * G)


def long_groups(D, first_gen=False):
    """Lane groups per CTA of mf_user_long_kernel / mf_item_long_kernel (LPR = D / 4), or with
    ``first_gen`` of the first-generation step's mf_bwd_long_kernel (LPR = lpr_for_dim(D))."""
    return 256 // (lpr_for_dim(D) if first_gen else D // 4)


def small_limit(sms):
    """mf_user_kernel runs its small-batch variant while B < this, mf_item_kernel while 2B < this."""
    return sms * 24 * 32


LOSSES = ('pointwise', 'bpr', 'hinge')


def small_case(D, loss, sms=132):
    """The matrix's small-batch case: both tile kernels take their small variant."""
    return make_case(D, 3001 + D, loss, seed=D + 7 * LOSSES.index(loss), sms=sms)


def large_case(D, loss, sms=132):
    """The matrix's large-batch case: B above the user kernel's threshold (and so 2B above the
    item kernel's)."""
    return make_case(D, small_limit(sms) + 1001, loss, seed=100 + D + LOSSES.index(loss), sms=sms)


def very_hot_length(D, first_gen=False):
    """Longer than cap + 1, and not a multiple of the long kernels' lane groups."""
    G = long_groups(D, first_gen)
    return (seg_sort_cap(D) // G + 2) * G + 5


def _user_lengths(D, rs, hot, extra_hot, first_gen=False):
    cap = seg_sort_cap(D)
    if cap >= 19:
        lens = [1] * 4 + [2] * 4 + list(range(3, 17)) + [17, int(rs.randint(18, cap)), cap - 1, cap]
    else:                   # cap 16 (LPR 1): no 17..cap class
        lens = [1] * 4 + [2] * 4 + list(range(3, cap + 1))
    if hot:
        lens += [cap + 1, very_hot_length(D, first_gen)]
    G = long_groups(D, first_gen)
    lens += [cap + 1 + int(rs.randint(0, 2 * G)) for _ in range(extra_hot)]
    return lens


def _item_lengths(D, rs, hot, first_gen=False):
    cap = seg_sort_cap(D)
    if cap >= 19:
        lens = [1, 2, 3, 4] * 2 + [5, 6, 7, 8] + [9] + list(range(10, 17)) + [17, int(rs.randint(18, cap)),
                                                                              cap - 1, cap]
    else:
        lens = [1, 2, 3, 4] * 2 + [5, 6, 7, 8] + [9] + list(range(10, cap + 1))
    if hot:
        lens += [cap + 1, very_hot_length(D, first_gen)]
    return lens


def _ids(n, forced, rs):
    """A random id for each of n lists, with forced[k] = id pinned for list k."""
    free = np.setdiff1d(np.arange(n), list(forced.values()))
    rs.shuffle(free)
    out = np.empty(n, dtype=np.int64)
    rest = [k for k in range(n) if k not in forced]
    out[rest] = free
    for k, v in forced.items():
        out[k] = v
    return out


def make_case(D, B, loss, seed, sms=132, hot=True, extra_hot_users=0, min_users=0, first_gen=False):
    """One minibatch of B interactions at dimension D: dict(D, B, loss, U, I, Wu, Wi, bu, bi,
    users, items, negs, cap, hot, fixed) with float32 tables and int64 ids.  ``fixed`` marks the
    interactions that carry a prescribed edge (same item, hinge tie, inactive user).
    ``extra_hot_users`` adds that many more users with cap + 1 .. cap + 2G interactions, and
    ``min_users`` pads the user table so that ids spread over many scan tiles.  ``first_gen``:
    the very hot lists are sized for the lane groups of the first-generation step's long kernel
    (any D that is a multiple of 4) instead of the planned step's."""
    rs = np.random.RandomState(seed)
    cap = seg_sort_cap(D)
    hinge = loss == 'hinge'
    ulens = _user_lengths(D, rs, hot, extra_hot_users, first_gen)
    nb = len(ulens) - extra_hot_users        # the last two prescribed lists get ids 0 and U - 1
    ilens = _item_lengths(D, rs, hot, first_gen)
    n_ded = 4 if hinge else 0                 # dedicated hinge interactions: 1 tie + 3 inactive
    Bf = B - n_ded
    if Bf < sum(ulens) or 2 * Bf < sum(ilens) + 2:
        raise ValueError('B = %d is too small for the list classes at D = %d' % (B, D))

    # users: prescribed lists, then filler from a pool (most filler users get 1 or 2)
    fill_u = Bf - sum(ulens)
    pool_u = max(1, int(fill_u * 1.3))
    nu_struct = len(ulens)
    U = max(nu_struct + pool_u + (2 if hinge else 0), min_users)
    uid = _ids(U, {nb - 1: 0, nb - 2: U - 1}, rs)                 # uid[k]: id of prescribed list k, then pool, then dedicated
    uslots = np.concatenate([np.repeat(uid[:nu_struct], ulens),
                             uid[nu_struct + rs.randint(0, pool_u, fill_u)]]).astype(np.int64)
    rs.shuffle(uslots)

    # items: prescribed term counts, filler from a pool; slot 2b is the positive, 2b + 1 the negative
    fill_i = 2 * Bf - sum(ilens)
    pool_i = max(1, fill_i // 2)
    ni_struct = len(ilens)
    I = ni_struct + pool_i + (8 if hinge else 0)
    iid = _ids(I, {ni_struct - 1: I - 1, 2: 0}, rs)
    islots = np.concatenate([np.repeat(iid[:ni_struct], ilens),
                             iid[ni_struct + rs.randint(0, pool_i, fill_i)]]).astype(np.int64)
    rs.shuffle(islots)
    # one interaction scores the same item as its positive and its negative (multiset kept)
    X = iid[ilens.index(6)]
    a, b = np.flatnonzero(islots == X)[:2]
    other = a + 1 if a % 2 == 0 else a - 1
    islots[b], islots[other] = islots[other], islots[b]
    same = a // 2
    users, items, negs = uslots, islots[0::2].copy(), islots[1::2].copy()
    fixed = np.zeros(Bf, dtype=bool)
    fixed[same] = True

    # tables: dots ~ N(0, sigma^2) (sigmoid arguments well inside +-8; hinge 20-80 % active)
    sigma = 1.5 if hinge else 1.0
    se = np.sqrt(sigma) / D ** 0.25
    Wu = rs.randn(U, D) * se
    Wi = rs.randn(I, D) * se
    bu = rs.randn(U, 1) * 0.1
    bi = rs.randn(I, 1) * 0.1
    case = dict(D=D, B=B, loss=loss, U=U, I=I, cap=cap, hot=hot, sms=sms, same=int(same), first_gen=first_gen)
    if hinge:
        # tie: zero user row, pos = 0.25 + 0.75, neg = 0.25 - 0.25, z = neg - pos + 1 = 0 exactly
        tu, iu = uid[nu_struct + pool_u], uid[nu_struct + pool_u + 1]
        ded = iid[ni_struct + pool_i:]
        Wu[tu] = 0.0
        bu[tu] = 0.25
        bi[ded[0]], bi[ded[1]] = 0.75, -0.25
        # inactive: small rows, positives lifted, negatives lowered -> z ~ -3 on rows nobody else has
        Wi[ded[2:]] *= 0.1
        bi[ded[2:5]], bi[ded[5:8]] = 2.0, -2.0
        users = np.concatenate([users, [tu, iu, iu, iu]])
        items = np.concatenate([items, [ded[0], ded[2], ded[3], ded[4]]])
        negs = np.concatenate([negs, [ded[1], ded[5], ded[6], ded[7]]])
        fixed = np.concatenate([fixed, [True] * 4])
        case.update(tie=Bf, inactive_user=int(iu), inactive_items=ded[2:].copy())
    case.update(Wu=Wu.astype(np.float32), Wi=Wi.astype(np.float32), bu=bu.astype(np.float32),
                bi=bi.astype(np.float32), users=users.astype(np.int64), items=items.astype(np.int64),
                negs=negs.astype(np.int64), fixed=fixed)
    _separate_scores(case, rs)
    return case


def _args(case, idx=slice(None)):
    """Float64 scores of the interactions idx: (pos, neg)."""
    P = [case[k].astype(np.float64) for k in ('Wu', 'Wi', 'bu', 'bi')]
    u, i, j = case['users'][idx], case['items'][idx], case['negs'][idx]
    return (omf.bilinear_scores(*P, u, i, np.float64), omf.bilinear_scores(*P, u, j, np.float64))


def _bad(case, pos, neg):
    if case['loss'] == 'hinge':
        return np.abs(neg - pos + 1.0) < 1e-3
    if case['loss'] == 'bpr':
        return np.abs(pos - neg) > 8.0
    return np.maximum(np.abs(pos), np.abs(neg)) > 8.0


def _separate_scores(case, rs):
    """Swap the negatives of interactions whose score sits at a hinge boundary (|z| < 1e-3) or
    outside the sigmoids' +-8 with those of random other interactions: list lengths stay."""
    free = np.flatnonzero(~case['fixed'])
    for _ in range(100):
        pos, neg = _args(case)
        bad = np.flatnonzero(_bad(case, pos, neg) & ~case['fixed'])
        if len(bad) == 0:
            return
        other = free[rs.randint(0, len(free), len(bad))]
        negs = case['negs']
        for k, m in zip(bad, other):
            negs[k], negs[m] = negs[m], negs[k]
    raise ValueError('could not separate the scores of case %r' % ((case['D'], case['B'], case['loss']),))


def member_lengths(case):
    """The list lengths the plan builds: dict(user=..., item=...) over touched rows; item lists
    count the positive and the negative terms."""
    lu = np.bincount(case['users'], minlength=case['U'])
    li = np.bincount(np.concatenate([case['items'], case['negs']]), minlength=case['I'])
    return dict(user=lu[lu > 0], item=li[li > 0])


def length_classes(D, hot=True):
    """(name, lo, hi) inclusive ranges every case must contain, per side."""
    cap = seg_sort_cap(D)
    user = [('1', 1, 1), ('2', 2, 2), ('3-16', 3, 16), ('17-cap', 17, cap - 1), ('cap', cap, cap)]
    item = [('1-4', 1, 4), ('5-8', 5, 8), ('9', 9, 9), ('10-16', 10, 16), ('17-cap', 17, cap - 1),
            ('cap', cap, cap)]
    if cap < 19:                      # cap 16: 3..16 reaches the cap
        user = [c for c in user if c[0] != '17-cap']
        item = [c for c in item if c[0] != '17-cap']
    if hot:
        user.append(('cap+1', cap + 1, cap + 1))
        item.append(('cap+1', cap + 1, cap + 1))
    return dict(user=user, item=item)


def check_properties(case, ref):
    """Problems (an empty list when none) of the case's scales on the oracle result ``ref``
    (oracle.mf.fused_step's dict: pos, neg, gp, gn)."""
    out = []
    D, cap, G = case['D'], case['cap'], long_groups(case['D'], case.get('first_gen', False))
    lens = member_lengths(case)
    for side, classes in length_classes(D, case['hot']).items():
        for name, lo, hi in classes:
            if not ((lens[side] >= lo) & (lens[side] <= hi)).any():
                out.append('no %s list of length %s' % (side, name))
        if case['hot'] and not ((lens[side] > cap + 1) & (lens[side] % G != 0)).any():
            out.append('no very hot %s list' % side)
        if not case['hot'] and (lens[side] > cap).any():
            out.append('a hot %s list in a case without hot rows' % side)
    if not (case['items'] == case['negs']).any():
        out.append('no interaction with the same positive and negative')
    for what, ids, n in (('user', case['users'], case['U']), ('item', np.r_[case['items'], case['negs']], case['I'])):
        if not (np.isin(0, ids) and np.isin(n - 1, ids)):
            out.append('%s ids 0 and %d not both present' % (what, n - 1))
    pos, neg = ref['pos'], ref['neg']
    if case['loss'] == 'hinge':
        z = neg - pos + 1.0
        act = (z >= 0).mean()
        if not 0.2 <= act <= 0.8:
            out.append('hinge activity %.2f outside 20-80 %%' % act)
        tie = case['tie']
        rest = np.ones(len(z), dtype=bool)
        rest[tie] = False
        if (np.abs(z[rest]) < 1e-3).any():
            out.append('hinge |z| < 1e-3')
        P32 = [case[k] for k in ('Wu', 'Wi', 'bu', 'bi')]
        u, i, j = case['users'][tie:tie + 1], case['items'][tie:tie + 1], case['negs'][tie:tie + 1]
        z32 = omf.bilinear_scores(*P32, u, j) - omf.bilinear_scores(*P32, u, i) + np.float32(1.0)
        if z[tie] != 0.0 or z32[0] != 0.0:
            out.append('tie interaction not at z = 0 in both precisions')
        mine = case['users'] == case['inactive_user']
        if (ref['gp'][mine] != 0).any() or (ref['gn'][mine] != 0).any():
            out.append('inactive user has an active interaction')
        others = np.r_[case['items'][~mine], case['negs'][~mine]]
        if np.isin(case['inactive_items'], others).any():
            out.append('inactive user shares an item row')
    else:
        arg = np.abs(pos - neg) if case['loss'] == 'bpr' else np.maximum(np.abs(pos), np.abs(neg))
        if arg.max() > 8.0:
            out.append('sigmoid argument %.2f beyond 8' % arg.max())
        if (ref['gp'] == 0).any() or (ref['gn'] == 0).any():
            out.append('a score gradient is 0')
    return out


def tables64(case):
    return [case[k].astype(np.float64) for k in ('Wu', 'Wi', 'bu', 'bi')]


def hparams(case, opt, wd_on, seed=0):
    """(lr, weight_decay, initial states) that make one step measure the gradient at 1e-5:
    SGD lr = 0.3 / max|g|; Adagrad accumulators ~ max|g|^2 per table, lr = half the largest
    weight, so that lr g / sqrt(s) is a sizeable part of the weights; wd = 0.5 max|g| / max|w|."""
    P = tables64(case)
    ref = omf.fused_step([p.copy() for p in P], case['users'], case['items'], case['negs'], case['loss'],
                         'sgd', 0.0)
    grads = (ref['dWu'], ref['dWi'], ref['dbu'], ref['dbi'])
    gmax = max(np.abs(ref['dWu']).max(), np.abs(ref['dWi']).max())
    wmax = max(np.abs(P[0]).max(), np.abs(P[1]).max())
    wd = 0.5 * gmax / wmax if wd_on else 0.0
    if opt == 'sgd':
        return 0.3 / gmax, wd, None
    rs = np.random.RandomState(seed)
    states = [(np.abs(g).max() ** 2 * rs.uniform(0.5, 1.5, g.shape)).astype(np.float32) for g in grads]
    return 0.5 * wmax, wd, states
