"""Explicit-feedback (rating) cases of the hashed-table MF step (csrc/mf.cu
slb_mf_bloom_train_step with a rating loss, mf_fwd_bloom_rating_kernel).

TEST INFRASTRUCTURE ONLY (tests/test_explicit_bloom_gpu.py, tests/test_explicit_bloom_oracle_cpu.py).

The ids and tables come from ``oracle.bloom_cases.make_case``, so a case carries what the
pairwise cases do: the padding id, real ids on row 0 and on the frozen row, an id with two hashes
on one row, hot item rows with exactly cap / cap + 1 / many terms (positives only, so a rating
loss keeps those counts), a hot user, and bias ids equal modulo the hash-bucket count.  Ratings
replace the negatives: 1..5 (regression), 0..3 (poisson), {-1, 0, 0.25, 1} (logistic: -1 is
clamped to 0).  ``check_properties`` verifies the promises on the rating oracle (oracle/explicit_bloom.py).
"""

import numpy as np

from oracle import bloom as ob
from oracle import bloom_cases as bc
from oracle import explicit_bloom as oeb

DIMS = (4, 8, 12, 20, 32, 64, 100, 128, 256)
HASHES = ((0, 3), (2, 0), (2, 3), (0, 24))
LOSSES = ('regression', 'poisson', 'logistic')
PADS = (0, 3, -1)


def ratings(loss, rs, n):
    if loss == 'regression':
        return rs.randint(1, 6, n).astype(np.float32)
    if loss == 'poisson':
        return rs.randint(0, 4, n).astype(np.float32)
    return rs.choice(np.array([-1.0, 0.0, 0.25, 1.0], dtype=np.float32), n)


def make_case(D, loss, Hu, Hi, pad, seed, B=None, hot=True):
    """One rating minibatch: bloom_cases.make_case's dict with ``loss``, ``ratings`` and
    ``negs=None``."""
    case = bc.make_case(D, 'pointwise', Hu, Hi, pad, seed, B=B, hot=hot)
    case.update(loss=loss, negs=None, ratings=ratings(loss, np.random.RandomState(seed + 1), case['B']))
    return case


def bias_buckets(B):
    """Hash-bucket count of the rating step's bias update (B pairs): the smallest power of two
    >= max(4096, 2B)."""
    nb = 4096
    while nb < 2 * B:
        nb <<= 1
    return nb


def step(case, P=None, opt=None, lr=0.0, weight_decay=0.0, states=None, norm=None, mutate=()):
    """The rating-mode oracle on ``case`` (tables from the case unless ``P`` is given)."""
    P = bc.tables64(case) if P is None else P
    return oeb.step(P, case['users'], case['items'], case['ratings'], case['loss'], case['Hu'], case['Hi'],
                    case['pad_u'], case['pad_i'], opt, lr, weight_decay, 1e-10, states, norm, mutate)


def term_counts(case, ref):
    """Members per table row as the kernel's segment index counts them (terms with g != 0)."""
    Mu, Mi = case['Wu'].shape[0], case['Wi'].shape[0]
    nu_, ni_ = max(case['Hu'], 1), max(case['Hi'], 1)
    a = ref['gs'] != 0
    cu, ci = np.zeros(Mu, dtype=np.int64), np.zeros(Mi, dtype=np.int64)
    np.add.at(cu, ob.table_rows(case['users'][a], case['Hu'], Mu, case['pad_u']).reshape(-1), ni_)
    np.add.at(ci, ob.table_rows(case['items'][a], case['Hi'], Mi, case['pad_i']).reshape(-1), nu_)
    return dict(user=cu, item=ci)


def check_properties(case, ref):
    """Problems (an empty list when none) of the case on the rating oracle's result."""
    out = []
    cap = case['cap']
    if (ref['gs'] == 0).any():
        out.append('an interaction with g == 0')
    if len(case['hot_items']):
        cnt = term_counts(case, ref)
        Mi = case['Wi'].shape[0]
        for x, want in zip(case['hot_items'], case['hot_expected']):
            rows = ob.table_rows([x], case['Hi'], Mi, case['pad_i']).reshape(-1)
            if (cnt['item'][rows] != want).any():
                out.append('hot item %d rows have %s terms, not %d' % (x, cnt['item'][rows], want))
        lo, hi, _ = case['hot_expected']
        if not lo <= cap < hi:
            out.append('hot counts %s do not straddle cap %d' % (case['hot_expected'], cap))
        if cnt['user'].max() <= cap:
            out.append('no hot user row')
    nb = bias_buckets(case['B'])
    for side, H, ids in (('user', case['Hu'], case['users']), ('item', case['Hi'], case['items'])):
        pad = case['pad_u'] if side == 'user' else case['pad_i']
        M = case['Wu' if side == 'user' else 'Wi'].shape[0]
        if H:
            r = ob.table_rows(ids, H, M, pad)
            real = ids != pad
            if pad >= 0 and not (ids == pad).any():
                out.append('%s padding id absent' % side)
            if not (r[real] == 0).any():
                out.append('no real %s id on row 0' % side)
            if pad > 0 and not (r[real] == pad).any():
                out.append('no real %s id on the frozen row' % side)
            if H >= 2 and not any(len(set(x)) < H for x in r):
                out.append('no %s id with two hashes on one row' % side)
        u = np.unique(ids)
        if len(u) == len(np.unique(u & (nb - 1))):
            out.append('no %s bias ids equal mod %d' % (side, nb))
    if np.abs(ref['pos']).max() > 8.0:
        out.append('score %.2f beyond 8' % np.abs(ref['pos']).max())
    return out


def hparams(case, opt, wd_on, seed=0):
    """(lr, weight_decay, initial states) that make one step measure the gradient at 1e-5, as
    oracle.bloom_cases.hparams, from the rating-mode gradients."""
    P = bc.tables64(case)
    ref = step(case)
    gmax = max(np.abs(ref['dWu']).max(), np.abs(ref['dWi']).max())
    wmax = max(np.abs(P[0]).max(), np.abs(P[1]).max())
    wd = 0.5 * gmax / wmax if wd_on else 0.0
    if opt == 'sgd':
        return 0.3 / gmax, wd, None
    rs = np.random.RandomState(seed)
    grads = (ref['dWu'], ref['dWi'], ref['dbu'], ref['dbi'])
    states = [(max(np.abs(g).max(), gmax * 1e-3) ** 2 * rs.uniform(0.5, 1.5, g.shape)).astype(np.float32)
              for g in grads]
    return 0.5 * wmax, wd, states


def matrix():
    """(D, loss, Hu, Hi, pad, seed) of the suite: every D with each loss, hash counts and padding
    cycling."""
    out = []
    for a, D in enumerate(DIMS):
        for b, loss in enumerate(LOSSES):
            Hu, Hi = HASHES[(a + b) % len(HASHES)]
            out.append((D, loss, Hu, Hi, PADS[(a + 2 * b) % 3], 3000 + 10 * a + b))
    return out


def case_for(D, loss, Hu, Hi, pad, seed):
    """The suite case of one matrix entry; when the murmur search finds no id for one seed, the
    next seed is taken."""
    for s in range(seed, seed + 50 * 7919, 7919):
        try:
            return make_case(D, loss, Hu, Hi, pad, s)
        except ValueError:
            continue
    raise ValueError('no case for %r' % ((D, loss, Hu, Hi, pad, seed),))
