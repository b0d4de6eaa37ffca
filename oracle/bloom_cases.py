"""Hashed-table (Bloom) MF step test cases (csrc/mf.cu slb_mf_bloom_train_step).

TEST INFRASTRUCTURE ONLY (tests/test_mf_bloom_oracle_gpu.py, tests/test_mf_bloom_oracle_cpu.py).

The ids of a case are found by searching the murmur oracle (oracle/murmur.py), so that each case
contains what it claims to, and ``check_properties`` verifies it on the oracle's result:

* the padding id among the positives and the negatives, real ids hashing to row 0 and to row
  ``pad``, and an id with two hashes on one row (hashed sides);
* hashed or plain item rows with prescribed term counts: the largest multiple of the user side's
  hash count <= ``seg_sort_cap``, the next one above it (exactly cap and cap + 1 when the user side
  has one row per id), and a very hot row whose count is not a multiple of the long kernel's lane
  groups; the hot ids are positives whose rows nothing else names;
* bias ids equal modulo the hash-bucket count of the sparse bias update, one id repeated more than
  100 times, and (``big_ids``) a hashed id space of a few million with ids at its top;
* hinge: one interaction exactly at z = 0 (a zero user vector and dyadic biases) and one user whose
  interactions are all inactive; adaptive hinge with a plain user table: an exact tie between two
  users' negatives, so that the first maximum decides which user is credited.

Scores stay within +-8 for the sigmoid losses and |z| >= 1e-3 for the hinge losses (the tie aside).
"""

import numpy as np

from oracle import bloom as ob
from oracle.mf_cases import lpr_for_dim, seg_sort_cap

DIMS = (4, 8, 12, 20, 24, 32, 48, 64, 100, 128, 256)
HASHES = ((0, 1), (0, 4), (0, 24), (2, 3), (3, 0), (0, 0))
LOSSES = (('pointwise', 1), ('bpr', 1), ('hinge', 1), ('adaptive_hinge', 2), ('adaptive_hinge', 5))
PADS = (0, 3, -1)


def long_groups(D):
    """Lane groups per CTA of mf_bwd_long_kernel (256 / LPR)."""
    return 256 // lpr_for_dim(D)


def very_hot_count(D):
    """Longer than cap + 1, and not a multiple of the long kernel's lane groups."""
    G = long_groups(D)
    return (seg_sort_cap(D) // G + 2) * G + 5


class _Ids:
    """An id space [0, N) of one side with its table (plain, or H hashes into M rows)."""

    def __init__(self, N, H, M, pad, rs):
        self.N, self.H, self.M, self.pad, self.rs = N, H, M, pad, rs
        self.used = set()

    def rows(self, ids):
        return ob.table_rows(np.asarray(ids, dtype=np.int64), self.H, self.M, self.pad)

    def search(self, cond, k=1, avoid_rows=(), lo=0):
        """k fresh ids (not the padding id) whose rows satisfy ``cond`` and avoid ``avoid_rows``."""
        out = []
        avoid = np.asarray(sorted(avoid_rows), dtype=np.int64)
        for _ in range(200):
            cand = self.rs.randint(lo, self.N, 4096).astype(np.int64)
            r = self.rows(cand)
            ok = cond(r) & ~np.isin(r, avoid).any(axis=1) & (cand != self.pad)
            for c in cand[ok]:
                if int(c) not in self.used and int(c) not in out:
                    out.append(int(c))
                if len(out) == k:
                    self.used.update(out)
                    return out
        raise ValueError('no id found')


def make_case(D, loss, Hu, Hi, pad, seed, n_neg=1, B=None, big_ids=False, hot=True):
    """One minibatch: dict(D, B, loss, n_neg, Hu, Hi, pad, NU, NI, Wu, Wi, bu, bi, users, items, negs,
    cap, hot_items, ...) with float32 tables and int64 ids."""
    rs = np.random.RandomState(seed)
    cap = seg_sort_cap(D)
    hinge = loss in ('hinge', 'adaptive_hinge')
    n = n_neg if loss == 'adaptive_hinge' else 1
    nu_, ni_ = max(Hu, 1), max(Hi, 1)
    # item slots of the hot ids: their rows get slots * nu_ terms (positives only)
    lo_cnt = (cap // nu_) * nu_
    hot_slots = [cap // nu_, cap // nu_ + 1, very_hot_count(D)] if hot else []
    B = B or max(1200, 2 * sum(hot_slots) + 400 + 3 * cap)
    nb = ob.bias_buckets(B)
    big = 3_000_000 + seed
    NU = big if (big_ids and Hu) else max(nb + 64, B)
    NI = big if (big_ids and Hi) else max(nb + 64, B)
    Mu = max(61, (2 * B * Hu) // 3) | 1 if Hu else NU
    Mi = max(61, (2 * B * Hi) // 3) | 1 if Hi else NI
    if pad >= 0:
        Mu, Mi = max(Mu, pad + 1), max(Mi, pad + 1)
    U, I = _Ids(NU, Hu, Mu, pad, rs), _Ids(NI, Hi, Mi, pad, rs)
    case = dict(D=D, B=B, loss=loss, n_neg=n, Hu=Hu, Hi=Hi, pad=pad, NU=NU, NI=NI, cap=cap,
                pad_u=pad if Hu else -1, pad_i=pad if Hi else -1)

    # hot item ids: all rows distinct, away from row 0 / pad and from each other
    def distinct(r):
        return np.array([len(set(x)) == r.shape[1] for x in r]) & ~np.isin(r, [0, max(pad, 0)]).any(axis=1)
    hot_ids, hot_rows = [], set()
    for _ in hot_slots:
        x = I.search(distinct, 1, hot_rows)[0]
        hot_ids.append(x)
        hot_rows.update(I.rows([x]).reshape(-1).tolist())
    case['hot_items'] = np.array(hot_ids, dtype=np.int64)
    case['hot_counts'] = np.array([s * nu_ for s in hot_slots], dtype=np.int64)
    case['hot_expected'] = [lo_cnt, lo_cnt + nu_, very_hot_count(D) * nu_] if hot else []

    # special ids per side: padding id, ids on row 0 / row pad, an id with a repeated row,
    # bucket twins (equal mod nb) and the top of the id space
    def specials(S):
        out = []
        if S.H:
            if 0 <= pad < S.N:
                out.append(pad)
            out += S.search(lambda r: (r == 0).any(axis=1), 1, hot_rows if S is I else ())
            if pad > 0:
                out += S.search(lambda r: (r == pad).any(axis=1), 1, hot_rows if S is I else ())
            if S.H >= 2:
                out += S.search(lambda r: np.array([len(set(x)) < len(x) for x in r]), 1,
                                hot_rows if S is I else ())
        else:
            out += [0]
        for _ in range(1000):
            base = int(S.rs.randint(0, min(nb, S.N - nb)))
            twins = [base + k * nb for k in range(3) if base + k * nb < S.N]
            if any(t in S.used or t == pad for t in twins):
                continue
            if S is I and np.isin(I.rows(twins), list(hot_rows)).any():
                continue
            break
        out += twins
        top = [S.N - 1, S.N - 2]
        out += [t for t in top if S is not I or not np.isin(I.rows([t]), list(hot_rows)).any()]
        S.used.update(out)
        return out, twins
    su, twins_u = specials(U)
    si, twins_i = specials(I)
    case['twins_u'], case['twins_i'] = twins_u, twins_i

    # filler pools (items avoid the hot rows)
    pool_u = np.array(U.search(lambda r: np.ones(len(r), dtype=bool), max(8, B // 3)), dtype=np.int64)
    pool_i = np.array(I.search(lambda r: np.ones(len(r), dtype=bool), max(8, B // 2), hot_rows), dtype=np.int64)
    items = list(np.repeat(hot_ids, hot_slots)) + list(si) * 2
    items += list(pool_i[rs.randint(0, len(pool_i), B - len(items))])
    items = np.array(items, dtype=np.int64)
    rs.shuffle(items)
    # a hot user: its rows get more than cap terms, whichever sides are active
    hot_u = U.search(lambda r: np.ones(len(r), dtype=bool), 1)[0] if hot else None
    hu_slots = (3 * cap if hinge else cap + 1) if hot else 0
    users = np.concatenate([np.array(su, dtype=np.int64).repeat(2), np.full(hu_slots, hot_u, dtype=np.int64),
                            pool_u[rs.randint(0, len(pool_u), B - 2 * len(su) - hu_slots)]])
    rs.shuffle(users)
    negs = np.concatenate([np.array(si, dtype=np.int64), pool_i[rs.randint(0, len(pool_i), B * n - len(si))]])
    rs.shuffle(negs)

    # tables: dot ~ N(0, sigma^2) whatever the hash counts
    sigma = 1.5 if hinge else 1.0
    Wu = rs.randn(Mu, D) * np.sqrt(sigma) / D ** 0.25 / np.sqrt(nu_)
    Wi = rs.randn(Mi, D) * np.sqrt(sigma) / D ** 0.25 / np.sqrt(ni_)
    bu = rs.randn(NU, 1) * 0.1
    bi = rs.randn(NI, 1) * 0.1
    fixed = np.zeros(B, dtype=bool)
    if hinge:
        bi[hot_ids] = -8.0                 # hot interactions active: every hot term has g != 0
    if loss == 'hinge':
        # tie at z = 0: a user whose vector is zero, pos = 0.25 + 0.75, neg = 0.25 - 0.25; and a
        # user whose interactions are all inactive (positives lifted, negatives lowered)
        taken = set(U.rows(pool_u).reshape(-1).tolist()) | set(U.rows(su).reshape(-1).tolist())
        tu, iu = U.search(lambda r: np.ones(len(r), dtype=bool), 2, taken | {0, max(pad, 0)})
        Wu[U.rows([tu]).reshape(-1)] = 0.0
        ti = I.search(lambda r: np.ones(len(r), dtype=bool), 8, hot_rows)
        bu[tu] = 0.25
        bi[ti[0]], bi[ti[1]] = 0.75, -0.25
        bi[ti[2:5]], bi[ti[5:8]] = 5.0, -5.0
        plain = np.flatnonzero(~np.isin(users, su + [hot_u]) & ~np.isin(items, hot_ids + si) & ~np.isin(negs, si))
        k = plain[:4]
        users[k] = [tu, iu, iu, iu]
        items[k] = [ti[0], ti[2], ti[3], ti[4]]
        negs[k] = [ti[1], ti[5], ti[6], ti[7]]
        fixed[k] = True
        case.update(tie=int(k[0]), inactive_user=int(iu), tie_user=int(tu))
    case.update(Wu=Wu.astype(np.float32), Wi=Wi.astype(np.float32), bu=bu.astype(np.float32),
                bi=bi.astype(np.float32), users=users.astype(np.int64), items=items.astype(np.int64),
                negs=negs.astype(np.int64), fixed=fixed)
    if loss == 'adaptive_hinge' and Hu == 0:
        _adaptive_tie(case, rs)
    _separate_scores(case, rs)
    return case


def _adaptive_tie(case, rs):
    """Two users with identical rows and biases score the same negative item of one interaction:
    an exact tie at the maximum, whichever precision."""
    B, n = case['B'], case['n_neg']
    free = np.flatnonzero(~case['fixed'])
    for b in free:
        ua, ub = b // n, (B + b) // n
        if ua == ub or case['fixed'][ua] or case['fixed'][ub]:
            continue
        a_id, b_id = case['users'][ua], case['users'][ub]
        if a_id == b_id or a_id == 0 or b_id == 0:
            continue
        if (case['users'] == b_id).sum() != 1:
            continue
        case['Wu'][b_id] = case['Wu'][a_id]
        case['bu'][b_id] = case['bu'][a_id]
        j = case['negs'][b]
        case['negs'][B + b] = j
        case['bi'][j] = 8.0
        case['fixed'][[b, ua, ub]] = True
        case['adaptive_tie'] = int(b)
        return
    raise ValueError('no adaptive tie placed')


def scores(case, mutate=()):
    P = tables64(case)
    return ob.step(P, case['users'], case['items'], case['negs'], case['loss'], case['Hu'], case['Hi'],
                   case['pad_u'], case['pad_i'], case['n_neg'], mutate=mutate)


def _bad(case, ref):
    pos, neg = ref['pos'], ref['neg'].reshape(case['n_neg'], -1)
    if case['loss'] in ('hinge', 'adaptive_hinge'):
        return (np.abs(neg - pos + 1.0) < 1e-3).any(axis=0)
    if case['loss'] == 'bpr':
        return np.abs(pos - neg[0]) > 8.0
    return np.maximum(np.abs(pos), np.abs(neg[0])) > 8.0


def _separate_scores(case, rs):
    """Swap the negatives of interactions at a hinge boundary or outside the sigmoids' +-8 with
    those of other free interactions (every count stays)."""
    B, n = case['B'], case['n_neg']
    free = np.flatnonzero(~case['fixed'])
    for _ in range(100):
        bad = np.flatnonzero(_bad(case, scores(case)) & ~case['fixed'])
        if len(bad) == 0:
            return
        other = free[rs.randint(0, len(free), len(bad))]
        nv = case['negs'].reshape(n, B)
        for k, m in zip(bad, other):
            r = rs.randint(0, n)
            nv[r, k], nv[r, m] = nv[r, m], nv[r, k]
    raise ValueError('could not separate the scores of case %r' % ((case['D'], case['B'], case['loss']),))


def tables64(case):
    return [case[k].astype(np.float64) for k in ('Wu', 'Wi', 'bu', 'bi')]


def term_counts(case, ref):
    """Members per table row as the kernel's segment index counts them (terms with g != 0):
    dict(user=..., item=...) over all rows."""
    Mu, Mi = case['Wu'].shape[0], case['Wi'].shape[0]
    nu_, ni_ = max(case['Hu'], 1), max(case['Hi'], 1)
    cu, ci = np.zeros(Mu, dtype=np.int64), np.zeros(Mi, dtype=np.int64)
    for u, i, g in ((case['users'], case['items'], ref['gp']), (ref['kstar_user'], ref['kstar_item'], ref['gn'])):
        a = g != 0
        ru = ob.table_rows(u[a], case['Hu'], Mu, case['pad_u']).reshape(-1)
        ri = ob.table_rows(i[a], case['Hi'], Mi, case['pad_i']).reshape(-1)
        np.add.at(cu, ru, ni_)
        np.add.at(ci, ri, nu_)
    return dict(user=cu, item=ci)


def check_properties(case, ref):
    """Problems (an empty list when none) of the case on the oracle's dense result ``ref``."""
    out = []
    D, cap, G = case['D'], case['cap'], long_groups(case['D'])
    cnt = term_counts(case, ref)
    if len(case['hot_items']):
        Mi = case['Wi'].shape[0]
        for x, want in zip(case['hot_items'], case['hot_expected']):
            rows = ob.table_rows([x], case['Hi'], Mi, case['pad_i']).reshape(-1)
            if (cnt['item'][rows] != want).any():
                out.append('hot item %d rows have %s terms, not %d' % (x, cnt['item'][rows], want))
        lo, hi, vh = case['hot_expected']
        if not (lo <= cap < hi and vh > cap + 1 and vh % G != 0):
            out.append('hot counts %s do not straddle cap %d' % (case['hot_expected'], cap))
        if max(case['Hu'], 1) == 1 and (lo, hi) != (cap, cap + 1):
            out.append('no rows of exactly cap and cap + 1 terms')
        if np.bincount(case['items']).max() <= 100:
            out.append('no bias id repeated more than 100 times')
        if cnt['user'].max() <= cap:
            out.append('no hot user row')
    for side, H, ids in (('user', case['Hu'], case['users']), ('item', case['Hi'], np.r_[case['items'], case['negs']])):
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
        nb = ob.bias_buckets(case['B'])
        u = np.unique(ids)
        if len(u) == len(np.unique(u & (nb - 1))):
            out.append('no %s bias ids equal mod %d' % (side, nb))
    if case['loss'] == 'adaptive_hinge' and case['Hu'] == 0:
        b, B = case['adaptive_tie'], case['B']
        nv = ref['neg'].reshape(case['n_neg'], B)[:, b]
        if not (nv[0] == nv[1] == nv.max()) or ref['kstar_user'][b] == case['users'][(B + b) // case['n_neg']]:
            out.append('adaptive tie not at the maximum')
    pos, neg = ref['pos'], ref['neg'].reshape(case['n_neg'], -1)
    if case['loss'] in ('hinge', 'adaptive_hinge'):
        z = neg - pos + 1.0
        act = (ref['gp'] != 0).mean()
        if not 0.2 <= act <= 0.99:
            out.append('hinge activity %.2f outside 20-99 %%' % act)
        mine = case['users'] == case.get('inactive_user', -1)
        if 'inactive_user' in case and (not mine.any() or (ref['gp'][mine] != 0).any()):
            out.append('inactive user has an active interaction')
        if 'tie' in case and z[0, case['tie']] != 0.0:
            out.append('tie interaction not at z = 0')
        rest = np.ones(z.shape[1], dtype=bool)
        if 'tie' in case:
            rest[case['tie']] = False
        if (np.abs(z[:, rest]) < 1e-3).any():
            out.append('hinge |z| < 1e-3')
    else:
        arg = np.abs(pos - neg[0]) if case['loss'] == 'bpr' else np.maximum(np.abs(pos), np.abs(neg[0]))
        if arg.max() > 8.0:
            out.append('sigmoid argument %.2f beyond 8' % arg.max())
    return out


def hparams(case, opt, wd_on, seed=0):
    """(lr, weight_decay, initial states) that make one step measure the gradient at 1e-5, as
    oracle.mf_cases.hparams: SGD lr = 0.3 / max|g|; Adagrad accumulators ~ max|g|^2 per table and
    lr = half the largest weight; wd = 0.5 max|g| / max|w|."""
    P = tables64(case)
    ref = scores(case)
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
    """(D, loss, n_neg, Hu, Hi, pad, seed) of the suite: every D with each loss (hash counts and
    padding cycling), and every hash count with each loss at D = 32 and D = 100."""
    out = []
    for a, D in enumerate(DIMS):
        for b, (loss, n) in enumerate(LOSSES):
            Hu, Hi = HASHES[(a + b) % len(HASHES)]
            out.append((D, loss, n, Hu, Hi, PADS[(a + 2 * b) % 3], 1000 + 10 * a + b))
    for D in (32, 100):
        for c, (Hu, Hi) in enumerate(HASHES):
            for b, (loss, n) in enumerate(LOSSES):
                if (D, loss, n, Hu, Hi) not in [o[:5] for o in out]:
                    out.append((D, loss, n, Hu, Hi, PADS[(c + b) % 3], 2000 + D + 10 * c + b))
    return out


def case_for(D, loss, n, Hu, Hi, pad, seed):
    """The suite case of one matrix entry (every fifth with a hashed side gets a big id space); when
    the murmur search finds no id for one seed, the next seed is taken."""
    for s in range(seed, seed + 50 * 7919, 7919):
        try:
            return make_case(D, loss, Hu, Hi, pad, s, n_neg=n, big_ids=(seed % 5 == 0))
        except ValueError:
            continue
    raise ValueError('no case for %r' % ((D, loss, n, Hu, Hi, pad, seed),))
