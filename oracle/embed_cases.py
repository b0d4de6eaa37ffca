"""Test cases of the generic route's kernels (csrc/embed.cu lookups, csrc/mf.cu scores,
csrc/loss.cu standalone losses).

TEST INFRASTRUCTURE ONLY (tests/test_embed_oracle_gpu.py, tests/test_embed_oracle_cpu.py).

Each case promises properties that ``check_properties`` verifies on the oracle (oracle/embed.py):

* lookups at widths that reach every (LPR, VEC4) instantiation of ``emb_fwd_kernel`` and
  ``emb_bwd_kernel``: the scalar path at D in ``SCALAR_DIMS`` (D = 1 is every bias lookup), the
  float4 path at D in ``VEC4_DIMS``; 33, 132, 260 and wider take several lane passes;
* ``segments`` cases (plain tables): rows with 1, 2, 3, exactly ``seg_sort_cap(G)``, cap + 1 and
  5 cap + 3 members, and one row with ``HOT`` >= 4096 members, which the backward sums on its
  long-segment (min-selection) path;
* hash counts ``HASHES`` (and 0), compressed tables of 1, 2 and 7 rows where two hashes of one id
  land on one row, padding ``pad`` in {none, 0, 5}: the padding id among the ids, real ids on row
  0 and on the frozen row, and (plain, pad 5) the id 0, whose row is trained;
* an all-distinct batch, n = 0, n = 1, and n >= 2^20 at D = 1, where the grid-stride loops of
  every kernel take several rounds (the grid is capped at 8 CTAs per SM: 1056 on 132 SMs);
* ``mf_scores`` at D in ``SCORE_DIMS`` with odd n, exact zeros among the score gradients, one
  user owning the whole batch, and the broadcast (``predict``) mode;
* losses at n in ``LOSS_NS`` (10^6 + 3 reaches the 1056-block fold), the adaptive hinge with
  2, 5, 10 negatives and exact ties at the maximum, masks with one unmasked element, hinge
  |z| >= 1e-3, poisson predictions below 1e-2 and logistic scores at |s| ~ 30.

Table and ``dout`` values have |x| in [2^-4, 2^4], so float32 partial sums are never subnormal.
"""

import numpy as np

from oracle import embed as oe

SCALAR_DIMS = (1, 2, 3, 5, 7, 10, 17, 31, 33, 63)
VEC4_DIMS = (4, 8, 12, 16, 32, 64, 100, 128, 132, 260, 512)
DIMS = SCALAR_DIMS + VEC4_DIMS
HASHES = (1, 2, 4, 24)
PADS = (-1, 0, 5)
HOT = 4096 + 7
HUGE = (1 << 20) + 5
GRID_THREADS = 132 * 8 * 256            # threads of one grid-stride round at 8 CTAs per SM
SCORE_DIMS = (4, 8, 12, 32, 100, 128, 256)
LOSS_NS = (1, 255, 256, 257, 10 ** 6 + 3)
PAIR_LOSSES = (('pointwise', 1), ('bpr', 1), ('hinge', 1), ('adaptive_hinge', 2), ('adaptive_hinge', 5),
               ('adaptive_hinge', 10))
RATING_LOSSES = ('regression', 'poisson', 'logistic')


def values(rs, shape):
    """float32 with random signs and |x| in [2^-4, 2^4], log-uniform."""
    mag = 2.0 ** rs.uniform(-4.0, 4.0, shape)
    return (np.where(rs.rand(*shape) < 0.5, -mag, mag)).astype(np.float32)


def _lookup(name, D, H, pad, M, ids, rs, **extra):
    ids = np.asarray(ids, dtype=np.int64)
    case = dict(kind='lookup', name=name, D=D, H=H, pad=pad, M=M, ids=ids, W=values(rs, (M, D)),
                dout=values(rs, (len(ids), D)))
    case.update(extra)
    return case


def _search(rs, N, H, M, pad, cond, k=1):
    """k ids in [1, N), not the padding id, whose hashed rows satisfy ``cond``."""
    for _ in range(400):
        cand = rs.randint(1, N, 4096).astype(np.int64)
        cand = cand[cand != pad]
        ok = cand[cond(oe.term_rows(cand, H, M, pad))]
        if len(ok) >= k:
            return list(ok[:k])
    raise ValueError('no id found')


def segments_case(D, pad, seed):
    """Plain table: rows with prescribed member counts around seg_sort_cap(G) and one hot row."""
    rs = np.random.RandomState(seed)
    cap = oe.seg_sort_cap(oe.pow2_lanes(D))
    lens = [1] * 12 + [2] * 6 + [3] * 4 + [cap] * 2 + [cap + 1] * 2 + [5 * cap + 3, HOT]
    M = 600
    free = rs.permutation(np.setdiff1d(np.arange(M), [0, max(pad, 0)]))
    ids = list(np.repeat(free[:len(lens)], lens))
    if pad >= 0:
        ids += [pad] * 7
    if pad != 0:
        ids += [0] * 3
    ids = np.array(ids, dtype=np.int64)
    rs.shuffle(ids)
    return _lookup('segments', D, 0, pad, M, ids, rs, lens=sorted(set(lens)))


def hashed_case(D, H, pad, seed, M=997, N=50000, n_rand=800):
    """Bloom table: random ids, two hot ids, the padding id, the id 0, ids on row 0 / the frozen
    row and an id with two hashes on one row."""
    rs = np.random.RandomState(seed)
    cap = oe.seg_sort_cap(oe.pow2_lanes(D))
    ids = list(rs.randint(1, N, n_rand))
    ids += _search(rs, N, H, M, pad, lambda r: np.ones(len(r), dtype=bool))[:1] * (cap + 1)
    ids += _search(rs, N, H, M, pad, lambda r: np.ones(len(r), dtype=bool))[:1] * (5 * cap + 3)
    if pad >= 0:
        ids += [pad] * 5
    ids += [0] * 3
    ids += _search(rs, N, H, M, pad, lambda r: (r == 0).any(axis=1)) * 2
    if pad > 0:
        ids += _search(rs, N, H, M, pad, lambda r: (r == pad).any(axis=1)) * 2
    if H >= 2:
        ids += _search(rs, N, H, M, pad, lambda r: np.array([len(set(x)) < len(x) for x in r])) * 2
    ids = np.array(ids, dtype=np.int64)
    rs.shuffle(ids)
    return _lookup('hashed', D, H, pad, M, ids, rs)


def tiny_case(D, H, pad, M, seed):
    """A compressed table of M rows (1, 2 or 7): hashes of one id collide."""
    rs = np.random.RandomState(seed)
    ids = list(rs.randint(0, 1000, 300))
    if pad >= 0:
        ids += [pad] * 4
    ids = np.array(ids, dtype=np.int64)
    rs.shuffle(ids)
    return _lookup('tiny', D, H, pad, M, ids, rs)


def distinct_case(D, seed):
    rs = np.random.RandomState(seed)
    return _lookup('distinct', D, 0, -1, 3000, rs.permutation(3000)[:2000], rs)


def sized_case(D, H, pad, n, seed):
    """n ids (0, 1, or HUGE with a hot row) in a plain table or a Bloom one."""
    rs = np.random.RandomState(seed)
    M = 1 << 17 if n > HOT else 5000
    ids = rs.randint(0, M, n).astype(np.int64)
    if n > HOT:
        ids[rs.permutation(n)[:HOT]] = 4242
    return _lookup('n%d' % n, D, H, pad, M, ids, rs)


def scores_case(D, n, mode, seed):
    """Score gradients with ~15 % exact zeros.  ``mode``: 'batch' (a hot user and a hot item),
    'owner' (one user owns the batch) or 'bcast' (one user, items 0..n-1, as predict does)."""
    rs = np.random.RandomState(seed)
    U, I = 700, (n if mode == 'bcast' else 900)
    Wu = (rs.randn(U, D) / D ** 0.25).astype(np.float32)
    Wi = (rs.randn(I, D) / D ** 0.25).astype(np.float32)
    bu = (rs.randn(U, 1) * 0.1).astype(np.float32)
    bi = (rs.randn(I, 1) * 0.1).astype(np.float32)
    if mode == 'bcast':
        users, items = np.array([17], dtype=np.int64), np.arange(n, dtype=np.int64)
    else:
        users = rs.randint(0, U, n).astype(np.int64)
        items = rs.randint(0, I, n).astype(np.int64)
        users[rs.rand(n) < (1.0 if mode == 'owner' else 0.4)] = 17
        items[rs.rand(n) < 0.3] = 5
    g = (rs.randn(n)).astype(np.float32)
    if n > 1:
        g[rs.rand(n) < 0.15] = 0.0
        g[0] = 0.0
    return dict(kind='scores', name=mode, D=D, n=n, Wu=Wu, Wi=Wi, bu=bu, bi=bi, users=users, items=items, g=g)


def pairwise_case(loss, n_neg, n, mask, seed):
    """pos, neg (n_neg, n) or (n,), and a mask: None, 'random' (~70 % on) or 'single'."""
    rs = np.random.RandomState(seed)
    pos = (rs.randn(n) * 2).astype(np.float32)
    neg = (rs.randn(n_neg, n) * 2).astype(np.float32)
    cols = np.array([rs.randint(0, n)])
    if loss == 'adaptive_hinge':
        # exact ties at the maximum of ~5 % of the columns (at least one), hinge active there
        cols = np.flatnonzero(rs.rand(n) < 0.05)
        cols = cols if len(cols) else np.array([0])
        for i in cols:
            k1, k2 = np.sort(rs.choice(n_neg, 2, replace=False))
            neg[k1, i] = neg[k2, i] = neg[:, i].max() + np.float32(0.25)
            pos[i] = min(pos[i], neg[k1, i] - np.float32(0.5))
    if loss in ('hinge', 'adaptive_hinge'):
        z = neg - pos[None] + 1.0
        neg[np.abs(z) < 1e-3] += np.float32(0.01)
    m = None
    if mask == 'random':
        m = rs.rand(n) < 0.7
        m[0] = True
    elif mask == 'single':
        m = np.zeros(n, dtype=bool)
        m[cols[0]] = True                    # (adaptive hinge: a tied column)
    return dict(kind='pairwise', name=loss, loss=loss, n_neg=n_neg, n=n, pos=pos,
                neg=neg if loss == 'adaptive_hinge' else neg[0], mask=m, mask_kind=mask)


def rating_case(loss, n, seed):
    rs = np.random.RandomState(seed)
    if loss == 'regression':
        pred, r = rs.randn(n) * 2, rs.randint(1, 6, n)
    elif loss == 'poisson':
        pred, r = np.exp(rs.uniform(-7.0, 2.0, n)), rs.randint(0, 6, n)
        pred[0] = 1e-3
    else:
        # |s| ~ 30 on both sides of the target; n = 1 keeps a gradient float32 can represent (at
        # s = 30, r = 1 it is 1 - sigmoid(30) ~ 1e-13 in float64 and exactly 0 in float32)
        pred, r = rs.uniform(-30.0, 30.0, n), rs.choice([-1, 1], n)
        pred[0], r[0] = (30.0, -1) if n == 1 else (-29.9, r[0])
        if n > 1:
            pred[1] = 30.0
    return dict(kind='rating', name=loss, loss=loss, n=n, pred=pred.astype(np.float32),
                ratings=r.astype(np.float32))


# ------------------------------------------------------------------ the matrix

def matrix():
    """Entries (a tuple whose first element is the builder's name) of the suite."""
    out = []
    for k, D in enumerate(DIMS):
        out.append(('segments', D, PADS[k % 3], 100 + k))
        out.append(('hashed', D, HASHES[k % 4], PADS[(k + 1) % 3], 200 + k))
    out += [('tiny', 3, 2, 0, 1, 301), ('tiny', 4, 24, -1, 1, 302), ('tiny', 8, 4, -1, 2, 303),
            ('tiny', 1, 2, 0, 2, 304), ('tiny', 33, 24, 5, 7, 305), ('tiny', 12, 1, 5, 7, 306)]
    out += [('distinct', 5, 401), ('distinct', 64, 402)]
    out += [('sized', 7, 0, -1, 0, 501), ('sized', 32, 4, 0, 0, 502), ('sized', 1, 0, 0, 1, 503),
            ('sized', 100, 4, 0, 1, 504), ('sized', 1, 0, 0, HUGE, 505), ('sized', 1, 2, 5, HUGE, 506)]
    for k, D in enumerate(SCORE_DIMS):
        out.append(('scores', D, 2001 + 2 * k, 'batch', 600 + k))
    out += [('scores', 32, 4097, 'owner', 610), ('scores', 256, 3, 'owner', 611), ('scores', 4, 1, 'batch', 612),
            ('scores', 12, 1001, 'bcast', 613), ('scores', 128, 1001, 'bcast', 614)]
    masks = (None, 'random', 'single')
    for a, (loss, n_neg) in enumerate(PAIR_LOSSES):
        for b, n in enumerate(LOSS_NS):
            out.append(('pairwise', loss, n_neg, n, masks[(a + b) % 3], 700 + 10 * a + b))
    for a, loss in enumerate(RATING_LOSSES):
        for b, n in enumerate(LOSS_NS):
            out.append(('rating', loss, n, 800 + 10 * a + b))
    return out


_BUILDERS = dict(segments=segments_case, hashed=hashed_case, tiny=tiny_case, distinct=distinct_case,
                 sized=sized_case, scores=scores_case, pairwise=pairwise_case, rating=rating_case)


def entry_id(e):
    return '-'.join(str(x) for x in e[:-1])


def case_for(entry):
    return _BUILDERS[entry[0]](*entry[1:])


# ------------------------------------------------------------------ properties

def _bounded(x):
    a = np.abs(x)
    return a.size == 0 or (a.min() >= 2.0 ** -4 and a.max() <= 2.0 ** 4)


def check_properties(case):
    """Problems of a case (an empty list when none)."""
    out = []
    if case['kind'] == 'lookup':
        D, H, pad, M, ids = case['D'], case['H'], case['pad'], case['M'], case['ids']
        if not (_bounded(case['W']) and _bounded(case['dout'])):
            out.append('values outside [2^-4, 2^4]')
        rows = oe.term_rows(ids, H, M, pad)
        if len(ids) and (rows.min() < 0 or rows.max() >= M or ids.min() < 0):
            out.append('ids or rows out of range')
        cnt = oe.term_counts(ids, H, M, pad)
        cap = oe.seg_sort_cap(oe.pow2_lanes(D))
        if case['name'] == 'segments':
            for L in case['lens']:
                if not (cnt == L).any():
                    out.append('no row with %d members' % L)
            if not (cap in case['lens'] and cap + 1 in case['lens'] and max(case['lens']) >= 4096):
                out.append('segment classes do not straddle cap %d' % cap)
            if pad != 0 and not (ids == 0).any():
                out.append('id 0 absent')
        if case['name'] == 'hashed' and cnt.max() <= cap:
            out.append('no row longer than cap')
        if case['name'] in ('segments', 'hashed', 'tiny') and pad >= 0 and not (ids == pad).any():
            out.append('padding id absent')
        if H and case['name'] in ('hashed', 'tiny'):
            real = ids != pad
            if not (rows[real] == 0).any():
                out.append('no real id on row 0')
            if 0 < pad < M and not (rows[real] == pad).any():
                out.append('no real id on the frozen row')
            if H >= 2 and not any(len(set(x)) < H for x in rows):
                out.append('no id with two hashes on one row')
        if case['name'] == 'distinct' and len(np.unique(ids)) != len(ids):
            out.append('ids not distinct')
        if case['name'] == 'n%d' % HUGE and not (D == 1 and len(ids) > 3 * GRID_THREADS and cnt.max() >= 4096):
            out.append('huge case: not D = 1 with several grid rounds and a hot row')
        if 0 <= pad and pad >= M:
            out.append('frozen row outside the table')
    elif case['kind'] == 'scores':
        n = case['n']
        if n % 2 != 1:
            out.append('n even')
        if n > 1 and not (case['g'] == 0).any():
            out.append('no exact zero score gradient')
        if case['name'] == 'owner' and len(np.unique(case['users'])) != 1:
            out.append('owner case with several users')
        if case['name'] == 'bcast' and not (case['users'].size == 1 and n > 1):
            out.append('broadcast case not broadcast')
    elif case['kind'] == 'pairwise':
        pos, neg, m = case['pos'], case['neg'], case['mask']
        if case['loss'] in ('hinge', 'adaptive_hinge'):
            top = neg.max(axis=0) if neg.ndim == 2 else neg
            if (np.abs(top.astype(np.float64) - pos + 1.0) < 1e-3).any():
                out.append('hinge |z| < 1e-3')
        if case['loss'] == 'adaptive_hinge':
            srt = np.sort(neg, axis=0)
            tie = (srt[-1] == srt[-2]) & (srt[-1] - pos + 1.0 > 0)
            if m is not None:
                tie &= m
            if not tie.any():
                out.append('no active tie at the maximum')
        if case['mask_kind'] == 'single' and m.sum() != 1:
            out.append('single mask with %d on' % m.sum())
    elif case['kind'] == 'rating':
        p = case['pred']
        if case['loss'] == 'poisson' and not (p.min() <= 1e-2 and p.min() > 0):
            out.append('no small poisson prediction')
        if case['loss'] == 'logistic' and np.abs(p).max() < 29.0:
            out.append('no logistic score near 30')
    return out


# ------------------------------------------------------------------ the oracle of a case

def oracle(case, mutate=()):
    """The float64 result of a case (and, for lookups, the ordered float32 one)."""
    if case['kind'] == 'lookup':
        args = (case['ids'], case['H'])
        return dict(out=oe.lookup(case['W'], *args, case['pad'], mutate=mutate),
                    dW=oe.lookup_backward(case['dout'], *args, case['M'], case['pad'], mutate=mutate),
                    rows=oe.term_rows(case['ids'], case['H'], case['M'], case['pad'], mutate))
    if case['kind'] == 'scores':
        s = oe.scores(case['Wu'], case['Wi'], case['bu'], case['bi'], case['users'], case['items'])
        d = oe.scores_backward(case['g'], case['Wu'], case['Wi'], case['users'], case['items'], mutate)
        return dict(scores=s, dWu=d[0], dWi=d[1], dbu=d[2], dbi=d[3])
    if case['kind'] == 'pairwise':
        l, gp, gn = oe.pairwise_loss(case['loss'], case['pos'], case['neg'], case['mask'], mutate)
        return dict(loss=np.array(l), gp=gp, gn=gn)
    l, g = oe.rating_loss(case['loss'], case['pred'], case['ratings'])
    return dict(loss=np.array(l), g=g)


def sum_bounds(case):
    """Element-wise bounds of the float32 rounding of a lookup case's sums: (k - 1) 2^-24 sum|x|
    over the k terms of an element (recursive summation).  A row of 4096 terms of either sign sits
    ~3e-6 of the table's largest gradient away from float64, so a flat 1e-6 cannot hold there."""
    u = 2.0 ** -24
    fan = max(case['H'], 1)
    out = oe.lookup(np.abs(case['W']), case['ids'], case['H'], case['pad']) * ((fan - 1) * u)
    cnt = oe.term_counts(case['ids'], case['H'], case['M'], case['pad'])
    dW = oe.lookup_backward(np.abs(case['dout']), case['ids'], case['H'], case['M'], case['pad'])
    return dict(out=out, dW=dW * (np.maximum(cnt - 1, 0) * u)[:, None])


def within(got, want, bound, rtol=1e-6):
    """|got - want| <= rtol * max|want| + bound, element-wise; returns the problem or None."""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    if got.shape != want.shape:
        return 'shape %s != %s' % (got.shape, want.shape)
    if want.size == 0:
        return None
    excess = np.abs(got - want) - (rtol * np.abs(want).max() + bound)
    if excess.max() > 0:
        k = np.unravel_index(np.argmax(excess), want.shape)
        return 'element %s: %r vs %r (bound %.3e)' % (k, float(got[k]), float(want[k]), float(np.broadcast_to(bound, want.shape)[k]))
    return None


def ordered(case, mutate=()):
    """The ordered float32 forward and backward of a lookup case."""
    args = (case['ids'], case['H'])
    return dict(out=oe.lookup(case['W'], *args, case['pad'], ordered=True, mutate=mutate),
                dW=oe.lookup_backward(case['dout'], *args, case['M'], case['pad'], ordered=True, mutate=mutate))
