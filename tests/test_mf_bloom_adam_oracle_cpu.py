"""Lazy-exact Adam on hashed (Bloom) tables without the GPU (tests/bloom_adam_common.py).

* The float64 lazy scheme -- every row and bias a minibatch reads caught up through t - 1 before the
  forward, the real step on the entries with a gradient, a flush at the end -- equals float64 dense
  Adam over several steps in which most rows miss steps, with and without weight decay.
* Each plausible kernel mistake, restated as a mutation of the scheme, moves a table or a moment by
  more than tests/test_mf_bloom_adam_gpu.py's tolerances.
* Replayed over the reference's own minibatch stream, the scheme reproduces the two fits the live
  reference recorded with its default dense Adam (tests/golden/make_golden_bloom_adam.py).
"""
import numpy as np
import pytest

from bloom_adam_common import MUTATIONS, dense_adam, lazy_step, make_tables
from conftest import assert_close
from oracle import bloom as ob
from oracle import bloom_cases as bc

LR = 1e-3
STEPS = 4
TABLES = ('Wu', 'Wi', 'bu', 'bi')


def minibatches(case, steps=STEPS, seed=0):
    """Step 1 is the whole case (hot rows, bucket twins); later steps take a random eighth of it, so
    rows miss steps between touches."""
    B, n = len(case['users']), case['n_neg']
    rs = np.random.RandomState(seed)
    out = [(case['users'], case['items'], case['negs'])]
    for _ in range(steps - 1):
        idx = np.sort(rs.choice(B, B // 8, replace=False))
        negs = case['negs'][rs.permutation(len(case['negs']))[:len(idx) * n]]
        out.append((case['users'][idx], case['items'][idx], negs))
    return out


def run_lazy(case, wd, mutate=()):
    tabs = make_tables(bc.tables64(case), LR, wd)
    for t, (u, i, j) in enumerate(minibatches(case), 1):
        lazy_step(tabs, case, u, i, j, t, mutate)
    return tabs


CASES = [(32, 'bpr', 1, 0, 4, 0), (12, 'adaptive_hinge', 2, 2, 3, 3), (64, 'hinge', 1, 3, 0, -1)]


@pytest.mark.parametrize('wd', [0.0, 0.1])
@pytest.mark.parametrize('entry', CASES, ids=['%d-%s%d-%d,%d-pad%d' % e for e in CASES])
def test_lazy_scheme_equals_dense_adam(entry, wd):
    case = bc.case_for(*entry, seed=300 + entry[0])
    batches = minibatches(case)
    tabs = run_lazy(case, wd)
    missed = sum(int((tab.last < STEPS).sum()) for tab in tabs)
    for tab in tabs:
        tab.flush(STEPS)

    def grads(P, t):
        u, i, j = batches[t - 1]
        ref = ob.step([p.copy() for p in P], u, i, j, case['loss'], case['Hu'], case['Hi'], case['pad_u'],
                      case['pad_i'], case['n_neg'])
        return ref['dWu'], ref['dWi'], ref['dbu'], ref['dbi']

    dense = dense_adam(bc.tables64(case), grads, STEPS, LR, wd)
    assert missed > 0, 'no entry missed a step'
    for tab, p, nm in zip(tabs, dense, TABLES):
        assert_close(tab.w, p, 1e-9, atol=1e-12, what=nm)


def caught(a, b):
    """True when tables b differ from a by more than the GPU test's tolerances (moments at 2e-5 of
    their scale, parameters at 5 % of one step)."""
    for x, y in zip(a, b):
        for u, v in ((x.m, y.m), (x.v, y.v)):
            if np.abs(u - v).max() > 2e-5 * max(np.abs(u).max(), 1e-30):
                return True
        if np.abs(x.w - y.w).max() > 0.05 * LR + 2e-6 * np.abs(x.w).max():
            return True
        if (x.last != y.last).any():
            return True
    return False


@pytest.mark.parametrize('mutation', MUTATIONS)
def test_tolerances_catch_each_mistake(mutation):
    """Bloom on both sides with a padding row, weight decay 0.1 (the frozen row moves only under
    weight decay), four steps."""
    case = bc.case_for(32, 'bpr', 1, 2, 3, 0, seed=411)
    good = run_lazy(case, 0.1)
    bad = run_lazy(case, 0.1, (mutation,))
    assert caught(good, bad), mutation



FIXTURES = ['fit_bloom_adam_bpr', 'fit_bloom_adam_both']


@pytest.mark.parametrize('name', FIXTURES)
def test_lazy_scheme_reproduces_reference_default_adam_fit(name):
    """tests/golden/make_golden_bloom_adam.py: two epochs of the reference's fit() with its default
    dense Adam, replayed through the float64 lazy scheme over the reference's own minibatch stream
    (per epoch one shuffle of arange(n), per minibatch one randint of len(batch) * n negatives).
    Epoch losses at 1e-5, final tables at 2e-3 of their scale (Adam's m / sqrt(v) turns last-bit
    gradient differences on near-zero components into fractions of a step, as in
    test_seq_adam_oracle_cpu), predict at 2e-3, RandomState position exact."""
    from bloom_adam_common import fixture_case, fixture_names
    from conftest import load_golden
    g = load_golden(name)
    case = fixture_case(g)
    names = fixture_names(g)
    tabs = make_tables([g['init.' + k] for k in names], float(g['lr']), float(g['l2']))
    rs = np.random.RandomState()
    rs.set_state(('MT19937', g['rs0_key'], int(g['rs0_pos'])))
    users, items = g['users'].astype(np.int64), g['items'].astype(np.int64)
    n, B, I = len(users), int(g['batch']), int(g['num_items'])
    t, losses, missed = 0, [], 0
    for _ in range(int(g['n_iter'])):
        order = np.arange(n)
        rs.shuffle(order)
        u, i = users[order], items[order]
        ep = []
        for lo in range(0, n, B):
            bu_, bi_ = u[lo:lo + B], i[lo:lo + B]
            negs = rs.randint(0, I, len(bu_) * case['n_neg'], dtype=np.int64)
            t += 1
            missed += sum(int((tab.last < t - 2).sum()) for tab in tabs)
            ep.append(lazy_step(tabs, case, bu_, bi_, negs, t)['loss'])
        losses.append(float(np.mean(ep)))
    for tab in tabs:
        tab.flush(t)
    assert missed > 0, 'no entry missed several steps'
    assert_close(np.array(losses), g['epoch_losses'], 1e-5, what='epoch losses')
    for tab, k in zip(tabs, names):
        assert_close(tab.w, g['final.' + k], 2e-3, atol=1e-7, what=k)
    st = rs.get_state()
    assert (st[1] == g['rs_key']).all() and st[2] == int(g['rs_pos'])
    Wu, Wi, bu, bi = (tab.w for tab in tabs)
    p = int(g['predict_user'])
    uv = Wu[ob.table_rows(np.array([p]), case['Hu'], Wu.shape[0], case['pad_u'])].sum(axis=1)[0]
    iv = Wi[ob.table_rows(np.arange(I), case['Hi'], Wi.shape[0], case['pad_i'])].sum(axis=1)
    assert_close(iv @ uv + bu[p, 0] + bi[:, 0], g['predict'], 2e-3, what='predict')
