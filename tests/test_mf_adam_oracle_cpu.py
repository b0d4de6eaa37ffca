"""The float64 lazy-exact Adam scheme of the first-generation MF step (oracle/adam.py lazy_mf_step,
LazyAdamTable) on the CPU: the vectorised catch-up equals the row loop; the lazy scheme followed by a
flush equals dense float64 Adam; and each mistake in oracle.adam.MF_MUTATIONS, run on the cases
tests/test_mf_adam_oracle_gpu.py uses, moves a quantity that test compares beyond its tolerance."""

import numpy as np
import pytest

from oracle import mf_adam_cases as mac
from oracle.adam import MF_MUTATIONS, LazyAdamTable, lazy_mf_step, mf_terms

LR = 1e-3
STEPS = 4           # as the GPU test


@pytest.mark.parametrize('wd', [0.0, 0.1])
def test_vectorised_catch_up_equals_row_loop(wd):
    """Rows far behind, one behind, current, ahead of ``upto`` and never touched (m = v = 0), with
    repeated ids: bit-identical tables, moments and ``last``."""
    rs = np.random.RandomState(1)
    rows, D = 300, 8
    tabs = []
    for _ in range(2):
        tab = LazyAdamTable(rs.randn(rows, D) * 0.3 if not tabs else tabs[0].w.copy(), lr=LR, weight_decay=wd)
        tabs.append(tab)
    last = rs.randint(0, 260, rows)
    last[:20] = 0
    m = rs.randn(rows, D) * 1e-3
    v = rs.uniform(0.25, 1.0, (rows, D)) * 1e-6
    m[:20] = v[:20] = 0.0
    for tab in tabs:
        tab.m, tab.v, tab.last = m.copy(), v.copy(), last.copy()
    ids = np.r_[rs.randint(0, rows, 400), np.arange(20)]
    tabs[0].catch_up(ids, 250)
    tabs[1].catch_up_loop(ids, 250)
    for a in ('w', 'm', 'v', 'last'):
        assert np.array_equal(getattr(tabs[0], a), getattr(tabs[1], a)), a
    tabs[0].flush(300)
    tabs[1].catch_up_loop(np.arange(rows), 300)
    for a in ('w', 'm', 'v', 'last'):
        assert np.array_equal(getattr(tabs[0], a), getattr(tabs[1], a)), 'flush ' + a


def _dense_run(case, wd, t0, state, bats):
    """Dense float64 Adam: the seeded state brought current for t0 - 1 (what dense Adam would hold),
    then every row steps at every step."""
    tabs = mac.tables(case, LR, wd, state)
    for tab in tabs:
        tab.flush(t0 - 1)
    losses = []
    for step, (u, i, j, r) in enumerate(bats, t0):
        ref = mf_terms([tab.w for tab in tabs], u, i, j, case['loss'], case['n_neg'], r)
        for tab, g in zip(tabs, (ref['dWu'], ref['dWi'], ref['dbu'], ref['dbi'])):
            tab._step(np.arange(tab.w.shape[0]), step, g.reshape(tab.w.shape))
            tab.last[:] = step
        losses.append(ref['loss'])
    return tabs, losses


DENSE = [(8, 'bpr', 1, 0.0, 1), (8, 'hinge', 1, 0.1, 1000), (12, 'adaptive_hinge', 5, 0.1, 1000),
         (4, 'pointwise', 1, 0.1, 30), (8, 'regression', 1, 0.1, 1000), (12, 'poisson', 1, 0.0, 1000),
         (4, 'logistic', 1, 0.1, 1)]


@pytest.mark.parametrize('D,loss,n,wd,t0', DENSE, ids=['%d-%s%d-wd%g-t%d' % e for e in DENSE])
def test_lazy_then_flush_equals_dense_adam(D, loss, n, wd, t0):
    """Several lazy steps (rows missing steps between touches), then a flush: the tables, moments and
    every step's loss of dense float64 Adam from the same state, to float64 rounding."""
    case = mac.make_case(D, 1500, loss, n, seed=D + t0)
    state = mac.seed_state(case, t0, seed=3)
    bats = mac.batches(case, 6, seed=5)
    tabs = mac.tables(case, LR, wd, state)
    losses = [lazy_mf_step(tabs, u, i, j, loss, s, case['n_neg'], r)['loss'] for s, (u, i, j, r) in enumerate(bats, t0)]
    assert any((tab.last < t0 + len(bats) - 2).any() for tab in tabs)
    for tab in tabs:
        tab.flush(t0 + len(bats) - 1)
    dense, dlosses = _dense_run(case, wd, t0, state, bats)
    np.testing.assert_allclose(losses, dlosses, rtol=1e-12)
    for tab, ref, nm in zip(tabs, dense, mac.TABLES):
        for a in ('w', 'm', 'v'):
            x, y = getattr(tab, a), getattr(ref, a)
            assert np.abs(x - y).max() <= 1e-12 * np.abs(y).max(), (nm, a)
        assert (tab.last == ref.last).all()


# ------------------------------------------------------------------ mutations
def _caught(case, wd, t0, mutate):
    """Whether the GPU test's checks (tests/test_mf_adam_oracle_gpu.py run_steps: loss at 1e-5, `last`
    exactly, moments at 2e-5 of their scale, parameters within its step rule; after every step and
    after the flush) tell the mutated scheme from the scheme.  Returns the set of quantities that
    differ."""
    state = mac.seed_state(case, t0, seed=case['D'] + t0)
    good, bad = mac.tables(case, LR, wd, state), mac.tables(case, LR, wd, state)
    seen = set()

    def compare(what):
        for k, (g, b) in enumerate(zip(good, bad)):
            if (g.last != b.last).any():
                seen.add('last')
            for a in ('m', 'v'):
                x, y = getattr(b, a), getattr(g, a)
                if np.abs(x - y).max() > 2e-5 * np.abs(y).max():
                    seen.add(a)
            quiet = np.abs(g.m) < 1e-3 * np.abs(g.m).max()
            err = np.abs(b.w - g.w)
            tol = 2e-6 * np.abs(g.w).max()
            if err[~quiet].max(initial=0.0) > 0.05 * LR + tol or err.max() > 2.1 * LR:
                seen.add('w')

    for step, (u, i, j, r) in enumerate(mac.batches(case, STEPS, seed=t0), t0):
        ra = lazy_mf_step(good, u, i, j, case['loss'], step, case['n_neg'], r)
        rb = lazy_mf_step(bad, u, i, j, case['loss'], step, case['n_neg'], r, mutate=mutate)
        if abs(ra['loss'] - rb['loss']) > 1e-5 * abs(ra['loss']):
            seen.add('loss')
        compare(step)
    for tabs in (good, bad):
        for tab in tabs:
            tab.flush(t0 + STEPS - 1)
    compare('flush')
    return seen


# (mutation, a GPU small-batch case it applies to, what must show); apply_all_referenced must show in `last`
MUTANTS = [('prepass_no_negs', (4, 'bpr', 1, 0.1, 1000), None),
           ('prepass_no_negs', (8, 'adaptive_hinge', 2, 0.0, 1000), None),
           ('bias_own_last', (4, 'bpr', 1, 0.1, 1000), None),
           ('bias_own_last', (16, 'poisson', 1, 0.1, 1000), None),
           ('catch_up_through_t', (8, 'hinge', 1, 0.1, 1), None),
           ('catch_up_through_t', (12, 'regression', 1, 0.1, 1), None),
           ('apply_all_referenced', (8, 'hinge', 1, 0.1, 1), 'last'),
           ('apply_all_referenced', (8, 'adaptive_hinge', 2, 0.0, 1000), 'last'),
           ('no_decay_replay', (4, 'bpr', 1, 0.1, 1000), None),
           ('no_decay_replay', (16, 'poisson', 1, 0.1, 1000), None)]


def test_mutants_cover_every_mistake_on_gpu_cases():
    assert {m for m, _, _ in MUTANTS} == set(MF_MUTATIONS)
    for _, e, _ in MUTANTS:
        assert e in mac.SMALL, e


@pytest.mark.parametrize('mutation,entry,must', MUTANTS, ids=['%s-%d-%s%d' % (m, e[0], e[1], e[2]) for m, e, _ in MUTANTS])
def test_gpu_tolerances_catch_mutation(mutation, entry, must):
    D, loss, n, wd, t0 = entry
    seen = _caught(mac.small_case(D, loss, n), wd, t0, (mutation,))
    assert seen, '%s passes the GPU checks' % mutation
    if must:
        assert must in seen, (mutation, seen)
