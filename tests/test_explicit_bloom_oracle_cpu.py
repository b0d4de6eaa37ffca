"""The hashed-table rating oracle (oracle/explicit_bloom.py) and the cases of
tests/test_explicit_bloom_gpu.py, checked without a GPU.

* It reproduces the live reference: one explicit-feedback minibatch with a Bloom item layer (and
  one with both layers hashed) per loss, and two-epoch fit() runs under SGD and Adagrad
  (tests/golden/explicit_bloom_*.npz, fit_explicit_bloom_*.npz).
* With plain tables on both sides it is oracle.explicit's step and fused step.
* Every matrix case carries the ids, term counts and score scales it promises.
* Each plausible kernel mistake, restated as a mutated oracle call, moves the update, the state
  change, a gradient or the loss by more than the GPU suite's 1e-5 tolerance.
"""

import numpy as np
import pytest

from conftest import assert_close, load_golden
from oracle import bloom as ob
from oracle import explicit as oex
from oracle import explicit_bloom as oeb
from oracle import explicit_bloom_cases as ebc

TABLES = ('Wu', 'Wi', 'bu', 'bi')
STEP_FIXTURES = ('explicit_bloom_regression', 'explicit_bloom_poisson', 'explicit_bloom_logistic',
                 'explicit_bloom_both_regression')


def _names(g):
    user = 'user_embeddings.embeddings.weight' if int(g.get('user_H', 0)) else 'user_embeddings.weight'
    return [user, 'item_embeddings.embeddings.weight', 'user_biases.weight', 'item_biases.weight']


@pytest.mark.parametrize('name', STEP_FIXTURES)
def test_reproduces_reference_step_fixtures(name):
    g = load_golden(name)
    loss, Hu, Hi = str(g['loss_kind']), int(g['user_H']), int(g['item_H'])
    names = _names(g)
    P = [g['sd.' + k].astype(np.float64) for k in names]
    out = oeb.step(P, g['users'], g['items'], g['ratings'], loss, Hu, Hi, 0, 0)
    assert_close(np.exp(out['pos']) if loss == 'poisson' else out['pos'], g['pred'], 1e-5, what='pred')
    assert_close(out['loss'], g['loss'], 1e-5, what='loss')
    for k, nm in zip(names, ('dWu', 'dWi', 'dbu', 'dbi')):
        assert_close(out[nm], g['grad.' + k], 1e-5, atol=1e-8, what=nm)


@pytest.mark.parametrize('name,opt', [('fit_explicit_bloom_sgd', 'sgd'), ('fit_explicit_bloom_adagrad', 'adagrad')])
def test_fit_reproduces_reference_trajectory(name, opt):
    """Two epochs of the reference's fit() with a Bloom item layer and torch.optim.SGD / Adagrad
    (wd = 0: the row-wise fused optimizers are the dense ones)."""
    g = load_golden(name)
    loss, H = str(g['loss_kind']), int(g['bloom_H'])
    names = _names(g)
    P = [g['init.' + k].astype(np.float64) for k in names]
    S = [np.zeros(p.shape) for p in P]
    rs = np.random.RandomState()
    rs.set_state(('MT19937', g['rs0_key'], int(g['rs0_pos'])))
    losses = oeb.fit(P, g['users'], g['items'], g['ratings'], loss, int(g['batch']), int(g['n_iter']), rs, opt,
                     float(g['lr']), Hu=0, Hi=H, pad_i=0, states=S)
    assert_close(np.array(losses), g['epoch_losses'], 1e-5, what='epoch losses')
    for p, k in zip(P, names):
        assert_close(p, g['final.' + k], 1e-5, atol=1e-7, what=k)
    st = rs.get_state()
    assert (st[1] == g['rs_key']).all() and st[2] == int(g['rs_pos'])

    def predict(u, i):
        rows = ob.table_rows(i, H, P[1].shape[0], 0)
        return oex.transform(loss, (P[1][rows].sum(1) * P[0][u]).sum(1) + P[2][u, 0] + P[3][i, 0])
    I = int(g['num_items'])
    u = int(g['predict_user'])
    assert_close(predict(np.full(I, u), np.arange(I)), g['predict'], 1e-5, what='predict')
    pred = predict(g['test_users'].astype(np.int64), g['test_items'].astype(np.int64))
    rmse = np.sqrt(((g['test_ratings'] - pred) ** 2).mean())
    assert_close(rmse, float(g['rmse']), 1e-5, what='rmse')


@pytest.mark.parametrize('loss', ebc.LOSSES)
def test_plain_tables_are_the_explicit_step(loss):
    case = ebc.make_case(32, loss, 0, 0, -1, seed=5)
    a = ebc.step(case)
    b = oex.explicit_step(*ebc.bc.tables64(case), case['users'], case['items'], case['ratings'], loss)
    assert_close(a['loss'], b['loss'], 1e-12, what='loss')
    assert_close(a['pos'], b['scores'], 1e-12, what='scores')
    for k in ('dWu', 'dWi', 'dbu', 'dbi'):
        assert_close(a[k], b[k], 1e-12, atol=1e-15, what=k)


@pytest.mark.parametrize('loss', ebc.LOSSES)
@pytest.mark.parametrize('opt,wd', [('sgd', 0.1), ('adagrad', 0.1)])
def test_plain_tables_are_the_explicit_fused_step(loss, opt, wd):
    case = ebc.make_case(32, loss, 0, 0, -1, seed=6)
    P1, P2 = ebc.bc.tables64(case), ebc.bc.tables64(case)
    S1 = [np.full(p.shape, 1e-3) for p in P1] if opt == 'adagrad' else None
    S2 = [s.copy() for s in S1] if S1 else None
    a = ebc.step(case, P1, opt, 0.05, wd, S1)
    b = oex.fused_step(P2, case['users'], case['items'], case['ratings'], loss, opt, 0.05, wd, 1e-10, S2)
    assert_close(a['loss'], b['loss'], 1e-12)
    for x, y in zip(P1 + (S1 or []), P2 + (S2 or [])):
        assert_close(x, y, 1e-12)


@pytest.mark.parametrize('entry', ebc.matrix(), ids=lambda e: '%d-%s-%d,%d-pad%d' % e[:5])
def test_matrix_cases_have_their_properties(entry):
    case = ebc.case_for(*entry)
    assert ebc.check_properties(case, ebc.step(case)) == []


def outcome(case, opt, wd_on, mutate=()):
    """What the GPU suite compares: the loss and the update / state change of every table (fused),
    and the dense gradients and scores."""
    lr, wd, S0 = ebc.hparams(case, opt, wd_on)
    P0 = ebc.bc.tables64(case)
    P = [p.copy() for p in P0]
    S = [s.astype(np.float64) for s in S0] if S0 else None
    out = ebc.step(case, P, opt, lr, wd, S, mutate=mutate)
    dense = ebc.step(case, mutate=mutate)
    res = dict(loss=np.array(out['loss']), pos=dense['pos'])
    for k, nm in enumerate(TABLES):
        res[nm] = P[k] - P0[k]
        res['d' + nm] = dense['d' + nm]
        if S:
            res['s' + nm] = S[k] - S0[k]
    return res


def differs(ref, mut):
    for k in ref:
        try:
            assert_close(mut[k], ref[k], 1e-5, what=k)
        except AssertionError:
            return True
    return False


# (mutation, case entry, opt, wd_on): a case and optimizer on which the mistake shows
CATCH = [
    ('pad_hashed', (32, 'regression', 0, 3, 0, 11), 'sgd', False),
    ('freeze_row0', (20, 'poisson', 2, 3, 3, 12), 'sgd', False),
    ('item_mean', (64, 'logistic', 0, 24, 0, 14), 'sgd', False),
    ('item_first_hash', (8, 'regression', 0, 3, -1, 13), 'sgd', False),
    ('dup_row_once', (12, 'regression', 2, 3, -1, 15), 'sgd', False),
    ('stash_post_update', (32, 'regression', 2, 3, 0, 18), 'sgd', False),
    ('poisson_grad_on_s', (100, 'poisson', 0, 3, 3, 19), 'adagrad', True),
    ('logistic_no_clamp', (128, 'logistic', 2, 0, 0, 20), 'sgd', True),
]


@pytest.mark.parametrize('mutation,entry,opt,wd_on', CATCH, ids=['%s-%d' % (c[0], k) for k, c in enumerate(CATCH)])
def test_catches_mutation(mutation, entry, opt, wd_on):
    case = ebc.case_for(*entry)
    assert ebc.check_properties(case, ebc.step(case)) == []
    ref = outcome(case, opt, wd_on)
    assert not differs(ref, outcome(case, opt, wd_on))
    assert differs(ref, outcome(case, opt, wd_on, (mutation,)))


def test_catches_full_batch_norm():
    """A short last batch normalised by the full batch size moves the fit() trajectory."""
    g = load_golden('fit_explicit_bloom_sgd')
    assert len(g['users']) % int(g['batch']) != 0        # the epoch ends with a short batch

    def final(mutate):
        P = [g['init.' + k].astype(np.float64) for k in _names(g)]
        rs = np.random.RandomState()
        rs.set_state(('MT19937', g['rs0_key'], int(g['rs0_pos'])))
        oeb.fit(P, g['users'], g['items'], g['ratings'], str(g['loss_kind']), int(g['batch']), 1, rs, 'sgd',
                float(g['lr']), Hi=int(g['bloom_H']), pad_i=0, mutate=mutate)
        return P
    clean, bad = final(()), final(('full_batch_norm',))
    assert not all(np.abs(b - c).max() <= 1e-5 * np.abs(c).max() for b, c in zip(bad, clean))
