"""The explicit-feedback oracle (oracle/explicit.py) against the live reference's fixtures, and
the GPU tolerance against plausible kernel mistakes.  No GPU needed."""

import os

import numpy as np
import pytest

from oracle import explicit as oex

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
TOL = 1e-5          # tests/test_explicit_gpu.py: loss, scores and gradients within 1e-5 of max|ref|


def _load(name):
    return dict(np.load(os.path.join(GOLDEN, name + '.npz')))


def _params(g, prefix):
    return [g[prefix + k].astype(np.float64).copy() for k in
            ('user_embeddings.weight', 'item_embeddings.weight', 'user_biases.weight', 'item_biases.weight')]


def _within(actual, expected, tol=TOL):
    actual, expected = np.asarray(actual, np.float64), np.asarray(expected, np.float64)
    return np.abs(actual - expected).max() <= tol * max(np.abs(expected).max(), 1e-30)


def _step(g, loss, mutate=()):
    return oex.explicit_step(g['sd.user_embeddings.weight'], g['sd.item_embeddings.weight'],
                             g['sd.user_biases.weight'], g['sd.item_biases.weight'], g['users'], g['items'],
                             g['ratings'], loss, mutate=mutate)


def _step_ok(g, out, loss):
    # the fixture's predictions are what the reference hands its loss: exp(s) for poisson, else s
    loss_input = out['pred'] if loss == 'poisson' else out['scores']
    return (_within(out['loss'], g['loss']) and _within(loss_input, g['pred']) and
            all(_within(out[k].reshape(g['grad.' + n].shape), g['grad.' + n]) for k, n in
                (('dWu', 'user_embeddings.weight'), ('dWi', 'item_embeddings.weight'),
                 ('dbu', 'user_biases.weight'), ('dbi', 'item_biases.weight'))))


@pytest.mark.parametrize('loss', oex.LOSSES)
def test_oracle_step_matches_reference(loss):
    g = _load('explicit_' + loss)
    assert _step_ok(g, _step(g, loss), loss)


@pytest.mark.parametrize('name,opt', [('fit_explicit_poisson', 'sgd'), ('fit_explicit_logistic', 'adagrad')])
def test_oracle_fit_matches_reference(name, opt):
    g = _load(name)
    params = _params(g, 'init.')
    states = [np.zeros_like(p) for p in params]
    rs = np.random.RandomState(int(g['seed']))
    rs.randint(-10**8, 10**8)                        # the constructor's set_seed draw
    loss = name.split('_')[-1]
    losses = oex.fit(params, g['users'].astype(np.int64), g['items'].astype(np.int64), g['ratings'], loss,
                     int(g['batch']), int(g['n_iter']), rs, opt, float(g['lr']), states=states)
    np.testing.assert_allclose(losses, g['epoch_losses'], rtol=1e-5)
    for p, ref in zip(params, _params(g, 'final.')):
        assert _within(p, ref)
    assert rs.get_state()[2] == int(g['rs_pos'])
    assert np.array_equal(rs.get_state()[1], g['rs_key'])
    Wu, Wi, bu, bi = params
    u, i = g['test_users'].astype(np.int64), g['test_items'].astype(np.int64)
    pred = oex.transform(loss, (Wu[u] * Wi[i]).sum(1) + bu[u, 0] + bi[i, 0])
    assert _within(pred, g['predict_pairs'])
    rmse = np.sqrt(((g['test_ratings'] - pred) ** 2).mean())
    assert abs(rmse - float(g['rmse'])) <= TOL * float(g['rmse'])


@pytest.mark.parametrize('loss,mutation', [
    ('regression', 'regression_no_factor2'),
    ('poisson', 'poisson_grad_r_minus_p'),
    ('poisson', 'poisson_grad_on_s'),
    ('logistic', 'logistic_no_clamp'),
    ('regression', 'no_user_bias_grad'),
    ('logistic', 'no_user_bias_grad'),
])
def test_tolerance_catches_step_mistakes(loss, mutation):
    g = _load('explicit_' + loss)
    assert _step_ok(g, _step(g, loss), loss)
    assert not _step_ok(g, _step(g, loss, (mutation,)), loss)


def _fit_final(g, loss, opt, mutate=(), weight_decay=0.0):
    params = _params(g, 'init.')
    states = [np.zeros_like(p) for p in params]
    rs = np.random.RandomState(int(g['seed']))
    rs.randint(-10**8, 10**8)
    oex.fit(params, g['users'].astype(np.int64), g['items'].astype(np.int64), g['ratings'], loss,
            int(g['batch']), 1, rs, opt, float(g['lr']), weight_decay=weight_decay, states=states,
            mutate=mutate)
    return params


def test_tolerance_catches_full_batch_norm():
    g = _load('fit_explicit_poisson')
    assert len(g['users']) % int(g['batch']) != 0        # the epoch ends with a short batch
    clean = _fit_final(g, 'poisson', 'sgd')
    bad = _fit_final(g, 'poisson', 'sgd', ('full_batch_norm',))
    assert not all(_within(b, c) for b, c in zip(bad, clean))


def test_tolerance_catches_skipped_decay():
    g = _load('fit_explicit_logistic')
    clean = _fit_final(g, 'logistic', 'sgd', weight_decay=0.05)
    bad = _fit_final(g, 'logistic', 'sgd', ('no_decay_items',), weight_decay=0.05)
    assert not all(_within(b, c) for b, c in zip(bad, clean))
