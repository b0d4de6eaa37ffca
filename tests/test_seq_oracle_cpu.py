"""The tolerances of tests/test_seq_oracle_gpu.py catch plausible sequence-kernel mistakes.

Each check restates one mistake as a mutated float64 oracle call on a case of the GPU suite
and asserts that the GPU comparison (conftest.assert_close at the same tolerance) would fail
between the correct and the mutated result.  Runs without a GPU."""

import numpy as np
import pytest

from conftest import assert_close
from oracle import seq_cases as sc

STEP_TOL = dict(pos=1e-5, loss=1e-5, dE=2e-5, dbias=2e-5)


def differs(ref, mut, tol=STEP_TOL):
    """True when at least one compared tensor misses its tolerance."""
    pairs = [(k, mut[k], ref[k], r) for k, r in tol.items()]
    for i, (dW, db) in enumerate(ref.get('dconvs', [])):
        pairs += [('dW%d' % i, mut['dconvs'][i][0], dW, 2e-5), ('db%d' % i, mut['dconvs'][i][1], db, 2e-5)]
    for what, a, e, rtol in pairs:
        try:
            assert_close(a, e, rtol, what=what)
        except AssertionError:
            return True
    return False


def cnn_case(D=32, **kw):
    args = dict(S=20, B=16, loss='bpr', kernel_width=(3, 2), dilation=(2, 1), seed=7)
    args.update(kw)
    return sc.make_case('cnn', D=D, **args)


@pytest.mark.parametrize('D', [32, 128])
def test_case_properties_hold(D):
    """The generator's scale checks pass on cases of the GPU suite (hinge activity, tanh range)."""
    for g, geo in enumerate(sc.GEOMETRIES):
        geo = dict(geo)
        S, B = geo.pop('S'), geo.pop('B')
        case = sc.make_case('cnn', D=D, S=S, B=B, loss=sc.LOSS_CYCLE[(g + (D == 128)) % 4], n_neg=3,
                            seed=100 + g, **geo)
        assert sc.check_properties(case, sc.oracle_step(case)) == [], g


@pytest.mark.parametrize('D', [32, 128])
def test_catches_layer0_pad_rf_minus_1(D):
    case = cnn_case(D)
    assert differs(sc.oracle_step(case), sc.oracle_step(case, mutate=('pad0_rf_minus_1',)))


@pytest.mark.parametrize('D', [32, 128])
def test_catches_last_tap_dropped(D):
    case = cnn_case(D)
    convs = [(W.copy(), b) for W, b in case['convs']]
    for W, _ in convs:
        W[:, :, -1] = 0
    assert differs(sc.oracle_step(case), sc.oracle_step(case, convs=convs))


@pytest.mark.parametrize('D', [32, 128])
def test_catches_dilation_off_by_one(D):
    case = cnn_case(D, dilation=(3, 1))
    ref = sc.oracle_step(case)
    assert differs(ref, sc.oracle_step(case, dilation=[2, 1]))
    assert differs(ref, sc.oracle_step(case, dilation=[4, 1]))


@pytest.mark.parametrize('D', [32, 128])
def test_catches_residual_shift_off_by_one(D):
    case = cnn_case(D)
    assert differs(sc.oracle_step(case), sc.oracle_step(case, mutate=('residual_shift',)))


def test_catches_per_row_nonzero_count():
    """PoolNet counts non-zero entries per element; zero entries inside rows make a per-row count differ."""
    case = sc.make_case('pool', D=32, S=30, B=9, loss='bpr', e0_nonzero=True, zero_frac=0.3, seed=5)
    assert differs(sc.oracle_step(case), sc.oracle_step(case, mutate=('count_per_row',)))


@pytest.mark.parametrize('net,D', [('pool', 32), ('cnn', 32), ('cnn', 128)])
def test_catches_last_maximal_negative_credited(net, D):
    """Crediting the last of two tied negatives instead of the first: the mutated call reverses
    the negatives' order, so the first maximal index becomes the last one."""
    case = sc.make_case(net, D=D, S=20, B=16, loss='adaptive_hinge', n_neg=2, neg_tie=True, seed=11)
    n, (B, S) = case['n_neg'], case['seqs'].shape
    flipped = case['negs'].reshape(n, B, S)[::-1].reshape(n * B, S)
    ref, mut = sc.oracle_step(case), sc.oracle_step(case, negs=flipped)
    assert_close(mut['loss'], ref['loss'], 1e-12)          # the scores tie: the loss cannot tell
    assert differs(ref, mut, dict(dE=2e-5, dbias=2e-5))


@pytest.mark.parametrize('opt', ['sgd', 'adagrad'])
def test_catches_weight_decay_skipped_on_zero_gradient_row(opt):
    """S = 1 PoolNet: every row's embedding gradient is zero (r_0 = 0), its bias gradient is not.
    Decaying only the non-zero 4-element chunks of the gradient (and the bias when its
    gradient is non-zero) leaves those embedding rows undecayed."""
    case = sc.make_case('pool', D=16, S=1, B=64, loss='bpr', seed=3)
    ref = sc.oracle_step(case)
    rows = sc.updated_rows(case, ref)
    g = ref['dE']
    chunk_nz = np.repeat((g.reshape(g.shape[0], -1, 4) != 0).any(axis=2), 4, axis=1)
    assert rows.sum() > 0 and not chunk_nz.any()
    wd, lr = 0.1, 0.05
    if opt == 'sgd':
        good = sc.sgd(case['E'], g, rows[:, None], lr, wd)
        bad = sc.sgd(case['E'], g, chunk_nz, lr, wd)
    else:
        s0 = np.full(case['E'].shape, 0.01)
        good = sc.adagrad(case['E'], s0, g, rows[:, None], lr, wd, 1e-10)[0]
        bad = sc.adagrad(case['E'], s0, g, chunk_nz, lr, wd, 1e-10)[0]
    with pytest.raises(AssertionError):
        assert_close(bad, good, 5e-6, what='E')


def test_updated_rows_follow_the_mf_rule():
    """A row is updated when one of its terms has a non-zero score gradient, even if its
    embedding gradient is zero; the padding row never is."""
    case = sc.make_case('pool', D=16, S=1, B=64, loss='bpr', seed=3)
    ref = sc.oracle_step(case)
    rows = sc.updated_rows(case, ref)
    live = case['seqs'] != 0                       # a term at a padded position has no gradient
    ids = np.unique(np.concatenate([case['seqs'][live], case['negs'][live]]))
    assert not rows[0]
    assert rows[ids[ids != 0]].all() and rows.sum() == (ids != 0).sum()
    assert (ref['dE'][rows] == 0).all() and (ref['dbias'][rows] != 0).all()
