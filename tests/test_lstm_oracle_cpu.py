"""The float64 LSTMNet oracle against the live reference's fixtures, and the tolerances of
tests/test_lstm_gpu.py against plausible recurrence-kernel mistakes.  Runs without a GPU.

Each mutation check restates one mistake as a mutated oracle call on a case of the GPU suite and
asserts that the GPU comparison (loss and scores 1e-5, gradients 2e-5, relative to the tensor's
maximum) fails between the correct and the mutated result."""

import numpy as np
import pytest

from conftest import assert_close, load_golden
from oracle import lstm as olstm
from oracle import lstm_cases as lc
from oracle import seq_cases as sc

STEP_TOL = dict(pos=1e-5, loss=1e-5, dE=2e-5, dbias=2e-5)
LSTM_KEYS = ('w_ih', 'w_hh', 'b_ih', 'b_hh')


@pytest.mark.parametrize('name,loss', [('lstm_pointwise', 'pointwise'), ('lstm_adaptive_hinge', 'adaptive_hinge'),
                                       ('lstm_bpr_d128', 'bpr')])
def test_oracle_matches_reference_golden(name, loss):
    g = load_golden(name)
    n_neg = int(g['n_neg']) if loss == 'adaptive_hinge' else 1
    lstm, rows = lc.golden_lstm(g)
    ref = olstm.lstm_step(g['sd.item_embeddings.weight'], g['sd.item_biases.weight'], lstm, g['seqs'],
                          g['negs'], loss, n_neg, np.float64)
    assert_close(ref['pos'], g['pos'], 1e-5, what='pos')
    assert_close(ref['neg'].reshape(g['neg'].shape), g['neg'], 1e-5, what='neg')
    assert_close(ref['loss'], g['loss'], 1e-5, what='loss')
    assert_close(ref['final'], g['final'], 1e-5, what='final')
    assert_close(ref['dE'], g['grad.item_embeddings.weight'], 2e-5, what='dE')
    assert_close(ref['dbias'], g['grad.item_biases.weight'], 2e-5, what='dbias')
    for k, tag in zip(LSTM_KEYS, ('weight_ih_l0', 'weight_hh_l0', 'bias_ih_l0', 'bias_hh_l0')):
        d = ref['dlstm'][k]
        assert_close(d if rows is None or d.ndim == 1 else d[rows], g['grad.lstm.' + tag], 2e-5, what=k)


def test_compact_fixture_weights():
    """The D = 128 fixture stores a seed for the LSTM weight matrices and their gradients at a seeded
    sample of rows; the regenerated weights are float32 draws inside nn.LSTM's init range."""
    g = load_golden('lstm_bpr_d128')
    lstm, rows = lc.golden_lstm(g)
    D = int(g['dim'])
    assert 'sd.lstm.weight_ih_l0' not in g and lstm['w_ih'].shape == (4 * D, D) and lstm['w_hh'].dtype == np.float32
    assert np.abs(lstm['w_hh']).max() <= 1 / np.sqrt(D) and np.unique(lstm['w_ih']).size > 0.99 * lstm['w_ih'].size
    assert np.array_equal(rows, lc.sampled_grad_rows(int(g['lstm_weight_seed']), D))
    assert all(((rows >= q * D) & (rows < (q + 1) * D)).sum() == lc.GRAD_ROWS_PER_GATE for q in range(4))
    assert g['grad.lstm.weight_hh_l0'].shape == (rows.size, D)


def differs(ref, mut):
    """True when at least one compared tensor misses its tolerance."""
    pairs = [(k, mut[k], ref[k], r) for k, r in STEP_TOL.items()]
    pairs += [(k, mut['dlstm'][k], ref['dlstm'][k], 2e-5) for k in LSTM_KEYS]
    for what, a, e, rtol in pairs:
        try:
            assert_close(a, e, rtol, what=what)
        except AssertionError:
            return True
    return False


def lstm_case(D=32, **kw):
    args = dict(S=20, B=16, loss='bpr', seed=7)
    args.update(kw)
    return lc.make_case(D=D, **args)


@pytest.mark.parametrize('D', [4, 32, 128, 256])
def test_case_properties_hold(D):
    """The generator's scale checks pass: gates unsaturated, hinge activity, sigmoid range."""
    for loss in sc.LOSS_CYCLE:
        case = lstm_case(D, loss=loss, n_neg=2)
        assert lc.check_properties(case, lc.oracle_step(case)) == [], loss


MUTATIONS = ['swap_if', 'no_zero_step', 'no_b_hh', 'dc_no_f', 'dwhh_ht', 'skip_padding']


@pytest.mark.parametrize('mutation', MUTATIONS)
@pytest.mark.parametrize('D', [32, 128])
def test_catches_mutation(D, mutation):
    case = lstm_case(D)
    assert differs(lc.oracle_step(case), lc.oracle_step(case, mutate=(mutation,)))


def test_mutations_change_only_what_they_name():
    """The forward-only mistakes move the representation; the BPTT ones leave it exact."""
    case = lstm_case(32)
    rep = lc.oracle_representation(case)
    for m in ('swap_if', 'no_zero_step', 'no_b_hh', 'skip_padding'):
        assert np.abs(lc.oracle_representation(case, mutate=(m,)) - rep).max() > 1e-3, m
    ref = lc.oracle_step(case)
    for m in ('dc_no_f', 'dwhh_ht'):
        mut = lc.oracle_step(case, mutate=(m,))
        assert mut['loss'] == ref['loss'] and np.array_equal(mut['pos'], ref['pos']), m
