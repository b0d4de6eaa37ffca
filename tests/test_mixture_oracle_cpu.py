"""The float64 MixtureLSTMNet oracle against the live reference's fixtures, and the tolerances of
tests/test_mixture_gpu.py against plausible mistakes of the mixture head and its projection.  Runs
without a GPU.

Each mutation check restates one mistake as a mutated oracle call on a case of the GPU suite and
asserts that the GPU comparison (loss and scores 1e-5, gradients 2e-5, relative to the tensor's
maximum) fails between the correct and the mutated result."""

import numpy as np
import pytest

from conftest import assert_close, load_golden
from oracle import mixture as omix
from oracle import mixture_cases as mc
from oracle import seq_cases as sc

STEP_TOL = dict(pos=1e-5, loss=1e-5, dE=2e-5, dbias=2e-5)
LSTM_KEYS = ('w_ih', 'w_hh', 'b_ih', 'b_hh')
STEP_GOLDENS = [('mixture_pointwise', 'pointwise'), ('mixture_adaptive_hinge', 'adaptive_hinge'),
                ('mixture_bpr_d128', 'bpr')]


@pytest.mark.parametrize('name,loss', STEP_GOLDENS)
def test_oracle_matches_reference_golden(name, loss):
    g = load_golden(name)
    n_neg = int(g['n_neg']) if loss == 'adaptive_hinge' else 1
    M = int(g['num_mixtures'])
    lstm, proj, rows, prows = mc.golden_params(g)
    ref = omix.mixture_step(g['sd.item_embeddings.weight'], g['sd.item_biases.weight'], lstm, proj, g['seqs'],
                            g['negs'], M, loss, n_neg, np.float64)
    B, D = g['seqs'].shape[0], int(g['dim'])
    assert_close(ref['pos'], g['pos'], 1e-5, what='pos')
    assert_close(ref['neg'].reshape(g['neg'].shape), g['neg'], 1e-5, what='neg')
    assert_close(ref['loss'], g['loss'], 1e-5, what='loss')
    assert_close(ref['final'].reshape(g['final'].shape), g['final'], 1e-5, what='final')
    if 'user_rep' in g:                            # (B, 2M, D, S) from the time-major (B, S+1, 2MD)
        rep = omix.mixture_representation(g['sd.item_embeddings.weight'], lstm, proj, g['seqs'], M, np.float64)[0]
        rep = rep[:, :-1].reshape(B, -1, 2 * M, D).transpose(0, 2, 3, 1)
        assert_close(rep, g['user_rep'], 1e-5, what='user_rep')
    assert_close(ref['dE'], g['grad.item_embeddings.weight'], 2e-5, what='dE')
    assert_close(ref['dbias'], g['grad.item_biases.weight'], 2e-5, what='dbias')
    for k, tag in zip(LSTM_KEYS, ('weight_ih_l0', 'weight_hh_l0', 'bias_ih_l0', 'bias_hh_l0')):
        d = ref['dlstm'][k]
        assert_close(d if rows is None or d.ndim == 1 else d[rows], g['grad.lstm.' + tag], 2e-5, what=k)
    dw = ref['dmix']['w']
    assert_close(dw if prows is None else dw[prows], g['grad.projection.weight'], 2e-5, what='dmix w')
    assert_close(ref['dmix']['b'], g['grad.projection.bias'], 2e-5, what='dmix b')


def test_compact_fixture_weights():
    """The D = 128 fixture stores seeds for the LSTM and projection weights and their gradients at
    seeded rows; the regenerated projection is a float32 draw of the stated scale."""
    g = load_golden('mixture_bpr_d128')
    lstm, proj, rows, prows = mc.golden_params(g)
    D, M = int(g['dim']), int(g['num_mixtures'])
    assert 'sd.projection.weight' not in g and proj['w'].shape == (2 * M * D, D, 1) and proj['w'].dtype == np.float32
    assert np.abs(proj['w']).max() <= float(g['proj_weight_scale']) / np.sqrt(D)
    assert np.array_equal(prows, mc.sampled_proj_rows(int(g['proj_weight_seed']), D, M))
    assert all(((prows >= j * D) & (prows < (j + 1) * D)).sum() == mc.PROJ_ROWS_PER_BLOCK for j in range(2 * M))
    assert g['grad.projection.weight'].shape == (prows.size, D, 1)


def test_fit_fixture_shapes():
    g = load_golden('fit_mixture_sgd')
    D = int(g['dim'])
    assert g['init.projection.weight'].shape == (8 * D, D, 1) and len(g['epoch_losses']) == int(g['n_iter'])


def differs(ref, mut):
    """True when at least one compared tensor misses its tolerance."""
    pairs = [(k, mut[k], ref[k], r) for k, r in STEP_TOL.items()]
    pairs += [(k, mut['dlstm'][k], ref['dlstm'][k], 2e-5) for k in LSTM_KEYS]
    pairs += [('dmix ' + k, mut['dmix'][k], ref['dmix'][k], 2e-5) for k in ('w', 'b')]
    for what, a, e, rtol in pairs:
        try:
            assert_close(a, e, rtol, what=what)
        except AssertionError:
            return True
    return False


def mixture_case(D=32, **kw):
    args = dict(S=20, B=16, loss='bpr', seed=7, M=4)
    args.update(kw)
    return mc.make_case(D=D, **args)


@pytest.mark.parametrize('D', [4, 32, 128, 256])
def test_case_properties_hold(D):
    """The generator's scale checks pass: gates and mixture weights unsaturated, weights not
    uniform, hinge activity, sigmoid range."""
    for loss in sc.LOSS_CYCLE:
        for M in (2, 4, 8):
            case = mixture_case(D, loss=loss, n_neg=2, M=M, seed=D + M)
            assert mc.check_properties(case, mc.oracle_step(case)) == [], (loss, M)


MUTATIONS = ['swap_cv', 'softmax_over_d', 'dv_no_sbar', 'de_no_v', 'no_proj_bias', 'proj_hprev']


@pytest.mark.parametrize('mutation', MUTATIONS)
@pytest.mark.parametrize('D', [32, 128])
def test_catches_mutation(D, mutation):
    case = mixture_case(D)
    assert differs(mc.oracle_step(case), mc.oracle_step(case, mutate=(mutation,)))


def test_mutations_change_only_what_they_name():
    """The forward mistakes move the scores; the backward ones leave them exact and move only
    the gradients they name."""
    case = mixture_case(32)
    ref = mc.oracle_step(case)
    for m in ('swap_cv', 'softmax_over_d', 'no_proj_bias', 'proj_hprev'):
        assert np.abs(mc.oracle_step(case, mutate=(m,))['pos'] - ref['pos']).max() > 1e-3, m
    for m in ('dv_no_sbar', 'de_no_v'):
        mut = mc.oracle_step(case, mutate=(m,))
        assert mut['loss'] == ref['loss'] and np.array_equal(mut['pos'], ref['pos']), m
        assert not np.allclose(mut['dE'], ref['dE'], rtol=0, atol=1e-6 * np.abs(ref['dE']).max()), m
    mut = mc.oracle_step(case, mutate=('dv_no_sbar',))
    D, M = 32, case['M']
    assert np.array_equal(mut['dmix']['w'][:M * D], ref['dmix']['w'][:M * D])      # dc untouched


def test_single_mixture_is_lstm_plus_projection():
    """M = 1: every mixture weight is 1, the score is beta + c_0 . e, and the LSTM gradients are
    those of an LSTMNet whose representation is the component block."""
    case = mixture_case(32, M=1, loss='pointwise')
    ref = mc.oracle_step(case)
    assert (ref['w_pos'] == 1.0).all()
    P = mc.oracle_representation(case)
    S = case['seqs'].shape[1]
    c0 = P[:, :S, :32]
    e = case['E'][case['seqs']].astype(np.float64)
    assert_close(ref['pos'], (c0 * e).sum(-1) + case['bias'][case['seqs']][..., 0], 1e-12, what='pos')
