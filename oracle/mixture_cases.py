"""MixtureLSTMNet sequence-step test cases.

TEST INFRASTRUCTURE ONLY (tests/test_mixture_gpu.py, tests/test_mixture_oracle_cpu.py).

``make_case`` draws the minibatch and the ``nn.LSTM`` parameters of ``oracle.lstm_cases.make_case``
and adds the ``nn.Conv1d(D, 2MD, 1)`` projection, scaled on the case's own hidden states so the
mixture logits v_m . e and the taste scores c_m . e spread by about 0.85 RMS.  ``check_properties``
adds to the LSTM checks that the mixture weights are neither saturated nor uniform, so the
softmax and its (z_m - s_bar) gradient path are measured.
"""

import numpy as np

from oracle import lstm as olstm
from oracle import lstm_cases as lc
from oracle import mixture as omix


def _projection(case, M, rs):
    D = case['E'].shape[1]
    h, _ = olstm.lstm_representation(case['E'], case['lstm'], case['seqs'], np.float64)
    rms_h = max(float(np.sqrt((h ** 2).mean())), 1e-3)
    # projected entries of RMS ~0.6; with |e|^2 ~ 2 their dots with an item row have RMS ~0.85
    w = (rs.randn(2 * M * D, D, 1) * (0.6 / (rms_h * np.sqrt(D)))).astype(np.float32)
    b = (rs.randn(2 * M * D) * 0.1).astype(np.float32)
    return dict(w=w, b=b)


def make_case(D=32, S=9, B=8, I=400, loss='bpr', n_neg=1, M=4, seed=0, **kw):
    """One minibatch: the dict of ``lstm_cases.make_case`` with net = 'mixture', M and
    proj = dict(w (2MD, D, 1), b (2MD,)).  ``kw``: seq_cases.make_case's padding / draw switches."""
    case = lc.make_case(D=D, S=S, B=B, I=I, loss=loss, n_neg=n_neg, seed=seed, **kw)
    case['net'] = 'mixture'
    case['M'] = M
    case['proj'] = _projection(case, M, np.random.RandomState(seed + 104729))
    return case


def oracle_step(case, dtype=np.float64, mutate=(), negs=None):
    """oracle.mixture.mixture_step on a case (``negs`` override)."""
    return omix.mixture_step(case['E'], case['bias'], case['lstm'], case['proj'], case['seqs'],
                             case['negs'] if negs is None else negs, case['M'], case['loss'], case['n_neg'],
                             dtype, mutate)


def oracle_representation(case, dtype=np.float64, mutate=()):
    """The projection output at all S+1 positions, (B, S+1, 2MD)."""
    return omix.mixture_representation(case['E'], case['lstm'], case['proj'], case['seqs'], case['M'],
                                       dtype, mutate)[0]


def check_properties(case, ref):
    """lstm_cases.check_properties plus, for M >= 2: the largest mixture weight of the target is
    below 0.99 at >= 99 % of the positions, and the weights are not uniform (their max - min
    averages at least 0.1)."""
    bad = lc.check_properties(case, ref)
    if case['M'] >= 2:
        w = ref['w_pos'].reshape(-1, case['M'])
        wmax = w.max(1)
        if float((wmax < 0.99).mean()) < 0.99:
            bad.append('mixture weights saturated at %.3f of the positions' % float((wmax >= 0.99).mean()))
        spread = float((wmax - w.min(1)).mean())
        if spread < 0.1:
            bad.append('mixture weights near uniform (mean max - min %.3f)' % spread)
    return bad


# ------------------------------------------------------------------ live-reference fixtures
# The compact D = 128 fixture stores seeds for the LSTM weight matrices (lstm_cases.seeded_lstm_weights)
# and the projection weight, and the projection's weight gradient at PROJ_ROWS_PER_BLOCK seeded rows
# of each of its 2M blocks.
PROJ_ROWS_PER_BLOCK = 16


def seeded_projection_weight(seed, D, M):
    """float32 (2MD, D, 1), drawn like nn.Conv1d's default init: U(-1/sqrt(D), 1/sqrt(D))."""
    rs = np.random.RandomState(seed + 2)
    k = 1.0 / np.sqrt(D)
    return rs.uniform(-k, k, (2 * M * D, D, 1)).astype(np.float32)


def sampled_proj_rows(seed, D, M):
    """Sorted rows of a compact fixture's projection weight gradient: PROJ_ROWS_PER_BLOCK of each block."""
    rs = np.random.RandomState(seed + 3)
    n = min(PROJ_ROWS_PER_BLOCK, D)
    return np.concatenate([j * D + np.sort(rs.choice(D, n, replace=False)) for j in range(2 * M)]).astype(np.int64)


def golden_params(g):
    """(lstm dict, proj dict, LSTM gradient rows or None, projection gradient rows or None) of a
    step fixture, float32 numpy."""
    lstm, rows = lc.golden_lstm(g)
    if 'proj_weight_seed' in g:
        w = seeded_projection_weight(int(g['proj_weight_seed']), int(g['dim']), int(g['num_mixtures']))
        w = w * np.float32(g['proj_weight_scale'])
    else:
        w = g['sd.projection.weight']
    proj = dict(w=w, b=g['sd.projection.bias'])
    return lstm, proj, rows, (g['proj_rows'] if 'proj_rows' in g else None)
