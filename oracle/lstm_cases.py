"""LSTMNet sequence-step test cases.

TEST INFRASTRUCTURE ONLY (tests/test_lstm_gpu.py, tests/test_lstm_oracle_cpu.py).

``make_case`` draws the minibatch of ``oracle.seq_cases.make_case`` (same item table, biases,
sequences, negatives and padding edges) and adds ``nn.LSTM`` parameters scaled so the gates
stay in their working range; ``check_properties`` adds a gate-saturation check to
``oracle.seq_cases.check_properties``.  Row updates and the optimizer restatements are those
of ``oracle.seq_cases``.
"""

import numpy as np

from oracle import lstm as olstm
from oracle import seq_cases as sc


def make_case(D=32, S=9, B=8, I=400, loss='bpr', n_neg=1, seed=0, **kw):
    """One minibatch: the dict of ``seq_cases.make_case`` with net = 'lstm' and
    lstm = dict(w_ih, w_hh, b_ih, b_hh).  ``kw``: make_case's padding / draw switches."""
    case = sc.make_case('pool', D=D, S=S, B=B, I=I, loss=loss, n_neg=n_neg, seed=seed, **kw)
    case['net'] = 'lstm'
    rs = np.random.RandomState(seed + 7919)
    # gate pre-activation RMS ~0.8: the input projection gives ~0.7 (|x|^2 ~ 2), the
    # recurrence and the biases the rest
    case['lstm'] = dict(w_ih=(rs.randn(4 * D, D) * 0.5).astype(np.float32),
                        w_hh=(rs.randn(4 * D, D) / np.sqrt(D)).astype(np.float32),
                        b_ih=(rs.randn(4 * D) * 0.2).astype(np.float32),
                        b_hh=(rs.randn(4 * D) * 0.2).astype(np.float32))
    return case


def oracle_step(case, dtype=np.float64, mutate=(), lstm=None, negs=None):
    """oracle.lstm.lstm_step on a case (``lstm`` / ``negs`` override)."""
    return olstm.lstm_step(case['E'], case['bias'], case['lstm'] if lstm is None else lstm, case['seqs'],
                           case['negs'] if negs is None else negs, case['loss'], case['n_neg'], dtype, mutate)


def oracle_representation(case, dtype=np.float64, mutate=()):
    """All S+1 hidden states, (B, S+1, D)."""
    return olstm.lstm_representation(case['E'], case['lstm'], case['seqs'], dtype, mutate)[0]


def check_properties(case, ref):
    """seq_cases.check_properties plus: at most 1 % of the gate activations saturated (a sigmoid
    within 0.005 of 0 or 1, tanh beyond +-0.99)."""
    bad = sc.check_properties(case, ref)
    _, sv = olstm.lstm_representation(case['E'], case['lstm'], case['seqs'], np.float64)
    g = sv['gates']                                          # (B, T, 4, D): sigmoid i, f, o; tanh g
    span = np.concatenate([np.abs(g[:, :, [0, 1, 3]] - 0.5) * 2, np.abs(g[:, :, 2:3])], axis=2)
    sat = float((span > 0.99).mean())
    if sat > 0.01:
        bad.append('LSTM gates saturated at %.3f of the entries' % sat)
    return bad


# ------------------------------------------------------------------ live-reference fixtures
# A D = 128 fixture holding both (4D, D) weight matrices and both gradients would take 1 MB.  The
# compact fixtures therefore store a seed instead of the two weight matrices (NumPy's legacy
# RandomState stream is fixed, so the generator and the tests draw the same float32 values) and
# the weight gradients at a seeded sample of rows: GRAD_ROWS_PER_GATE rows of each gate block.
GRAD_ROWS_PER_GATE = 32


def seeded_lstm_weights(seed, D):
    """(w_ih, w_hh), float32 (4D, D), drawn like nn.LSTM's default init: U(-1/sqrt(D), 1/sqrt(D))."""
    rs = np.random.RandomState(seed)
    k = 1.0 / np.sqrt(D)
    return (rs.uniform(-k, k, (4 * D, D)).astype(np.float32),
            rs.uniform(-k, k, (4 * D, D)).astype(np.float32))


def sampled_grad_rows(seed, D):
    """Sorted gate rows of a compact fixture's weight gradients: GRAD_ROWS_PER_GATE of each gate."""
    rs = np.random.RandomState(seed + 1)
    n = min(GRAD_ROWS_PER_GATE, D)
    return np.concatenate([g * D + np.sort(rs.choice(D, n, replace=False)) for g in range(4)]).astype(np.int64)


def golden_lstm(g):
    """(lstm parameter dict (float32 numpy), gradient row ids or None) of a step fixture."""
    if 'lstm_weight_seed' in g:
        w_ih, w_hh = seeded_lstm_weights(int(g['lstm_weight_seed']), int(g['dim']))
    else:
        w_ih, w_hh = g['sd.lstm.weight_ih_l0'], g['sd.lstm.weight_hh_l0']
    lstm = dict(w_ih=w_ih, w_hh=w_hh, b_ih=g['sd.lstm.bias_ih_l0'], b_hh=g['sd.lstm.bias_hh_l0'])
    return lstm, (g['grad_rows'] if 'grad_rows' in g else None)
