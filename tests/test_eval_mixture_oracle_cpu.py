"""Pin the float64 all-items mixture head (oracle.mixture_eval.score_items) against the live reference's
MixtureLSTMNet predict rows recorded in tests/golden/eval_mixture.npz, and the NumPy evaluation
oracle over those rows against the reference's sequence_mrr_score / sequence_precision_recall_score.

The final representation comes from the fixture's state through oracle.mixture's LSTM and
projection; a Bloom item layer is read as its virtual table (the summed hashed rows)."""

import numpy as np
import pytest

from conftest import load_golden
from oracle import evaluation as oev
from oracle import mixture as om
from oracle import mixture_eval as ome
from oracle import seq_bloom as sb

MODELS = ('mixture', 'm2', 'bloom')
KS = (1, 3)


def _items(g, name):
    I = int(g['num_items'])
    if name + '.bloom' in g:
        return sb.virtual_table(g[name + '.sd.item_embeddings.embeddings.weight'], I, int(g[name + '.bloom'][1]))
    return g[name + '.sd.item_embeddings.weight'].astype(np.float64)


def oracle_rows(g, name, k):
    """(N, I) float64 scores of every item after seqs[:, :-k] under the fixture's model."""
    pre = name + '.sd.'
    M, D = int(g[name + '.num_mixtures']), int(g['dim'])
    E = _items(g, name)
    lstm = dict(w_ih=g[pre + 'lstm.weight_ih_l0'], w_hh=g[pre + 'lstm.weight_hh_l0'],
                b_ih=g[pre + 'lstm.bias_ih_l0'], b_hh=g[pre + 'lstm.bias_hh_l0'])
    proj = dict(w=g[pre + 'projection.weight'], b=g[pre + 'projection.bias'])
    seqs = g['seqs'][:, :-k].astype(np.int64)
    P, _ = om.mixture_representation(E, lstm, proj, seqs, M, dtype=np.float64)
    final = P[:, -1].reshape(len(seqs), 2 * M, D)
    return ome.score_items(final, E, g[pre + 'item_biases.weight'], M)


def test_golden_is_small():
    g = load_golden('eval_mixture')
    assert sum(v.nbytes for v in g.values()) < 200_000


@pytest.mark.parametrize('name', MODELS)
@pytest.mark.parametrize('k', KS)
def test_score_items_equals_reference_predict(name, k):
    g = load_golden('eval_mixture')
    got = oracle_rows(g, name, k)
    want = g['%s.scores.k%d' % (name, k)].astype(np.float64)
    assert got.shape == want.shape
    atol = 1e-5 * np.abs(want).max(axis=1, keepdims=True)
    assert (np.abs(got - want) <= 1e-5 * np.abs(want) + atol).all(), np.abs(got - want).max()


@pytest.mark.parametrize('name', MODELS)
@pytest.mark.parametrize('ex', [False, True])
def test_metrics_over_oracle_rows_equal_reference(name, ex):
    g = load_golden('eval_mixture')
    seqs = g['seqs']
    rows = oracle_rows(g, name, 1)
    mrr = oev.mrr(rows, seqs[:, -1:], seqs[:, :-1] if ex else None)
    np.testing.assert_allclose(mrr, g['%s.mrr.ex%d' % (name, ex)], rtol=1e-6)
    for k in KS:
        rows = oracle_rows(g, name, k)
        p, r = oev.precision_recall(rows, seqs[:, -k:], [k], seqs[:, :-k] if ex else None, recall_denominator=k)
        assert np.array_equal(p[:, 0], g['%s.pr.ex%d.k%d.p' % (name, ex, k)]), k
        assert np.array_equal(r[:, 0], g['%s.pr.ex%d.k%d.r' % (name, ex, k)]), k
