"""Pin the NumPy restatement of the evaluation scorers (oracle/evaluation.py) against the live
reference's mrr_score / precision_recall_score / sequence_mrr_score /
sequence_precision_recall_score outputs recorded in tests/golden/eval_metrics.npz, given the
score rows the reference ranked."""

import numpy as np
import pytest
import scipy.sparse as sp

from conftest import load_golden
from oracle import evaluation as oev


def _csr(users, items, U, I):
    return sp.coo_matrix((np.ones(len(users), np.float32), (users, items)), shape=(U, I)).tocsr()


def test_golden_is_small():
    g = load_golden('eval_metrics')
    assert sum(v.nbytes for v in g.values()) < 200_000


@pytest.mark.parametrize('with_train', [False, True])
def test_mf_scorers_golden(with_train):
    g = load_golden('eval_metrics')
    U, I = int(g['num_users']), int(g['num_items'])
    test = _csr(g['test_users'], g['test_items'], U, I)
    train = _csr(g['train_users'], g['train_items'], U, I)
    users = np.nonzero(np.diff(test.indptr))[0]
    rows = g['mf_scores'][users]
    targets = [test[u].indices for u in users]
    excluded = [train[u].indices for u in users] if with_train else None
    tag = 'train' if with_train else 'notrain'
    np.testing.assert_allclose(oev.mrr(rows, targets, excluded), g['mrr.' + tag], rtol=1e-6)
    for ktag, k in (('1', 1), ('3', 3), ('list', [1, 5, 10])):
        p, r = oev.precision_recall(rows, targets, k, excluded)
        assert np.array_equal(p.squeeze(), g['pr.%s.k%s.p' % (tag, ktag)])
        assert np.array_equal(r.squeeze(), g['pr.%s.k%s.r' % (tag, ktag)])


@pytest.mark.parametrize('rep', ['pooling', 'cnn', 'lstm'])
@pytest.mark.parametrize('ex', [False, True])
def test_sequence_scorers_golden(rep, ex):
    g = load_golden('eval_metrics')
    seqs = g['seqs']
    rows = g['seq.%s.scores.k1' % rep]
    got = oev.mrr(rows, seqs[:, -1:], seqs[:, :-1] if ex else None)
    np.testing.assert_allclose(got, g['seq.%s.mrr.ex%d' % (rep, ex)], rtol=1e-6)
    for k in (1, 3):
        rows = g['seq.%s.scores.k%d' % (rep, k)]
        p, r = oev.precision_recall(rows, seqs[:, -k:], k, seqs[:, :-k] if ex else None, recall_denominator=k)
        assert np.array_equal(p[:, 0], g['seq.%s.pr.ex%d.k%d.p' % (rep, ex, k)])
        assert np.array_equal(r[:, 0], g['seq.%s.pr.ex%d.k%d.r' % (rep, ex, k)])
