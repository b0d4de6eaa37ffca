"""Generate the evaluation golden fixture (tests/golden/eval_metrics.npz) from the LIVE
reference (build container only).

Run:  SPOTLIGHT_REFERENCE=<reference checkout> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_eval.py

Imports the unmodified reference from the checkout SPOTLIGHT_REFERENCE names (read-only), builds
small models with fixed weights and records their score rows and the reference's
mrr_score / precision_recall_score / sequence_mrr_score / sequence_precision_recall_score
outputs.  The tests read only the committed fixture.
"""

import os
import sys

import numpy as np

sys.dont_write_bytecode = True
sys.path.insert(0, os.environ['SPOTLIGHT_REFERENCE'])

import torch  # noqa: E402

from spotlight.factorization.implicit import ImplicitFactorizationModel  # noqa: E402
from spotlight.interactions import Interactions, SequenceInteractions  # noqa: E402
from spotlight.sequence.implicit import ImplicitSequenceModel  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
torch.set_num_threads(1)


def _state(net):
    return {'sd.' + k: v.detach().cpu().numpy().copy() for k, v in net.state_dict().items()}


def _separated(row):
    """No two scores of the row within 1e-4 of the row's largest magnitude: fp32 summation-order
    differences between implementations then cannot reorder the row."""
    s = np.sort(row.astype(np.float64))
    return bool(np.all(np.diff(s) > 1e-4 * np.abs(s).max()))


def eval_case():
    """The reference's mrr_score / precision_recall_score / sequence_mrr_score /
    sequence_precision_recall_score on small models with fixed weights, with their score rows.
    Users and sequences whose score rows hold a near-tie are redrawn (seeded), so every compared
    ranking is exact; the item count leaves more than max(k) items after any exclusion."""
    from spotlight.evaluation import (mrr_score, precision_recall_score, sequence_mrr_score,
                                      sequence_precision_recall_score)
    rs = np.random.RandomState(21)
    U, I, D = 24, 30, 8
    out = dict(num_users=np.int64(U), num_items=np.int64(I), dim=np.int64(D))
    train = Interactions(rs.randint(0, U, 6 * U).astype(np.int32), rs.randint(0, I, 6 * U).astype(np.int32),
                         num_users=U, num_items=I)
    te_u = rs.randint(0, U - 4, 3 * U).astype(np.int32)          # the last users have no test items
    test = Interactions(te_u, rs.randint(0, I, 3 * U).astype(np.int32), num_users=U, num_items=I)
    assert np.diff(train.tocsr().indptr).max() <= I - 10
    model = ImplicitFactorizationModel(loss='bpr', embedding_dim=D, random_state=np.random.RandomState(21))
    model._initialize(train)
    net = model._net
    with torch.no_grad():
        net.user_biases.weight.copy_(torch.from_numpy(rs.randn(U, 1).astype(np.float32) * 0.1))
        net.item_biases.weight.copy_(torch.from_numpy(rs.randn(I, 1).astype(np.float32) * 0.1))
        for u in range(U):
            for _ in range(100):
                if _separated(model.predict(u)):
                    break
                net.user_embeddings.weight[u] = torch.from_numpy(rs.randn(D).astype(np.float32) / D)
            assert _separated(model.predict(u)), u
    out.update({'mf.' + k: v for k, v in _state(net).items()})
    out.update(train_users=train.user_ids, train_items=train.item_ids, test_users=test.user_ids,
               test_items=test.item_ids, mf_scores=np.stack([model.predict(u) for u in range(U)]))
    for tag, tr in (('notrain', None), ('train', train)):
        out['mrr.' + tag] = mrr_score(model, test, tr)
        for ktag, k in (('1', 1), ('3', 3), ('list', [1, 5, 10])):
            p, r = precision_recall_score(model, test, tr, k=k)
            out['pr.%s.k%s.p' % (tag, ktag)], out['pr.%s.k%s.r' % (tag, ktag)] = p, r

    N, S = 16, 8
    seqs = rs.randint(1, I, (N, S)).astype(np.int32)
    for b in range(0, N, 3):
        seqs[b, :rs.randint(1, S - 3)] = 0                         # leading padding
    seqs[1, 2] = seqs[1, -1]                                       # a target inside its own input
    seqs[2, -2] = seqs[2, -1]                                      # a repeated target
    models = {}
    for rep in ('pooling', 'cnn', 'lstm'):
        m = ImplicitSequenceModel(representation=rep, embedding_dim=D, random_state=np.random.RandomState(22))
        m._initialize(SequenceInteractions(seqs, num_items=I))
        with torch.no_grad():
            b = rs.randn(I, 1).astype(np.float32) * 0.1
            b[0] = 0.0
            m._net.item_biases.weight.copy_(torch.from_numpy(b))
        models[rep] = m
    ks = (1, 3)
    for n in range(N):                                             # redraw rows holding a near-tie
        for _ in range(100):
            if all(_separated(m.predict(seqs[n, :-k])) for m in models.values() for k in ks):
                break
            seqs[n] = rs.randint(1, I, S)
        assert all(_separated(m.predict(seqs[n, :-k])) for m in models.values() for k in ks), n
    out['seqs'] = seqs
    for rep, m in models.items():
        out.update({'seq.%s.%s' % (rep, k): v for k, v in _state(m._net).items()})
        inter = SequenceInteractions(seqs, num_items=I)
        for k in ks:
            out['seq.%s.scores.k%d' % (rep, k)] = np.stack([m.predict(seqs[n, :-k]) for n in range(N)])
        for ex in (False, True):
            out['seq.%s.mrr.ex%d' % (rep, ex)] = sequence_mrr_score(m, inter, exclude_preceding=ex)
            for k in ks:
                p, r = sequence_precision_recall_score(m, inter, k=k, exclude_preceding=ex)
                out['seq.%s.pr.ex%d.k%d.p' % (rep, ex, k)], out['seq.%s.pr.ex%d.k%d.r' % (rep, ex, k)] = p, r
    np.savez_compressed(os.path.join(HERE, 'eval_metrics.npz'), **out)


if __name__ == '__main__':
    eval_case()
