"""Evaluation on the device: slb_rank_targets against slb_rank_pairs and a stable argsort, the
four scorers of spotlight_b200.evaluation against the live reference's outputs
(tests/golden/eval_metrics.npz) and against restated reference loops over model.predict."""

import ctypes

import numpy as np
import pytest
import torch

from conftest import load_golden

pytestmark = pytest.mark.gpu

FLOAT_MAX = np.finfo(np.float32).max


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _rank_both(scores, row_ptr, targets):
    """(slb_rank_targets avg_rank, position, slb_rank_pairs ranks) on the same block."""
    from spotlight_b200 import _lib, ops
    lib = _lib.load()
    R, I = scores.shape
    rp = torch.from_numpy(row_ptr.astype(np.int64)).cuda()
    tg = torch.from_numpy(targets.astype(np.int64)).cuda()
    pr = torch.from_numpy(np.repeat(np.arange(R), np.diff(row_ptr)).astype(np.int64)).cuda()
    n = len(targets)
    avg = torch.full((n,), -1.0, device='cuda')
    pos = torch.full((n,), -1, dtype=torch.int64, device='cuda')
    ref = torch.full((n,), -1.0, device='cuda')
    _lib.check(lib.slb_rank_targets(_p(scores), R, I, _p(rp), _p(tg), n, _p(avg), _p(pos), ops._stream()))
    _lib.check(lib.slb_rank_pairs(_p(scores), R, I, _p(pr), _p(tg), n, _p(ref), ops._stream()))
    return avg.cpu().numpy(), pos.cpu().numpy(), ref.cpu().numpy()


@pytest.mark.parametrize('n_items', [1003, 1024, 6])
def test_rank_targets_vs_rank_pairs_and_stable_argsort(n_items):
    rs = np.random.RandomState(n_items)
    R = 9
    scores = rs.randn(R, n_items).astype(np.float32)
    scores[:, 1::3] = np.round(scores[:, 1::3], 1)                  # many exact ties
    if n_items > 8:
        scores[:, 7] = scores[:, 3]                                 # a duplicated item
    scores[2, rs.randint(0, n_items, n_items // 3)] = -FLOAT_MAX    # excluded items
    counts = [0, 1, 5000, 3, 1, 0, 1100, 2, 40]                     # 0, 1, one and several chunks
    row_ptr = np.concatenate([[0], np.cumsum(counts)])
    targets = rs.randint(0, n_items, row_ptr[-1])                   # duplicates included
    targets[row_ptr[2]] = targets[row_ptr[2] + 1]
    avg, pos, ref = _rank_both(torch.from_numpy(scores).cuda(), row_ptr, targets)
    assert np.array_equal(avg.view(np.int32), ref.view(np.int32))  # bit-identical
    for r in range(R):
        inv = np.empty(n_items, np.int64)
        inv[np.argsort(-scores[r], kind='stable')] = np.arange(n_items)
        sl = slice(row_ptr[r], row_ptr[r + 1])
        assert np.array_equal(pos[sl], inv[targets[sl]]), r


def _golden_mf(g):
    from spotlight_b200.factorization.implicit import ImplicitFactorizationModel
    from spotlight_b200.interactions import Interactions
    U, I = int(g['num_users']), int(g['num_items'])
    train = Interactions(g['train_users'], g['train_items'], num_users=U, num_items=I)
    test = Interactions(g['test_users'], g['test_items'], num_users=U, num_items=I)
    model = ImplicitFactorizationModel(loss='bpr', embedding_dim=int(g['dim']), use_cuda=True)
    model._initialize(train)
    model._net.load_state_dict({k[6:]: torch.from_numpy(v) for k, v in g.items() if k.startswith('mf.sd.')})
    return model, train, test


def test_mf_scorers_match_reference_golden():
    from spotlight_b200.evaluation import mrr_score, precision_recall_score
    g = load_golden('eval_metrics')
    model, train, test = _golden_mf(g)
    for tag, tr in (('notrain', None), ('train', train)):
        got = mrr_score(model, test, tr, user_block=7)
        assert got.shape == g['mrr.' + tag].shape
        np.testing.assert_allclose(got, g['mrr.' + tag], rtol=1e-6)
        for ktag, k in (('1', 1), ('3', 3), ('list', [1, 5, 10])):
            p, r = precision_recall_score(model, test, tr, k=k, user_block=7)
            assert np.array_equal(p, g['pr.%s.k%s.p' % (tag, ktag)]), (tag, ktag)
            assert np.array_equal(r, g['pr.%s.k%s.r' % (tag, ktag)]), (tag, ktag)


@pytest.mark.parametrize('rep', ['pooling', 'cnn', 'lstm'])
def test_sequence_scorers_match_reference_golden(rep):
    from spotlight_b200.evaluation import sequence_mrr_score, sequence_precision_recall_score
    from spotlight_b200.interactions import SequenceInteractions
    from spotlight_b200.sequence.implicit import ImplicitSequenceModel
    g = load_golden('eval_metrics')
    seqs, I = g['seqs'], int(g['num_items'])
    inter = SequenceInteractions(seqs, num_items=I)
    model = ImplicitSequenceModel(representation=rep, embedding_dim=int(g['dim']), use_cuda=True)
    model._initialize(inter)
    pre = 'seq.%s.sd.' % rep
    model._net.load_state_dict({k[len(pre):]: torch.from_numpy(v) for k, v in g.items() if k.startswith(pre)})
    for ex in (False, True):
        got = sequence_mrr_score(model, inter, exclude_preceding=ex, sequence_block=5)
        np.testing.assert_allclose(got, g['seq.%s.mrr.ex%d' % (rep, ex)], rtol=1e-6)
        for k in (1, 3):
            p, r = sequence_precision_recall_score(model, inter, k=k, exclude_preceding=ex, sequence_block=5)
            assert np.array_equal(p, g['seq.%s.pr.ex%d.k%d.p' % (rep, ex, k)]), (ex, k)
            assert np.array_equal(r, g['seq.%s.pr.ex%d.k%d.r' % (rep, ex, k)]), (ex, k)


def _loop_precision_recall(predict_rows, targets, ks, excluded, recall_den=None):
    """The reference loop (evaluation.py:194-215, 131-139) over predict() rows, with the stable
    argsort the device ranks ties by."""
    P, R = [], []
    for r, row in enumerate(predict_rows):
        pred = -row
        if excluded is not None:
            pred[excluded[r]] = FLOAT_MAX
        order = pred.argsort(kind='stable')
        t = set(np.asarray(targets[r]).tolist())
        hits = [len(set(order[:k].tolist()) & t) for k in ks]
        P.append([h / len(order[:k]) for h, k in zip(hits, ks)])
        R.append([h / (recall_den or len(t)) for h in hits])
    return np.array(P), np.array(R)


def _loop_mrr(predict_rows, targets, excluded):
    import scipy.stats as st
    out = []
    for r, row in enumerate(predict_rows):
        pred = -row
        if excluded is not None:
            pred[excluded[r]] = FLOAT_MAX
        out.append((1.0 / st.rankdata(pred)[targets[r]]).mean())
    return np.array(out)


def _statistically_equal(got, want):
    # block scores come from a GEMM, predict() from the gather / elementwise path: two fp32
    # summation orders, so items whose scores differ by ~1e-7 relative may swap for a few rows
    err = np.abs(np.asarray(got, np.float64) - want).reshape(len(want), -1).max(1)
    assert np.median(err) < 1e-7 and (err < 1e-6).mean() > 0.9, (np.median(err), err.max())


def _mf_model(bloom):
    from spotlight_b200 import optim
    from spotlight_b200.factorization.implicit import ImplicitFactorizationModel
    from spotlight_b200.factorization.representations import BilinearNet
    from spotlight_b200.interactions import Interactions
    from spotlight_b200.layers import BloomEmbedding
    rs = np.random.RandomState(1)
    U, I = 300, 120
    train = Interactions(rs.randint(0, U, 4000).astype(np.int32), rs.randint(0, I, 4000).astype(np.int32),
                         num_users=U, num_items=I)
    test = Interactions(rs.randint(0, U, 700).astype(np.int32), rs.randint(0, I, 700).astype(np.int32),
                        num_users=U, num_items=I)
    kw = {}
    if bloom:
        kw = dict(representation=BilinearNet(U, I, 16, item_embedding_layer=BloomEmbedding(I, 16, 0.5, 2)))
    else:
        kw = dict(optimizer_func=optim.fused_adagrad(lr=0.05))
    model = ImplicitFactorizationModel(loss='bpr', embedding_dim=16, n_iter=2, batch_size=256, use_cuda=True,
                                       random_state=np.random.RandomState(2), **kw)
    model.fit(train)
    if not bloom:
        with torch.no_grad():                   # exact ties: two identical item rows
            model._net.item_embeddings.weight[7] = model._net.item_embeddings.weight[3]
            model._net.item_biases.weight[7] = model._net.item_biases.weight[3]
    return model, train, test


@pytest.mark.parametrize('bloom', [False, True])
@pytest.mark.parametrize('with_train', [False, True])
def test_mf_scorers_equal_reference_loop(bloom, with_train):
    from spotlight_b200.evaluation import mrr_score, precision_recall_score
    model, train, test = _mf_model(bloom)
    tcsr, trcsr = test.tocsr(), train.tocsr()
    users = np.nonzero(np.diff(tcsr.indptr))[0]
    rows = np.stack([model.predict(int(u)) for u in users])
    targets = [tcsr[u].indices for u in users]
    excluded = [trcsr[u].indices for u in users] if with_train else None
    ks = [1, 5, 10, 200]                        # 200 > every user's non-excluded items
    p, r = precision_recall_score(model, test, train if with_train else None, k=ks, user_block=64)
    wp, wr = _loop_precision_recall(rows, targets, ks, excluded)
    assert p.shape == wp.shape == (len(users), len(ks))
    _statistically_equal(p, wp)
    _statistically_equal(r, wr)
    assert (r[:, 3] == 1.0).all()              # 200 > num_items: every test item is a hit
    if bloom:
        _statistically_equal(mrr_score(model, test, train if with_train else None, user_block=64),
                             _loop_mrr(rows, targets, excluded))
    # deterministic: a second call is identical
    p2, r2 = precision_recall_score(model, test, train if with_train else None, k=ks, user_block=64)
    assert np.array_equal(p, p2) and np.array_equal(r, r2)


def test_precision_recall_shapes():
    from spotlight_b200.evaluation import precision_recall_score
    from spotlight_b200.interactions import Interactions
    model, train, test = _mf_model(False)
    n = int((np.diff(test.tocsr().indptr) > 0).sum())
    assert precision_recall_score(model, test, k=5)[0].shape == (n,)
    assert precision_recall_score(model, test, k=[1, 5])[1].shape == (n, 2)
    one = Interactions(np.array([4], np.int32), np.array([9], np.int32), num_users=300, num_items=120)
    assert precision_recall_score(model, one, k=5)[0].shape == ()


@pytest.mark.parametrize('rep', ['pooling', 'cnn', 'lstm', 'mixture'])
@pytest.mark.parametrize('ex', [False, True])
def test_sequence_scorers_equal_reference_loop(rep, ex):
    from spotlight_b200.evaluation import sequence_mrr_score, sequence_precision_recall_score
    from spotlight_b200.interactions import SequenceInteractions
    from spotlight_b200.sequence.implicit import ImplicitSequenceModel
    rs = np.random.RandomState(3)
    I, N, S = 2000, 300, 12
    seqs = rs.randint(1, I, (N, S)).astype(np.int32)
    seqs[::4, :5] = 0
    seqs[1::7, 3] = seqs[1::7, -1]
    inter = SequenceInteractions(seqs, num_items=I)
    model = ImplicitSequenceModel(representation=rep, embedding_dim=16, n_iter=1, batch_size=64, use_cuda=True,
                                  random_state=np.random.RandomState(4))
    model.fit(inter)
    with torch.no_grad():                       # exact ties: two identical item rows
        model._net.item_embeddings.weight[7] = model._net.item_embeddings.weight[3]
        model._net.item_biases.weight[7] = model._net.item_biases.weight[3]
    rows = np.stack([model.predict(seqs[n, :-1]) for n in range(N)])
    got = sequence_mrr_score(model, inter, exclude_preceding=ex, sequence_block=64)
    assert got.shape == (N,)
    _statistically_equal(got, _loop_mrr(rows, seqs[:, -1:], seqs[:, :-1] if ex else None))
    assert np.array_equal(got, sequence_mrr_score(model, inter, exclude_preceding=ex, sequence_block=64))
    k = 4
    rows = np.stack([model.predict(seqs[n, :-k]) for n in range(N)])
    p, r = sequence_precision_recall_score(model, inter, k=k, exclude_preceding=ex, sequence_block=64)
    wp, wr = _loop_precision_recall(rows, seqs[:, -k:], [k], seqs[:, :-k] if ex else None, recall_den=k)
    _statistically_equal(p, wp[:, 0])
    _statistically_equal(r, wr[:, 0])
    with pytest.raises(ValueError):
        sequence_precision_recall_score(model, inter, k=S)
