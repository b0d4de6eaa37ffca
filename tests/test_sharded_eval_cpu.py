"""Sharded evaluation of factorization models on the CPU (gloo, worlds 1, 2 and 3, NumPy backend):
mrr_score, precision_recall_score and predict of a ShardedImplicitFactorizationModel against
oracle/evaluation.py on the gathered tables.

The tables hold small integers, so every score is exact in float32 whatever the summation order, and
ties are common: items share score values, and equal item rows sit on different shards.  The results
must then be equal, not close."""

import numpy as np
import pytest
import torch

from oracle import evaluation as oev
from oracle.murmur import bloom_rows
from sharded_common import NumpyBackend, run_world

U, I, D = 11, 13, 4                 # world 3: users [0,4) [4,8) [8,11), items [0,5) [5,10) [10,13)
M, H = 6, 2                         # Bloom: 13 ids hashed to 6 rows, 2 hashes
KS = [1, 2, 5, 20]


class EvalNumpyBackend(NumpyBackend):
    """NumPy stand-ins for GpuBackend's evaluation pieces (float64 arithmetic, float32 results)."""

    def bloom_item_rows(self, W_full, ids, seeds):
        rows = bloom_rows(ids.numpy(), len(seeds), W_full.shape[0], 0)
        return torch.from_numpy(W_full.numpy().astype(np.float64)[rows].sum(1).astype(np.float32))

    def shard_scores(self, users, user_bias, items, item_bias):
        s = (users.numpy().astype(np.float64) @ items.numpy().astype(np.float64).T
             + user_bias.numpy().reshape(-1, 1) + item_bias.numpy().reshape(1, -1))
        return torch.from_numpy(s.astype(np.float32))

    def pair_scores(self, users, user_bias, items, item_bias, u_idx, i_idx):
        u, i = u_idx.numpy(), i_idx.numpy()
        s = ((users.numpy().astype(np.float64)[u] * items.numpy().astype(np.float64)[i]).sum(1)
             + user_bias.numpy()[u] + item_bias.numpy()[i])
        return torch.from_numpy(s.astype(np.float32))

    def rank_counts(self, scores, col_offset, row_ptr, targets, target_scores):
        sc, ts = scores.numpy(), target_scores.numpy()
        gid = col_offset + np.arange(sc.shape[1])
        out = np.zeros((3, len(targets)), dtype=np.int32)
        for r in range(len(row_ptr) - 1):
            for p in range(row_ptr[r], row_ptr[r + 1]):
                row, s = sc[r], ts[p]
                out[:, p] = [(row > s).sum(), (row == s).sum(), ((row == s) & (gid < targets[p])).sum()]
        return torch.from_numpy(out)


def _tables(bloom):
    rs = np.random.RandomState(5)
    Wu = rs.randint(-2, 3, (U, D)).astype(np.float32)
    bu = rs.randint(-1, 2, (U, 1)).astype(np.float32)
    if bloom:
        Wi = rs.randint(-1, 2, (M, D)).astype(np.float32)
        Wi[0] = 0                                   # the hashed table's padding row
    else:
        Wi = rs.randint(-2, 3, (I, D)).astype(np.float32)
        Wi[12], Wi[7] = Wi[1], Wi[3]                # equal rows on different shards
    bi = rs.randint(-1, 2, (I, 1)).astype(np.float32)
    if not bloom:
        bi[12], bi[7] = bi[1], bi[3]
    return Wu, Wi, bu, bi


def _sets():
    """(test, narrow test, train) Interactions, with at most 7 test items per user."""
    from spotlight_b200.interactions import Interactions
    rs = np.random.RandomState(6)
    tu, ti = rs.randint(0, U, 30), rs.randint(0, I, 30)
    tu = np.concatenate([tu, [0, 0, 0, 0]])
    ti = np.concatenate([ti, [1, 6, 12, 7]])        # user 0: test items on every shard
    keep = np.ones(len(tu), bool)
    for u in range(U):                              # at most 7 distinct items per user
        idx = np.nonzero(tu == u)[0]
        _, first = np.unique(ti[idx], return_index=True)
        drop = np.setdiff1d(np.arange(len(idx)), np.sort(first)[:7])
        keep[idx[drop]] = False
    tu, ti = tu[keep], ti[keep]
    ru, ri = rs.randint(0, U, 40), rs.randint(0, I, 40)
    ru, ri = np.concatenate([ru, tu[:6]]), np.concatenate([ri, ti[:6]])    # targets that are train items
    nu, ni = rs.randint(0, U, 12), rs.randint(0, 5, 12)                    # only rank 0 of world 3 owns targets
    mk = lambda u, i: Interactions(u.astype(np.int32), i.astype(np.int32), num_users=U, num_items=I)  # noqa: E731
    return mk(tu, ti), mk(nu, ni), mk(ru, ri)


def _model(rank, world, dev, bloom):
    from spotlight_b200.factorization.representations import BilinearNet
    from spotlight_b200.layers import BloomEmbedding
    from spotlight_b200.sharded import ShardedImplicitFactorizationModel
    Wu, Wi, bu, bi = _tables(bloom)
    kw = dict(backend=EvalNumpyBackend(), embedding_dim=D, random_state=np.random.RandomState(0))
    if bloom:
        net = BilinearNet(U, I, D, item_embedding_layer=BloomEmbedding(I, D, M / float(I) + 1e-9, H))
        assert net.item_embeddings.compressed_num_embeddings == M
        with torch.no_grad():
            net.user_embeddings.weight.copy_(torch.from_numpy(Wu))
            net.user_biases.weight.copy_(torch.from_numpy(bu))
            net.item_embeddings.embeddings.weight.copy_(torch.from_numpy(Wi))
            net.item_biases.weight.copy_(torch.from_numpy(bi))
        return ShardedImplicitFactorizationModel(U, I, rank, world, dev, loss='hinge', representation=net, **kw)
    return ShardedImplicitFactorizationModel(U, I, rank, world, dev,
                                             init=[torch.from_numpy(x) for x in (Wu, Wi, bu, bi)], **kw)


def _eval_job(rank, world, dev, bloom):
    from spotlight_b200.evaluation import mrr_score, precision_recall_score
    from spotlight_b200.interactions import Interactions
    model = _model(rank, world, dev, bloom)
    test, narrow, train = _sets()
    out = {}
    for name, te in (('test', test), ('narrow', narrow)):
        for tag, tr in (('notrain', None), ('train', train)):
            out['mrr', name, tag] = mrr_score(model, te, tr, user_block=3)
            out['pr', name, tag, 'scalar'] = precision_recall_score(model, te, tr, k=5, user_block=4)
            out['pr', name, tag, 'array'] = precision_recall_score(model, te, tr, k=KS, user_block=4)
    pu, pi = np.random.RandomState(7).randint(0, U, 25), np.random.RandomState(8).randint(0, I, 25)
    out['predict pairs'] = (pu, pi, model.predict(pu, pi))
    out['predict all'] = model.predict(9)
    # an out-of-range item id raises on every rank before any collective
    bad = Interactions(np.array([1, 2], np.int32), np.array([3, I], np.int32), num_users=U, num_items=I + 1)
    raised = []
    for call in (lambda: mrr_score(model, bad), lambda: precision_recall_score(model, test, bad),
                 lambda: model.predict(np.array([1, 2]), np.array([0, I]))):
        try:
            call()
        except ValueError:
            raised.append(True)
    out['raised'] = raised
    net = model.gathered_net()
    out['tables'] = [t.detach().numpy() for t in (net.user_embeddings.weight, net.user_biases.weight,
                                                  net.item_biases.weight)]
    out['tables'].append((net.item_embeddings.embeddings.weight if bloom else net.item_embeddings.weight)
                         .detach().numpy())
    return out


def _mrr_from_oracle_ranks(rows, targets, excluded):
    """Per row, the mean of 1 / oracle average rank over its targets, summed as the scorer sums them
    (np.add.reduceat; oracle.evaluation.mrr's np.mean adds in another order, a last-bit difference)."""
    ranks, starts = [], []
    for r, row in enumerate(rows):
        if excluded is not None:
            row = oev.exclude(row, excluded[r])
        starts.append(len(ranks))
        ranks += [oev.average_rank(row, t) for t in targets[r]]
    return np.add.reduceat(1.0 / np.array(ranks), starts) / np.array([len(t) for t in targets])


def _oracle_rows(tables, bloom):
    Wu, bu, bi, Wi = [t.astype(np.float64) for t in tables]
    items = Wi[bloom_rows(np.arange(I), H, M, 0)].sum(1) if bloom else Wi
    return Wu @ items.T + bu.reshape(-1, 1) + bi.reshape(1, -1), Wu, bu, bi, items


@pytest.mark.parametrize('bloom', [False, True], ids=['plain', 'bloom'])
@pytest.mark.parametrize('world', [1, 2, 3])
def test_sharded_scorers_equal_the_oracle(world, bloom):
    res = run_world(_eval_job, world, (bloom,), timeout=240)
    test, narrow, train = _sets()
    for rank in range(world):
        out = res[rank]
        assert out['raised'] == [True, True, True], rank
        rows, Wu, bu, bi, items = _oracle_rows(out['tables'], bloom)
        assert np.array_equal(rows, rows.astype(np.float32))           # integer scores, exact in float32
        rows = rows.astype(np.float32)
        for name, te in (('test', test), ('narrow', narrow)):
            tcsr = te.tocsr()
            users = np.nonzero(np.diff(tcsr.indptr))[0]
            targets = [tcsr[u].indices for u in users]
            for tag, tr in (('notrain', None), ('train', train)):
                excluded = None if tr is None else [tr.tocsr()[u].indices for u in users]
                got = out['mrr', name, tag]
                assert np.array_equal(got, _mrr_from_oracle_ranks(rows[users], targets, excluded)), (rank, name, tag)
                np.testing.assert_allclose(got, oev.mrr(rows[users], targets, excluded), rtol=1e-15, atol=0)
                wp, wr = oev.precision_recall(rows[users], targets, KS, excluded)
                p, r = out['pr', name, tag, 'array']
                assert np.array_equal(p, wp) and np.array_equal(r, wr), (rank, name, tag)
                wp, wr = oev.precision_recall(rows[users], targets, 5, excluded)
                p, r = out['pr', name, tag, 'scalar']
                assert p.shape == (len(users),)
                assert np.array_equal(p, wp[:, 0]) and np.array_equal(r, wr[:, 0]), (rank, name, tag)
        pu, pi, got = out['predict pairs']
        want = (Wu[pu] * items[pi]).sum(1) + bu[pu, 0] + bi[pi, 0]
        assert got.dtype == np.float32 and np.array_equal(got, want.astype(np.float32)), rank
        assert np.array_equal(out['predict all'], rows[9]), rank
    for rank in range(1, world):                    # every rank has the whole result
        for key in res[0]:
            if key[0] in ('mrr', 'pr'):
                assert np.array_equal(np.asarray(res[rank][key]), np.asarray(res[0][key])), key


def test_fixture_has_the_cases_it_claims():
    """Ties across shards, a user whose targets span every shard of world 3, targets that are train
    items and a test set whose targets only rank 0 of world 3 owns."""
    from spotlight_b200.sharded import ShardPlan
    test, narrow, train = _sets()
    plan = ShardPlan(U, I, 3)
    owner = lambda items: np.asarray(items) // plan.ichunk          # noqa: E731
    assert set(owner(test.tocsr()[0].indices)) == {0, 1, 2}
    assert set(owner(narrow.item_ids)) == {0}
    pairs = set(zip(test.user_ids.tolist(), test.item_ids.tolist()))
    assert pairs & set(zip(train.user_ids.tolist(), train.item_ids.tolist()))
    for bloom in (False, True):
        Wu, Wi, bu, bi = _tables(bloom)
        rows = _oracle_rows([Wu, bu, bi, Wi], bloom)[0]
        tied = [(r[a] == r[b]) for r in rows for a in range(5) for b in range(10, 13)]
        assert np.sum(tied) >= 10, bloom             # equal scores of rank 0's and rank 2's items
