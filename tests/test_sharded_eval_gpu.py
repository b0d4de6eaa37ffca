"""Sharded evaluation on the device: slb_rank_counts against NumPy counts, column-range counts summed
and finalized against slb_rank_targets bit for bit, and the collective mrr_score,
precision_recall_score and predict of ShardedImplicitFactorizationModel (NCCL, world 1, and 2 when two
GPUs are visible) against the single-GPU scorers on gathered_net(), after fit()."""

import copy
import ctypes
import types

import numpy as np
import pytest
import torch

from conftest import assert_close
import sharded_common as sc

pytestmark = pytest.mark.gpu

FLOAT_MAX = np.finfo(np.float32).max


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _counts(block, col_offset, row_ptr, targets, target_scores):
    """slb_rank_counts on the device: (status, (3, n) int32 counts)."""
    from spotlight_b200 import _lib, ops
    n = len(targets)
    out = torch.full((3, n), -7, dtype=torch.int32, device='cuda')
    rp = torch.from_numpy(np.asarray(row_ptr, np.int64)).cuda()
    tg = torch.from_numpy(np.asarray(targets, np.int64)).cuda()
    ts = torch.from_numpy(np.asarray(target_scores, np.float32)).cuda()
    rc = _lib.load().slb_rank_counts(_p(block), block.shape[0], block.shape[1], col_offset, _p(rp), _p(tg), _p(ts), n,
                                     _p(out[0]), _p(out[1]), _p(out[2]), ops._stream())
    return rc, out.cpu().numpy()


def _numpy_counts(block, col_offset, row_ptr, targets, target_scores):
    gid = col_offset + np.arange(block.shape[1])
    out = np.zeros((3, len(targets)), np.int64)
    for r in range(len(row_ptr) - 1):
        row = block[r]
        for p in range(row_ptr[r], row_ptr[r + 1]):
            s = np.float32(target_scores[p])
            out[:, p] = [(row > s).sum(), (row == s).sum(), ((row == s) & (gid < targets[p])).sum()]
    return out


def _block(rs, R, n_items, ties):
    scores = rs.randn(R, n_items).astype(np.float32)
    if ties:
        scores = np.round(scores * 2) / 2                           # a handful of distinct values
    else:
        scores[:, 1::3] = np.round(scores[:, 1::3], 1)
    scores[2, rs.randint(0, n_items, n_items // 3)] = -FLOAT_MAX    # excluded items
    counts = [0, 1, 2100, 3, 1, 0, 1030, 2, 40]                     # 0, 1, one and several chunks
    row_ptr = np.concatenate([[0], np.cumsum(counts)])
    targets = rs.randint(0, n_items, row_ptr[-1])
    return scores, row_ptr[:R + 1], targets


@pytest.mark.parametrize('ties', [False, True], ids=['random', 'ties'])
@pytest.mark.parametrize('n_items,lo,hi', [(1003, 0, 1003), (1003, 301, 702), (1024, 1000, 1024), (6, 2, 3)])
def test_rank_counts_against_numpy(n_items, lo, hi, ties):
    """Counts over the columns [lo, hi) of the full rows, with the targets' full-row scores supplied:
    targets inside and outside the range, NaN and excluded targets."""
    rs = np.random.RandomState(n_items + lo)
    scores, row_ptr, targets = _block(rs, 9, n_items, ties)
    ts = scores[np.repeat(np.arange(9), np.diff(row_ptr)), targets]
    ts[::17] = np.nan
    block = np.ascontiguousarray(scores[:, lo:hi])
    rc, got = _counts(torch.from_numpy(block).cuda(), lo, row_ptr, targets, ts)
    assert rc == 0
    want = _numpy_counts(block, lo, row_ptr, targets, ts)
    assert np.array_equal(got, want)
    assert got[1].sum() > 0 and got[0].sum() > 0


@pytest.mark.parametrize('n_items', [1003, 1024, 6])
@pytest.mark.parametrize('parts', [1, 2, 3, 4])
def test_range_counts_sum_to_rank_targets(n_items, parts):
    """Splitting the block into column ranges, summing the ranges' counts and finalizing them gives
    slb_rank_targets' average rank (float32 bits) and stable position exactly."""
    from spotlight_b200 import _lib, ops
    from spotlight_b200.sharded import _finalize_ranks
    rs = np.random.RandomState(parts * 7 + n_items)
    for ties in (False, True):
        scores, row_ptr, targets = _block(rs, 9, n_items, ties)
        if n_items > 8:
            scores[:, 7] = scores[:, n_items - 2]                    # equal items far apart
        full = torch.from_numpy(scores).cuda()
        n = len(targets)
        avg = torch.empty(n, device='cuda')
        pos = torch.empty(n, dtype=torch.int64, device='cuda')
        rp = torch.from_numpy(row_ptr.astype(np.int64)).cuda()
        tg = torch.from_numpy(targets.astype(np.int64)).cuda()
        _lib.check(_lib.load().slb_rank_targets(_p(full), 9, n_items, _p(rp), _p(tg), n, _p(avg), _p(pos),
                                                ops._stream()))
        ts = scores[np.repeat(np.arange(9), np.diff(row_ptr)), targets]
        cuts = np.linspace(0, n_items, parts + 1).astype(int)
        total = np.zeros((3, n), np.int64)
        for lo, hi in zip(cuts[:-1], cuts[1:]):
            rc, c = _counts(torch.from_numpy(np.ascontiguousarray(scores[:, lo:hi])).cuda(), lo, row_ptr, targets, ts)
            assert rc == 0
            total += c
        got_avg, got_pos = _finalize_ranks(total)
        assert np.array_equal(got_avg.astype(np.float32).view(np.int32), avg.cpu().numpy().view(np.int32)), ties
        assert np.array_equal(got_pos, pos.cpu().numpy()), ties


def test_rank_counts_rejections():
    """n_cols past INT32_MAX, a range ending past INT32_MAX and null pointers are rejected before a
    launch; an empty column range writes zeros."""
    from spotlight_b200 import _lib, ops
    lib = _lib.load()
    block = torch.zeros((1, 4), device='cuda')
    rp = torch.tensor([0, 2], dtype=torch.int64, device='cuda')
    tg = torch.tensor([1, 3], dtype=torch.int64, device='cuda')
    ts = torch.zeros(2, device='cuda')
    out = torch.full((3, 2), -7, dtype=torch.int32, device='cuda')
    o = [_p(out[k]) for k in range(3)]
    args = dict(scores=_p(block), cols=4, off=0, rp=_p(rp), tg=_p(tg), ts=_p(ts), o=o)

    def call(**kw):
        a = dict(args, **kw)
        return lib.slb_rank_counts(a['scores'], 1, a['cols'], a['off'], a['rp'], a['tg'], a['ts'], 2, *a['o'],
                                   ops._stream())
    assert call(cols=(1 << 31)) == -1
    assert call(off=(1 << 31) - 2) == -1
    for k in ('scores', 'rp', 'tg', 'ts'):
        assert call(**{k: None}) == -1, k
    assert call(o=[o[0], None, o[2]]) == -1
    assert (out == -7).all()
    assert call(cols=0, scores=None) == 0
    assert (out == 0).all()
    assert call() == 0
    assert out.cpu().numpy().tolist() == [[0, 0], [4, 4], [1, 3]]


# ------------------------------------------------------------------ the collective scorers after fit()

FIT = dict(U=300, I=1000, D=16, H=3, B=256, n=4000, n_iter=2, seed=11)
KINDS = [('plain', 'adagrad'), ('plain', 'adam'), ('bloom', 'adagrad'), ('bloom', 'adam')]
KS = [1, 5, 10, 50]
WORLDS = [1] + ([2] if torch.cuda.is_available() and torch.cuda.device_count() >= 2 else [])


def _data():
    rs = np.random.RandomState(4)
    train = (rs.randint(0, FIT['U'], FIT['n']), rs.randint(1, FIT['I'], FIT['n']))
    test = (rs.randint(0, FIT['U'], 900), rs.randint(0, FIT['I'], 900))
    return train, test


def _inter(pair):
    from spotlight_b200.interactions import Interactions
    return Interactions(pair[0].astype(np.int32), pair[1].astype(np.int32), num_users=FIT['U'], num_items=FIT['I'])


def _model(rank, world, dev, kind, opt):
    from spotlight_b200 import optim
    from spotlight_b200.factorization.representations import BilinearNet
    from spotlight_b200.layers import BloomEmbedding
    from spotlight_b200.sharded import ShardedImplicitFactorizationModel
    kw = dict(loss='bpr', embedding_dim=FIT['D'], n_iter=FIT['n_iter'], batch_size=FIT['B'],
              random_state=np.random.RandomState(FIT['seed']),
              optimizer_func=optim.fused_adagrad(lr=0.05) if opt == 'adagrad' else optim.fused_adam(lr=1e-2))
    if kind == 'bloom':
        torch.manual_seed(3)
        kw['representation'] = BilinearNet(FIT['U'], FIT['I'], FIT['D'], item_embedding_layer=BloomEmbedding(
            FIT['I'], FIT['D'], compression_ratio=0.2, num_hash_functions=FIT['H']))
    return ShardedImplicitFactorizationModel(FIT['U'], FIT['I'], rank, world, dev, **kw)


def _integer_tables(model):
    """Overwrites this rank's shards with small integers (functions of the global row), so that every
    score is exact in float32 and ties are common."""
    st = model.state
    D = st.Wu.shape[1]
    dev = st.Wu.device
    ints = lambda rows, salt, width: ((rows.reshape(-1, 1) * 7 + torch.arange(width, device=dev) * 3 + salt)  # noqa: E731
                                      % 5 - 2).float().reshape(len(rows), width)
    with torch.no_grad():
        st.Wu.copy_(ints(torch.arange(st.ulo, st.uhi, device=dev), 1, D))
        st.bu.copy_(ints(torch.arange(st.ulo, st.uhi, device=dev), 2, 1).reshape(-1))
        if model._net is None:
            n = st.ihi - st.ilo
            st.Wi[:n] = ints(torch.arange(st.ilo, st.ihi, device=dev) % 97, 3, D)     # equal rows across shards
            st.bi[:n] = ints(torch.arange(st.ilo, st.ihi, device=dev) % 97, 4, 1).reshape(-1)
        else:
            n = st.mhi - st.mlo
            st.Wi[:n] = ints(torch.arange(st.mlo, st.mhi, device=dev), 3, D) % 2
            if st.mlo == 0:
                st.Wi[0] = 0
            st.bi.copy_(ints(torch.arange(st.num_ids, device=dev), 4, 1).reshape(-1))


def _scores(model, test, train):
    from spotlight_b200.evaluation import mrr_score, precision_recall_score
    out = {'mrr': mrr_score(model, test, train, user_block=100)}
    out['pr'] = precision_recall_score(model, test, train, k=KS, user_block=64)
    out['pr5'] = precision_recall_score(model, test, None, k=5)
    return out


def _eval_jobs(rank, world, dev):
    train, test = _data()
    pu, pi = np.random.RandomState(9).randint(0, FIT['U'], 500), np.random.RandomState(10).randint(0, FIT['I'], 500)
    res = {}
    for kind, opt in KINDS:
        model = _model(rank, world, dev, kind, opt)
        model.fit(_inter(train))
        # a copy: a Bloom model's gathered_net() is its own net, which the integer tables overwrite below
        r = {'float': (_scores(model, _inter(test), _inter(train)), copy.deepcopy(model.gathered_net()).cpu(),
                       model.predict(pu, pi), model.predict(17))}
        _integer_tables(model)
        r['int'] = (_scores(model, _inter(test), _inter(train)), model.gathered_net().cpu(),
                    model.predict(pu, pi), model.predict(17))
        res[kind, opt] = r
    return res


_RES = {}


def _results(world):
    if world not in _RES:
        _RES[world] = sc.run_world(_eval_jobs, world, backend='nccl', timeout=900)
    return _RES[world]


def _single(net):
    net = net.cuda()
    return types.SimpleNamespace(_net=net, _optimizer=None, _num_items=FIT['I'], _num_users=FIT['U'])


def _near_tie_users(model, test, train, users_differing):
    """The users among ``users_differing`` with a test target whose score lies within 4 ulp of another
    item's score in the single-GPU block."""
    from spotlight_b200 import evaluation as ev
    tcsr, trcsr = test.tocsr(), train.tocsr()
    out = []
    for u in users_differing:
        row = ev._score_block(model, torch.tensor([u], device='cuda'))
        ev._exclude(row, np.zeros(len(trcsr[u].indices), np.int64), trcsr[u].indices)
        row = row[0].cpu().numpy()
        for t in tcsr[u].indices:
            gap = np.abs(np.delete(row, t) - row[t])
            if (gap <= 4 * np.spacing(np.abs(row[t]))).any():
                out.append(u)
                break
    return out


@pytest.mark.parametrize('kind,opt', KINDS, ids=['%s-%s' % k for k in KINDS])
@pytest.mark.parametrize('world', WORLDS)
def test_sharded_scorers_equal_single_gpu_scorers(world, kind, opt):
    """On integer tables every result equals the single-GPU scorers' on gathered_net() exactly; on the
    trained float tables too, except at users with a target within a few ulp of another item's score
    (the per-range GEMM may round such a score differently from the full GEMM)."""
    train, test = _data()
    test_i, train_i = _inter(test), _inter(train)
    users = np.nonzero(np.diff(test_i.tocsr().indptr))[0]
    pu, pi = np.random.RandomState(9).randint(0, FIT['U'], 500), np.random.RandomState(10).randint(0, FIT['I'], 500)
    for rank, res in _results(world).items():
        for tables in ('int', 'float'):
            got, net, pred, pred_all = res[kind, opt][tables]
            one = _single(net)
            want = _scores(one, test_i, train_i)
            exact = tables == 'int' or world == 1
            if exact:
                assert np.array_equal(got['mrr'], want['mrr']), (rank, tables)
                for key in ('pr', 'pr5'):
                    for a, b in zip(got[key], want[key]):
                        assert np.array_equal(a, b), (rank, tables, key)
            else:
                differ = np.nonzero(got['mrr'] != want['mrr'])[0]
                for key in ('pr', 'pr5'):
                    for a, b in zip(got[key], want[key]):
                        a, b = a.reshape(len(users), -1), b.reshape(len(users), -1)
                        differ = np.union1d(differ, np.nonzero((a != b).any(1))[0])
                assert len(differ) <= len(users) // 20, (rank, len(differ))
                near = _near_tie_users(one, test_i, train_i, users[differ])
                assert len(near) == len(differ), (rank, sorted(set(users[differ]) - set(near)))
            with torch.no_grad():
                fwd = net.cuda()(torch.from_numpy(pu).cuda(), torch.from_numpy(pi).cuda()).cpu().numpy()
                fwd_all = net(torch.tensor([17], device='cuda'), torch.arange(FIT['I'], device='cuda')).cpu().numpy()
            if tables == 'int':
                assert np.array_equal(pred, fwd) and np.array_equal(pred_all, fwd_all), rank
            else:
                assert_close(pred, fwd, 1e-5, what='predict pairs')
                assert_close(pred_all, fwd_all, 1e-5, what='predict one user')
