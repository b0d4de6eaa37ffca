"""Sharded evaluation of sequence models on the device: slb_shard_mask_targets against NumPy and its
rejected arguments, and the collective sequence_mrr_score, sequence_precision_recall_score and predict
of ShardedImplicitSequenceModel (PoolNet, CNNNet, LSTMNet, MixtureLSTMNet; Adagrad and lazy-exact Adam;
NCCL world 1, and 2 when two GPUs are visible) against the single-GPU scorers on gathered_net(), after
fit()."""

import copy
import ctypes

import numpy as np
import pytest
import torch

from conftest import assert_close
import sharded_common as sc

pytestmark = pytest.mark.gpu

FLOAT_MAX = np.finfo(np.float32).max


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _mask(block, col_offset, excluded, row_ptr, targets):
    """slb_shard_mask_targets on the device: (status, block afterwards, target scores)."""
    from spotlight_b200 import _lib, ops
    sc_ = torch.from_numpy(np.ascontiguousarray(block)).cuda()
    ex = None if excluded is None else torch.from_numpy(np.ascontiguousarray(excluded, np.int64)).cuda()
    rp = torch.from_numpy(np.asarray(row_ptr, np.int64)).cuda()
    tg = torch.from_numpy(np.asarray(targets, np.int64)).cuda()
    out = torch.full((len(targets),), -7.0, device='cuda')
    rc = _lib.load().slb_shard_mask_targets(_p(sc_), block.shape[0], block.shape[1], col_offset, _p(ex),
                                            0 if ex is None else ex.shape[1], _p(rp), _p(tg), _p(out), ops._stream())
    return rc, sc_.cpu().numpy(), out.cpu().numpy()


def _numpy_mask(block, col_offset, excluded, row_ptr, targets):
    block = block.copy()
    n_cols = block.shape[1]
    if excluded is not None:
        for r, ids in enumerate(excluded):
            c = ids - col_offset
            block[r, c[(c >= 0) & (c < n_cols)]] = -FLOAT_MAX
    out = np.zeros(len(targets), np.float32)
    for r in range(len(row_ptr) - 1):
        for p in range(row_ptr[r], row_ptr[r + 1]):
            c = targets[p] - col_offset
            if 0 <= c < n_cols:
                out[p] = block[r, c]
    return block, out


@pytest.mark.parametrize('exclude', [False, True], ids=['no-exclusion', 'exclusion'])
@pytest.mark.parametrize('n_items,lo,hi', [(1003, 0, 1003), (1003, 301, 702), (1024, 1000, 1024), (1003, 500, 500)])
def test_shard_mask_targets_against_numpy(n_items, lo, hi, exclude):
    """The full column range, sub-ranges and an empty one: excluded ids (padding 0 and repeats included)
    inside the range become -FLOAT_MAX, and every target reads its score after that overwrite when the
    range holds it, 0 otherwise; targets inside and outside the excluded set."""
    rs = np.random.RandomState(n_items + lo + 7 * exclude)
    R, L = 9, 40
    scores = rs.randn(R, n_items).astype(np.float32)
    excluded = rs.randint(0, n_items, (R, L))
    excluded[:, :5] = 0                                             # left padding
    excluded[:, 5] = excluded[:, 6]                                 # a repeated id
    counts = [0, 1, 3, 7, 300, 1, 2, 0, 20]
    row_ptr = np.concatenate([[0], np.cumsum(counts)])
    rows = np.repeat(np.arange(R), counts)
    targets = rs.randint(0, n_items, row_ptr[-1])
    from_excluded = rs.rand(len(targets)) < 0.3
    targets[from_excluded] = excluded[rows[from_excluded], rs.randint(0, L, from_excluded.sum())]
    block = np.ascontiguousarray(scores[:, lo:hi])
    ex = excluded if exclude else None
    rc, got_block, got = _mask(block, lo, ex, row_ptr, targets)
    assert rc == 0
    want_block, want = _numpy_mask(block, lo, ex, row_ptr, targets)
    assert np.array_equal(got_block, want_block)
    assert np.array_equal(got, want)
    inside = (targets >= lo) & (targets < hi)
    if hi > lo:
        assert inside.any() and (got[inside] != 0).all()
        if exclude:
            assert (got[inside & from_excluded] == -FLOAT_MAX).all() and (inside & from_excluded).any()
    assert (got[~inside] == 0).all()


def test_shard_mask_targets_rejections():
    """Negative sizes, ranges past INT32_MAX and null pointers are rejected before a launch; n_rows = 0
    does nothing; an empty column range writes zeros (a null block allowed)."""
    from spotlight_b200 import _lib, ops
    lib = _lib.load()
    block = torch.ones((2, 4), device='cuda')
    ex = torch.tensor([[0, 2], [3, 3]], dtype=torch.int64, device='cuda')
    rp = torch.tensor([0, 2, 3], dtype=torch.int64, device='cuda')
    tg = torch.tensor([1, 2, 3], dtype=torch.int64, device='cuda')
    out = torch.full((3,), -7.0, device='cuda')
    args = dict(scores=_p(block), rows=2, cols=4, off=0, ex=_p(ex), L=2, rp=_p(rp), tg=_p(tg), out=_p(out))

    def call(**kw):
        a = dict(args, **kw)
        return lib.slb_shard_mask_targets(a['scores'], a['rows'], a['cols'], a['off'], a['ex'], a['L'], a['rp'],
                                          a['tg'], a['out'], ops._stream())
    for bad in (dict(rows=-1), dict(cols=-1), dict(L=-1), dict(off=-1), dict(cols=1 << 31),
                dict(off=(1 << 31) - 3), dict(scores=None), dict(ex=None), dict(rp=None), dict(tg=None),
                dict(out=None)):
        assert call(**bad) == -1, bad
        assert lib.slb_last_error()
    assert call(rows=0, scores=None, ex=None, rp=None, tg=None, out=None) == 0
    torch.cuda.synchronize()
    assert (out == -7).all() and (block == 1).all()
    assert call(cols=0, scores=None) == 0
    assert (out == 0).all() and (block == 1).all()
    assert call(ex=None, L=0) == 0
    assert out.cpu().numpy().tolist() == [1, 1, 1] and (block == 1).all()
    assert call() == 0
    f = -float(FLOAT_MAX)
    assert out.cpu().numpy().tolist() == [1, f, f]
    assert block.cpu().numpy().tolist() == [[f, 1, f, 1], [1, 1, 1, f]]


# ------------------------------------------------------------------ the collective scorers after fit()

FIT = dict(seed=29, I=1500, D=32, S=20, n=700, B=128, n_iter=2, n_test=300, block=64)
NETS = ['pooling', 'cnn', 'lstm', 'mixture']
OPTS = ['adagrad', 'adam']
WORLDS = [1] + ([2] if torch.cuda.is_available() and torch.cuda.device_count() >= 2 else [])
PRED_IDS = np.random.RandomState(3).randint(0, 1500, 400)


def _data():
    rs = np.random.RandomState(FIT['seed'] + 3)
    seqs = rs.randint(1, FIT['I'], (FIT['n'] + FIT['n_test'], FIT['S'])).astype(np.int64)
    for b in range(len(seqs)):
        seqs[b, :rs.randint(0, FIT['S'])] = 0
    test = seqs[FIT['n']:]
    test[::7, -1] = test[::7, -4]                    # targets that are prefix items
    return seqs[:FIT['n']], test


def _net(kind):
    from spotlight_b200.sequence.representations import CNNNet, LSTMNet, MixtureLSTMNet, PoolNet
    torch.manual_seed(5)
    I, D = FIT['I'], FIT['D']
    return {'pooling': lambda: PoolNet(I, D),
            'cnn': lambda: CNNNet(I, D, kernel_width=[3, 2], dilation=[1, 2], num_layers=2),
            'lstm': lambda: LSTMNet(I, D),
            'mixture': lambda: MixtureLSTMNet(I, D, num_mixtures=2)}[kind]()


def _scores(model, test):
    from spotlight_b200.evaluation import sequence_mrr_score, sequence_precision_recall_score
    b = FIT['block']
    return {'mrr': sequence_mrr_score(model, test, sequence_block=b),
            'mrr_ex': sequence_mrr_score(model, test, exclude_preceding=True, sequence_block=b),
            'pr3_ex': sequence_precision_recall_score(model, test, k=3, exclude_preceding=True, sequence_block=b),
            'pr5': sequence_precision_recall_score(model, test, k=5, sequence_block=b)}


def _eval_jobs(rank, world, dev):
    from spotlight_b200 import optim
    from spotlight_b200.interactions import SequenceInteractions
    from spotlight_b200.sharded import ShardedImplicitSequenceModel
    train, test = _data()
    res = {}
    for kind in NETS:
        for opt in OPTS:
            model = ShardedImplicitSequenceModel(
                FIT['I'], rank, world, dev, loss='bpr', representation=_net(kind), embedding_dim=FIT['D'],
                n_iter=FIT['n_iter'], batch_size=FIT['B'], random_state=np.random.RandomState(FIT['seed']),
                optimizer_func=None if opt == 'adagrad' else optim.fused_adam(lr=1e-2))
            model.fit(SequenceInteractions(train, num_items=FIT['I']))
            got = _scores(model, SequenceInteractions(test, num_items=FIT['I']))
            got['predict all'] = model.predict(test[0])
            got['predict ids'] = model.predict(test[1, :-2], item_ids=PRED_IDS)
            res[kind, opt] = (got, copy.deepcopy(model.gathered_net()).cpu())
    return res


_RES = {}


def _results(world):
    if world not in _RES:
        _RES[world] = sc.run_world(_eval_jobs, world, backend='nccl', timeout=900)
    return _RES[world]


def _single(net):
    from spotlight_b200.sequence.implicit import ImplicitSequenceModel
    one = ImplicitSequenceModel(use_cuda=True, random_state=np.random.RandomState(0))
    one._net, one._num_items = net.cuda(), FIT['I']
    return one


def _near_tie_rows(one, test, k, exclude, rows):
    """The rows among ``rows`` with a target whose single-GPU score lies within 4 ulp of another item's."""
    from spotlight_b200 import evaluation as ev
    out = []
    for r in rows:
        inp = test[r:r + 1, :-k]
        row = ev._score_sequences(one, torch.from_numpy(inp).cuda())
        if exclude:
            ev._exclude(row, np.zeros(inp.shape[1], np.int64), inp[0])
        row = row[0].cpu().numpy()
        for t in test[r, -k:]:
            gap = np.abs(np.delete(row, t) - row[t])
            if (gap <= 4 * np.spacing(np.abs(row[t]))).any():
                out.append(r)
                break
    return out


@pytest.mark.parametrize('opt', OPTS)
@pytest.mark.parametrize('kind', NETS)
@pytest.mark.parametrize('world', WORLDS)
def test_sharded_sequence_scorers_equal_single_gpu_scorers(world, kind, opt):
    """Several blocks and a partial last one.  World 1: equal bit for bit.  World 2: the mixture head
    equal; the dot heads too, except at sequences with a target within a few ulp of another item's
    score (the per-range GEMM may round such a score differently from the full GEMM), which must be
    rare.  predict: within 1e-5 of the single-GPU predict's torch-op arithmetic."""
    from spotlight_b200.interactions import SequenceInteractions
    _, test = _data()
    assert FIT['n_test'] % FIT['block'] and FIT['n_test'] > 2 * FIT['block']
    for rank, res in _results(world).items():
        got, net = res[kind, opt]
        one = _single(net)
        want = _scores(one, SequenceInteractions(test, num_items=FIT['I']))
        for key, k, ex in (('mrr', 1, False), ('mrr_ex', 1, True), ('pr3_ex', 3, True), ('pr5', 5, False)):
            a, b = np.asarray(got[key]), np.asarray(want[key])
            if world == 1 or kind == 'mixture':
                assert np.array_equal(a, b), (rank, key)
            else:
                differ = np.nonzero((a != b).reshape(-1, len(test)).any(0))[0]
                assert len(differ) <= len(test) // 20, (rank, key, len(differ))
                near = _near_tie_rows(one, test, k, ex, differ)
                assert near == list(differ), (rank, key, sorted(set(differ) - set(near)))
        assert got['predict all'].dtype == np.float32 and got['predict all'].shape == (FIT['I'],)
        assert_close(got['predict all'], one.predict(test[0]), 1e-5, what='predict all')
        assert_close(got['predict ids'], one.predict(test[1, :-2], item_ids=PRED_IDS), 1e-5, what='predict ids')
