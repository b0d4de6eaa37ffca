"""Device data preparation (csrc/prepare.cu) against the host code, integer-exact: to_sequence of
CUDA Interactions, both train/test splits, and fit() / the scorers on the device outputs."""

import numpy as np
import pytest
import torch

from conftest import load_golden
from spotlight_b200.cross_validation import (random_train_test_split, shuffle_interactions,
                                             user_based_train_test_split)
from spotlight_b200.interactions import Interactions, SequenceInteractions

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda:0')
COLUMNS = ('user_ids', 'item_ids', 'ratings', 'timestamps', 'weights')


def _dev(inter):
    kw = {k: None if getattr(inter, k) is None else torch.from_numpy(np.ascontiguousarray(getattr(inter, k))).to(DEV)
          for k in COLUMNS}
    return Interactions(kw.pop('user_ids'), kw.pop('item_ids'), num_users=inter.num_users,
                        num_items=inter.num_items, **kw)


def _same_seq(host, dev, what=''):
    assert torch.is_tensor(dev.sequences) and dev.sequences.is_cuda and dev.sequences.dtype == torch.int32
    assert dev.user_ids.dtype == torch.int32, what
    assert dev.sequences.shape == host.sequences.shape, (what, dev.sequences.shape, host.sequences.shape)
    assert np.array_equal(dev.sequences.cpu().numpy(), host.sequences), what
    assert np.array_equal(dev.user_ids.cpu().numpy(), host.user_ids), what
    assert dev.num_items == host.num_items


def _check(users, items, ts, cases, num_items=None):
    inter = Interactions(users, items, timestamps=ts, num_users=int(users.max()) + 1 if users.max() >= 0 else 1,
                         num_items=num_items or int(items.max()) + 1)
    d = _dev(inter)
    for L, step, m in cases:
        kw = dict(max_sequence_length=L, min_sequence_length=m, step_size=step)
        _same_seq(inter.to_sequence(**kw), d.to_sequence(**kw), (L, step, m, ts.dtype, users.dtype, items.dtype))


def _timestamps(rs, n, dtype):
    if np.dtype(dtype).kind == 'f':
        return rs.choice(np.array([-2.5, -0.0, 0.0, np.nan, 1.0, 3.0, np.inf, -np.inf], dtype=dtype), n)
    return rs.randint(-50, 50, n).astype(dtype) * (2 ** 40 if dtype == np.int64 else 1)


GRID = [(L, step, m) for L in (1, 2, 7, 200) for step in (None, 1, 3, L + 5) for m in (None, 0, 1, L)]


@pytest.mark.parametrize('ts_dtype', [np.int32, np.int64, np.float32, np.float64])
@pytest.mark.parametrize('id_dtype', [np.int32, np.int64])
def test_to_sequence_matches_host(ts_dtype, id_dtype):
    rs = np.random.RandomState(5)
    n = 5000
    users = (rs.randint(-10, 300, n) * 3).astype(id_dtype)          # gaps and negative ids
    users[:700] = 33                                                 # a long history
    items = rs.randint(1, 400, n).astype(np.int64 if id_dtype == np.int32 else np.int32)   # the other width
    _check(users, items, _timestamps(rs, n, ts_dtype), GRID)


def test_to_sequence_edge_fixture():
    g = load_golden('to_sequence_edges')
    for name in ('ties_i32', 'neg_i64', 'float64', 'float32'):
        _check(g['users'], g['items'], g['ts.' + name], [(5, None, m) for m in (None, 0, 1, 5)] +
               [(5, 1, 1), (5, 8, 5), (7, 3, 0)], num_items=90)


def test_to_sequence_sizes_and_key_spans():
    rs = np.random.RandomState(9)
    for n in (1, 2, 2047, 2048, 2049, 4097, 70001):
        users = rs.randint(0, max(1, n // 20), n).astype(np.int32)
        _check(users, rs.randint(1, 50, n).astype(np.int32), rs.randint(0, 100, n).astype(np.int64),
               [(7, None, None), (7, 2, 3)])
    # every radix pass: the full int64 timestamp span and the full int64 user span
    n = 30000
    ts = rs.randint(np.iinfo(np.int64).min, np.iinfo(np.int64).max, n, dtype=np.int64)
    ts[:3] = [np.iinfo(np.int64).min, np.iinfo(np.int64).max, 0]
    users = rs.randint(0, 500, n).astype(np.int64)
    users[:2] = [-2 ** 62, 2 ** 40]
    _check(users, rs.randint(1, 50, n).astype(np.int32), ts, [(10, None, None), (10, 1, 10)],
           num_items=50)


def test_to_sequence_hot_user_and_large():
    rs = np.random.RandomState(2)
    n = 10 ** 6 + 50000
    users = rs.randint(0, 1000, n).astype(np.int32)
    users[:10 ** 6] = 17                                              # one user with 1e6 interactions
    _check(users, rs.randint(1, 5000, n).astype(np.int32), rs.randint(0, 10 ** 5, n).astype(np.int32),
           [(200, None, None), (50, 1, 50)])
    n = 3 * 10 ** 7
    users = rs.randint(0, 10 ** 6, n).astype(np.int32)
    items = rs.randint(1, 10 ** 5, n).astype(np.int32)
    ts = rs.randint(0, 10 ** 9, n).astype(np.int64)
    _check(users, items, ts, [(50, None, None)])


def test_to_sequence_is_deterministic_and_checks_input():
    rs = np.random.RandomState(4)
    n = 200000
    d = _dev(Interactions(rs.randint(0, 3000, n).astype(np.int32), rs.randint(1, 500, n).astype(np.int32),
                          timestamps=rs.randint(0, 20, n).astype(np.int32)))
    a, b = d.to_sequence(20, step_size=3), d.to_sequence(20, step_size=3)
    assert torch.equal(a.sequences, b.sequences) and torch.equal(a.user_ids, b.user_ids)
    with pytest.raises(IndexError):
        d.to_sequence(5, min_sequence_length=6)
    with pytest.raises(ValueError):
        d.to_sequence(5, step_size=0)
    bad = Interactions(torch.arange(4, device=DEV), torch.arange(4, device=DEV), timestamps=torch.arange(4, device=DEV))
    with pytest.raises(ValueError):
        bad.to_sequence()                                             # item id 0
    with pytest.raises(ValueError):
        Interactions(torch.arange(4, device=DEV), torch.arange(4, device=DEV) + 1).to_sequence()
    mixed = Interactions(torch.arange(4, device=DEV), torch.arange(4, device=DEV) + 1, timestamps=np.arange(4))
    with pytest.raises(ValueError):
        mixed.to_sequence()


def _same_inter(host, dev, what):
    for k in COLUMNS:
        h, d = getattr(host, k), getattr(dev, k)
        if h is None:
            assert d is None, (what, k)
            continue
        assert d.is_cuda and str(d.dtype).replace('torch.', '') == str(h.dtype), (what, k, d.dtype, h.dtype)
        assert d.cpu().numpy().tobytes() == h.tobytes(), (what, k)
    assert (host.num_users, host.num_items) == (dev.num_users, dev.num_items)


def _same_state(a, b):
    sa, sb = a.get_state(), b.get_state()
    assert (sa[1] == sb[1]).all() and sa[2] == sb[2]


@pytest.mark.parametrize('n', [5000, (1 << 17) + 3000])
@pytest.mark.parametrize('present', [(), ('ratings',), ('timestamps',), ('weights',),
                                     ('ratings', 'timestamps', 'weights')])
def test_splits_match_host(n, present):
    rs = np.random.RandomState(n)
    cols = dict(ratings=rs.randint(1, 6, n).astype(np.float64), timestamps=rs.randint(0, 10 ** 9, n),
                weights=rs.rand(n).astype(np.float32))
    host = Interactions(rs.randint(0, 5000, n).astype(np.int32), rs.randint(0, 800, n).astype(np.int64),
                        num_users=5000, num_items=800, **{k: cols[k] for k in present})
    dev = _dev(host)
    a, b = np.random.RandomState(1), np.random.RandomState(1)
    _same_inter(shuffle_interactions(host, random_state=a), shuffle_interactions(dev, random_state=b), 'shuffle')
    _same_state(a, b)
    for p in (0.2, 0.35):
        for split in (random_train_test_split, user_based_train_test_split):
            ht, hs = split(host, test_percentage=p, random_state=a)
            dt, ds = split(dev, test_percentage=p, random_state=b)
            _same_inter(ht, dt, split.__name__ + ' train')
            _same_inter(hs, ds, split.__name__ + ' test')
            _same_state(a, b)


def test_user_split_needs_int32_ids_on_device():
    d = Interactions(torch.arange(10, device=DEV), torch.arange(10, device=DEV))
    with pytest.raises(TypeError):
        user_based_train_test_split(d, random_state=np.random.RandomState(0))


def _epoch_losses(capsys, model, data):
    capsys.readouterr()
    model.fit(data, verbose=True)
    return [line for line in capsys.readouterr().out.splitlines() if line.startswith('Epoch')]


def _same_fit(capsys, make, host, dev):
    # each constructor reseeds torch and fit() draws the initial weights: build, then fit, in turn
    m1 = make()
    l1 = _epoch_losses(capsys, m1, host)
    m2 = make()
    l2 = _epoch_losses(capsys, m2, dev)
    assert l1 == l2 and len(l1) > 0
    s1, s2 = m1._net.state_dict(), m2._net.state_dict()
    assert all(torch.equal(s1[k], s2[k]) for k in s1)
    _same_state(m1._random_state, m2._random_state)
    return m1, m2


def _sequence_data(seed=0, n=20000):
    rs = np.random.RandomState(seed)
    return Interactions(rs.randint(0, 800, n).astype(np.int32), rs.randint(1, 300, n).astype(np.int32),
                        timestamps=rs.randint(0, 10 ** 6, n).astype(np.int64))


@pytest.mark.parametrize('rep', ['pooling', 'lstm'])
def test_sequence_fit_on_device_data(capsys, rep):
    from spotlight_b200.sequence.implicit import ImplicitSequenceModel
    inter = _sequence_data()
    host, dev = inter.to_sequence(20), _dev(inter).to_sequence(20)
    _same_fit(capsys, lambda: ImplicitSequenceModel(loss='bpr', representation=rep, embedding_dim=16, n_iter=2,
                                                    batch_size=64, use_cuda=True,
                                                    random_state=np.random.RandomState(3)), host, dev)


def test_factorization_fit_and_scorers_on_device_data(capsys):
    from spotlight_b200 import evaluation, optim
    from spotlight_b200.factorization.explicit import ExplicitFactorizationModel
    from spotlight_b200.factorization.implicit import ImplicitFactorizationModel
    rs = np.random.RandomState(8)
    n = 30000
    host = Interactions(rs.randint(0, 1000, n).astype(np.int32), rs.randint(0, 700, n).astype(np.int32),
                        ratings=rs.randint(1, 6, n).astype(np.float32), num_users=1000, num_items=700)
    dev = _dev(host)
    m1, m2 = _same_fit(capsys, lambda: ImplicitFactorizationModel(
        loss='bpr', embedding_dim=16, n_iter=2, batch_size=256, use_cuda=True,
        optimizer_func=optim.fused_adagrad(lr=0.05), random_state=np.random.RandomState(2)), host, dev)
    assert np.array_equal(evaluation.mrr_score(m1, host, train=host), evaluation.mrr_score(m1, dev, train=dev))
    p1, r1 = evaluation.precision_recall_score(m1, host, k=5)
    p2, r2 = evaluation.precision_recall_score(m1, dev, k=5)
    assert np.array_equal(p1, p2) and np.array_equal(r1, r2)
    e1, _ = _same_fit(capsys, lambda: ExplicitFactorizationModel(
        loss='regression', embedding_dim=16, n_iter=2, batch_size=256, use_cuda=True,
        random_state=np.random.RandomState(4)), host, dev)
    assert evaluation.rmse_score(e1, host) == evaluation.rmse_score(e1, dev)


def test_pipeline_on_device_equals_host(capsys):
    """user_based_train_test_split -> to_sequence -> fit -> sequence scorers, CUDA vs NumPy."""
    from spotlight_b200 import evaluation
    from spotlight_b200.sequence.implicit import ImplicitSequenceModel
    inter = _sequence_data(seed=1, n=40000)
    outs = []
    for data in (inter, _dev(inter)):
        train, test = user_based_train_test_split(data, random_state=np.random.RandomState(7))
        train_s, test_s = train.to_sequence(15), test.to_sequence(15)
        model = ImplicitSequenceModel(loss='adaptive_hinge', representation='pooling', embedding_dim=16,
                                      n_iter=2, batch_size=64, use_cuda=True,
                                      random_state=np.random.RandomState(5))
        losses = _epoch_losses(capsys, model, train_s)
        p, r = evaluation.sequence_precision_recall_score(model, test_s, k=3)
        outs.append((losses, evaluation.sequence_mrr_score(model, test_s), p, r))
    assert outs[0][0] == outs[1][0]
    for a, b in zip(outs[0][1:], outs[1][1:]):
        assert np.array_equal(a, b)
    assert isinstance(test_s, SequenceInteractions) and test_s.sequences.is_cuda
