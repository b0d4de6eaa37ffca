"""CPU tests of the data-preparation surface: the host splits against fixtures from the live
reference (tests/golden/make_golden_cv.py), and oracle/prepare.py -- the NumPy restatement of the
device sort, window count and split mask -- against np.lexsort and the host to_sequence."""

import numpy as np
import pytest

from conftest import load_golden
from oracle import prepare as op
from spotlight_b200.cross_validation import (random_train_test_split, shuffle_interactions,
                                             user_based_train_test_split)
from spotlight_b200.interactions import Interactions

COLUMNS = ('user_ids', 'item_ids', 'ratings', 'timestamps', 'weights')


def _same(g, tag, inter):
    for name in COLUMNS:
        value = getattr(inter, name)
        key = '%s.%s' % (tag, name)
        if key not in g:
            assert value is None, key
            continue
        assert value.dtype == g[key].dtype and value.shape == g[key].shape, key
        assert value.tobytes() == g[key].tobytes(), key
    assert [inter.num_users, inter.num_items] == g[tag + '.num'].tolist()


def _same_state(g, tag, rs):
    st = rs.get_state()
    assert (st[1] == g[tag + '.key']).all() and st[2] == int(g[tag + '.pos']), tag


@pytest.mark.parametrize('case', range(5))
def test_host_splits_match_reference(case):
    g = load_golden('cv_splits')
    present = str(g['present'][case]).split(',') if g['present'][case] else []
    cols = {name: g['in%d.%s' % (case, name)] for name in COLUMNS}
    inter = Interactions(cols['user_ids'], cols['item_ids'], num_users=400, num_items=250,
                         **{k: cols[k] for k in present})
    rs = np.random.RandomState(100 + case)
    _same(g, 'shuffle%d' % case, shuffle_interactions(inter, random_state=rs))
    _same_state(g, 'shuffle%d.rs' % case, rs)
    rs = np.random.RandomState(200 + case)
    train, test = random_train_test_split(inter, test_percentage=0.25, random_state=rs)
    _same(g, 'random%d.train' % case, train)
    _same(g, 'random%d.test' % case, test)
    _same_state(g, 'random%d.rs' % case, rs)
    rs = np.random.RandomState(300 + case)
    train, test = user_based_train_test_split(inter, test_percentage=0.3, random_state=rs)
    _same(g, 'user%d.train' % case, train)
    _same(g, 'user%d.test' % case, test)
    _same_state(g, 'user%d.rs' % case, rs)


def test_user_split_needs_int32_user_ids():
    inter = Interactions(np.arange(10, dtype=np.int64), np.arange(10, dtype=np.int32) + 1)
    with pytest.raises(TypeError):
        user_based_train_test_split(inter, random_state=np.random.RandomState(0))


def test_split_mask_is_the_float64_comparison():
    """murmur % 100 / 100.0 < p (uint32 array -> float64) equals the 100-entry mask lookup."""
    from oracle.murmur import murmurhash3_32
    rs = np.random.RandomState(3)
    ids = rs.randint(-2 ** 31, 2 ** 31 - 1, 5000).astype(np.int32)
    for p in (0.0, 0.2, 0.25, 0.3, 0.07, 0.555, 1.0, 1.5):
        h = murmurhash3_32(ids, 12345).view(np.uint32)
        assert ((h % 100 / 100.0 < p) == op.split_mask(p)[h % 100]).all(), p


TS_DTYPES = (np.int32, np.int64, np.float32, np.float64)


def _timestamps(rs, n, dtype):
    if np.dtype(dtype).kind == 'f':
        return rs.choice(np.array([-2.5, -0.0, 0.0, np.nan, 1.0, 3.0, np.inf], dtype=dtype), n)
    return rs.randint(-4, 4, n).astype(dtype) * (2 ** 40 if dtype == np.int64 else 1)


@pytest.mark.parametrize('dtype', TS_DTYPES)
def test_oracle_radix_order_is_lexsort(dtype):
    rs = np.random.RandomState(1)
    for n in (1, 2, 50, 700):
        users = rs.randint(-5, 30, n).astype(np.int64) * 7
        ts = _timestamps(rs, n, dtype)
        expect = np.lexsort((ts, users))
        got = op.radix_order(op.user_key(users), op.time_key(ts))
        assert (got == expect).all(), (dtype, n)
    full = np.array([np.iinfo(np.int64).min, np.iinfo(np.int64).max, 0, -1, 5, 5], dtype=np.int64)
    u = np.zeros(len(full), dtype=np.int64)
    assert (op.radix_order(op.user_key(u), op.time_key(full)) == np.lexsort((full, u))).all()


def _one_user(c, dtype, rs):
    users = np.zeros(c, dtype=np.int64)
    items = rs.randint(1, 50, c).astype(np.int32)
    return Interactions(users, items, timestamps=_timestamps(rs, c, dtype), num_users=1, num_items=50)


@pytest.mark.parametrize('L', [1, 2, 7, 200])
def test_oracle_kept_windows_match_host(L):
    """The closed-form kept-window count over c, step and min_sequence_length (with NumPy's
    IndexError for columns out of range)."""
    rs = np.random.RandomState(L)
    for step in sorted({1, 3, L, L + 5}):
        for m in (None, 0, 1, 5, L, L + 1, -1):
            for c in range(1, 24):
                inter = _one_user(c, np.int64, rs)
                try:
                    host = len(inter.to_sequence(max_sequence_length=L, min_sequence_length=m,
                                                 step_size=step).sequences)
                except IndexError:
                    with pytest.raises(IndexError):
                        op.need_for(m, L)
                    continue
                assert op.kept_windows(c, step, op.need_for(m, L)) == host, (c, L, step, m)


@pytest.mark.parametrize('dtype', TS_DTYPES)
@pytest.mark.parametrize('L,step', [(1, 1), (2, 3), (7, 7), (7, 12), (200, 3)])
def test_oracle_to_sequence_matches_host(dtype, L, step):
    rs = np.random.RandomState(11)
    n = 300
    users = rs.randint(-3, 25, n).astype(np.int64) * 5
    users[:80] = 10
    items = rs.randint(1, 60, n).astype(np.int32)
    ts = _timestamps(rs, n, dtype)
    inter = Interactions(users, items, timestamps=ts, num_users=200, num_items=60)
    for m in sorted({None, 0, 1, min(5, L), L}, key=str):
        host = inter.to_sequence(max_sequence_length=L, min_sequence_length=m, step_size=step)
        seqs, uids = op.to_sequence(users, items, ts, L, m, step)
        assert (seqs == host.sequences).all() and (uids == host.user_ids).all(), (dtype, L, step, m)


def test_edge_fixture_matches_host_to_sequence():
    g = load_golden('to_sequence_edges')
    checked = 0
    for key in g:
        if not key.startswith('seq.'):
            continue
        tag = key[4:]
        ts_name, L, step, m = tag.split('.')
        L = int(L[1:])
        step = None if step == 'sNone' else int(step[1:])
        m = None if m == 'mNone' else int(m[1:])
        inter = Interactions(g['users'], g['items'], timestamps=g['ts.' + ts_name], num_users=200, num_items=90)
        s = inter.to_sequence(max_sequence_length=L, min_sequence_length=m, step_size=step)
        assert s.sequences.tobytes() == g[key].tobytes() and s.sequences.shape == g[key].shape, tag
        assert s.user_ids.tobytes() == g['uid.' + tag].tobytes(), tag
        seqs, uids = op.to_sequence(g['users'], g['items'], g['ts.' + ts_name], L, m, step)
        assert (seqs == g[key]).all() and (uids == g['uid.' + tag]).all(), tag
        checked += 1
    assert checked == 64
