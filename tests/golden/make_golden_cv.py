"""Generate the data-preparation golden fixtures from the LIVE reference (build container only):
tests/golden/cv_splits.npz (shuffle_interactions, random_train_test_split and
user_based_train_test_split outputs with the generator state after each call) and
tests/golden/to_sequence_edges.npz (to_sequence on timestamp ties, negative timestamps, float
timestamps with +-0.0 and NaN, step_size > L and min_sequence_length in {0, 1, L}).

Run:  SPOTLIGHT_REFERENCE=<reference checkout> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_cv.py

The tests read only the committed fixtures.
"""

import os
import sys

import numpy as np

sys.dont_write_bytecode = True
sys.path.insert(0, os.environ['SPOTLIGHT_REFERENCE'])

from spotlight.cross_validation import (random_train_test_split, shuffle_interactions,  # noqa: E402
                                        user_based_train_test_split)
from spotlight.interactions import Interactions  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
COLUMNS = ('user_ids', 'item_ids', 'ratings', 'timestamps', 'weights')
# optional columns present in each case: none, each alone, all three
OPTIONAL = ((), ('ratings',), ('timestamps',), ('weights',), ('ratings', 'timestamps', 'weights'))


def split_inputs(seed, n=1000, num_users=400, num_items=250):
    rs = np.random.RandomState(seed)
    return dict(user_ids=rs.randint(0, num_users, n).astype(np.int32),
                item_ids=rs.randint(1, num_items, n).astype(np.int32),
                ratings=rs.randint(1, 6, n).astype(np.float32),
                timestamps=rs.randint(-10 ** 6, 10 ** 6, n).astype(np.int64),
                weights=rs.rand(n).astype(np.float32))


def store(out, tag, inter):
    for name in COLUMNS:
        value = getattr(inter, name)
        if value is not None:
            out['%s.%s' % (tag, name)] = value
    out[tag + '.num'] = np.array([inter.num_users, inter.num_items])


def store_state(out, tag, rs):
    st = rs.get_state()
    out[tag + '.key'] = st[1]
    out[tag + '.pos'] = np.array(st[2])


def make_splits():
    out = {}
    for case, present in enumerate(OPTIONAL):
        cols = split_inputs(case)
        for name in cols:
            out['in%d.%s' % (case, name)] = cols[name]
        inter = Interactions(cols['user_ids'], cols['item_ids'], num_users=400, num_items=250,
                             **{k: cols[k] for k in present})
        rs = np.random.RandomState(100 + case)
        store(out, 'shuffle%d' % case, shuffle_interactions(inter, random_state=rs))
        store_state(out, 'shuffle%d.rs' % case, rs)
        rs = np.random.RandomState(200 + case)
        train, test = random_train_test_split(inter, test_percentage=0.25, random_state=rs)
        store(out, 'random%d.train' % case, train)
        store(out, 'random%d.test' % case, test)
        store_state(out, 'random%d.rs' % case, rs)
        rs = np.random.RandomState(300 + case)
        train, test = user_based_train_test_split(inter, test_percentage=0.3, random_state=rs)
        store(out, 'user%d.train' % case, train)
        store(out, 'user%d.test' % case, test)
        store_state(out, 'user%d.rs' % case, rs)
    out['present'] = np.array([','.join(p) for p in OPTIONAL])
    np.savez_compressed(os.path.join(HERE, 'cv_splits.npz'), **out)


def edge_timestamps(rs, n):
    """(name, timestamps): ties, negative ints and floats with +-0.0 and NaN."""
    ties = rs.randint(0, 4, n).astype(np.int32)
    neg = rs.randint(-5, 3, n).astype(np.int64) * 10 ** 12
    f = rs.choice(np.array([-1.5, -0.0, 0.0, np.nan, 2.0, np.inf, -np.inf], dtype=np.float64), n)
    return [('ties_i32', ties), ('neg_i64', neg), ('float64', f), ('float32', f.astype(np.float32))]


def make_edges():
    out = {}
    rs = np.random.RandomState(7)
    n = 400
    users = rs.randint(-3, 40, n).astype(np.int64) * 3      # negative ids and gaps
    users[:60] = 5                                          # one long history
    items = rs.randint(1, 90, n).astype(np.int32)
    out['users'], out['items'] = users, items
    for ts_name, ts in edge_timestamps(rs, n):
        out['ts.' + ts_name] = ts
        inter = Interactions(users, items, timestamps=ts, num_users=200, num_items=90)
        for L, step in ((5, None), (5, 1), (5, 8), (7, 3)):
            for m in (None, 0, 1, L):
                s = inter.to_sequence(max_sequence_length=L, min_sequence_length=m, step_size=step)
                tag = '%s.L%d.s%s.m%s' % (ts_name, L, step, m)
                out['seq.' + tag] = s.sequences
                out['uid.' + tag] = s.user_ids
    np.savez_compressed(os.path.join(HERE, 'to_sequence_edges.npz'), **out)


if __name__ == '__main__':
    make_splits()
    make_edges()
