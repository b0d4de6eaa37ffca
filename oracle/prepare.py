"""NumPy restatement of the device data preparation (spotlight_b200/csrc/prepare.cu), so the
algorithms can be checked on the CPU against np.lexsort and the host ``to_sequence``:

* ``user_key`` / ``time_key``: the order-preserving uint64 keys;
* ``radix_order``: the stable LSD passes, 8 bits of (key - min) per pass, timestamps first;
* ``kept_windows``: the closed-form count of windows that survive ``min_sequence_length``;
* ``to_sequence``: the rows the emit kernel writes;
* ``split_mask``: the 100-entry test mask of ``user_based_train_test_split``.
"""

import numpy as np

_SIGN = np.uint64(1 << 63)


def user_key(ids):
    return ids.astype(np.int64).view(np.uint64) ^ _SIGN


def time_key(ts):
    if ts.dtype.kind in 'iu':
        return ts.astype(np.int64).view(np.uint64) ^ _SIGN
    v = ts.astype(np.float64)
    v = np.where(v == 0.0, 0.0, v)                     # -0.0 -> +0.0
    b = v.view(np.uint64)
    key = np.where(b >> np.uint64(63), ~b, b | _SIGN)
    return np.where(np.isnan(v), np.uint64(2 ** 64 - 1), key)


def _stable_pass(order, digit):
    """One histogram / exclusive scan / in-order scatter pass: a stable counting sort."""
    d = digit[order]
    counts = np.bincount(d, minlength=256)
    start = np.concatenate([[0], np.cumsum(counts)[:-1]])
    rank = np.empty(len(d), dtype=np.int64)
    for v in np.unique(d):
        where = np.nonzero(d == v)[0]
        rank[where] = start[v] + np.arange(len(where))
    out = np.empty_like(order)
    out[rank] = order
    return out


def radix_order(ukey, tkey):
    """np.lexsort((tkey, ukey)) by LSD passes over the used bits of the range-reduced keys."""
    order = np.arange(len(ukey), dtype=np.int64)
    for key in (tkey, ukey):
        rel = key - key.min()
        bits = int(rel.max()).bit_length()
        for shift in range(0, bits, 8):
            order = _stable_pass(order, ((rel >> np.uint64(shift)) & np.uint64(0xFF)).astype(np.int64))
    return order


def need_for(min_sequence_length, L):
    """-1 (no filter) or the items a window must reach: L minus the column that
    ``sequences[:, -min_sequence_length]`` reads; IndexError as NumPy raises it."""
    if min_sequence_length is None:
        return -1
    i = -int(min_sequence_length)
    if not -L <= i < L:
        raise IndexError('index %d is out of bounds for axis 1 with size %d' % (i, L))
    return L - (i + L if i < 0 else i)


def kept_windows(c, step, need):
    """Windows kept for a user with c interactions: the newest min(w, (c - need) // step + 1)."""
    w = -(-c // step)
    if need < 0:
        return w
    return min(w, (c - need) // step + 1) if c >= need else 0


def to_sequence(users, items, ts, L, min_sequence_length=None, step=None):
    step = L if step is None else step
    need = need_for(min_sequence_length, L)
    order = radix_order(user_key(users), time_key(ts))
    su, si = users[order], items[order]
    starts = np.nonzero(np.concatenate([[True], su[1:] != su[:-1]]))[0]
    ends = np.concatenate([starts[1:], [len(su)]])
    rows, row_users = [], []
    for s, e in zip(starts, ends):
        c = e - s
        for r in range(kept_windows(c, step, need)):
            end = c - r * step
            row = np.zeros(L, dtype=np.int32)
            src = end - L + np.arange(L)
            row[src >= 0] = si[s + src[src >= 0]]
            rows.append(row)
            row_users.append(np.int32(su[s]))
    return (np.array(rows, dtype=np.int32).reshape(-1, L), np.array(row_users, dtype=np.int32))


def split_mask(test_percentage):
    return np.array([(r / 100.0) < test_percentage for r in range(100)])
