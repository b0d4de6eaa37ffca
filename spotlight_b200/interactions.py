"""Data containers with the reference's attributes and behaviour
(spotlight/interactions.py:38-312).

An ``Interactions`` holds either NumPy arrays or CUDA tensors on one device.  With NumPy
arrays ``to_sequence`` is host code, vectorised instead of the reference's per-window Python
generator (interactions.py:11-35, 250-257) but returning the same matrices; with CUDA tensors
it runs on the device (csrc/prepare.cu) and returns the same matrices as CUDA tensors.
"""

import numpy as np
import scipy.sparse as sp
import torch

_COLUMNS = ('user_ids', 'item_ids', 'ratings', 'timestamps', 'weights')


def _device_of(data, names=_COLUMNS):
    """The CUDA device of ``data``'s present columns, or None when none is a CUDA tensor.
    A mix of CUDA tensors and other arrays, or of CUDA devices, raises ``ValueError``."""
    cols = [getattr(data, name) for name in names if getattr(data, name) is not None]
    on_cuda = [torch.is_tensor(c) and c.is_cuda for c in cols]
    if not any(on_cuda):
        return None
    if not all(on_cuda) or len(set(c.device for c in cols)) != 1:
        raise ValueError('Interactions must hold either all NumPy arrays or all CUDA tensors on one device')
    return cols[0].device


def _to_host(data):
    """``data`` itself when it holds no CUDA tensor, otherwise a copy with NumPy columns."""
    if isinstance(data, SequenceInteractions):
        if _device_of(data, ('sequences', 'user_ids')) is None:
            return data
        return SequenceInteractions(data.sequences.cpu().numpy(),
                                    user_ids=None if data.user_ids is None else data.user_ids.cpu().numpy(),
                                    num_items=data.num_items)
    if _device_of(data) is None:
        return data
    cols = {name: None if getattr(data, name) is None else getattr(data, name).cpu().numpy()
            for name in _COLUMNS}
    return Interactions(cols.pop('user_ids'), cols.pop('item_ids'), num_users=data.num_users,
                        num_items=data.num_items, **cols)


def _column_index(min_sequence_length, L):
    """The column ``sequences[:, -min_sequence_length]`` reads, with NumPy's IndexError."""
    i = -int(min_sequence_length)
    if not -L <= i < L:
        raise IndexError('index %d is out of bounds for axis 1 with size %d' % (i, L))
    return i + L if i < 0 else i


class Interactions(object):
    """User-item interaction pairs, optionally with ratings, timestamps and
    weights (interactions.py:38-149).

    Attributes: ``user_ids, item_ids, ratings, timestamps, weights, num_users,
    num_items``.
    """

    def __init__(self, user_ids, item_ids, ratings=None, timestamps=None, weights=None,
                 num_users=None, num_items=None):
        self.num_users = num_users or int(user_ids.max() + 1)
        self.num_items = num_items or int(item_ids.max() + 1)
        self.user_ids = user_ids
        self.item_ids = item_ids
        self.ratings = ratings
        self.timestamps = timestamps
        self.weights = weights
        self._check()

    def __repr__(self):
        return ('<Interactions dataset ({num_users} users x {num_items} items '
                'x {num_interactions} interactions)>'
                .format(num_users=self.num_users, num_items=self.num_items,
                        num_interactions=len(self)))

    def __len__(self):
        return len(self.user_ids)

    def _check(self):
        if self.user_ids.max() >= self.num_users:
            raise ValueError('Maximum user id greater than declared number of users.')
        if self.item_ids.max() >= self.num_items:
            raise ValueError('Maximum item id greater than declared number of items.')
        n = len(self.user_ids)
        for name, value in (('item IDs', self.item_ids), ('ratings', self.ratings),
                            ('timestamps', self.timestamps), ('weights', self.weights)):
            if value is not None and len(value) != n:
                raise ValueError('Invalid {} dimensions: length must be equal to number of '
                                 'interactions'.format(name))

    def tocoo(self):
        """scipy.sparse COO matrix of the interactions (interactions.py:151-161)."""
        data = self.ratings if self.ratings is not None else np.ones(len(self))
        return sp.coo_matrix((data, (self.user_ids, self.item_ids)),
                             shape=(self.num_users, self.num_items))

    def tocsr(self):
        return self.tocoo().tocsr()

    def to_sequence(self, max_sequence_length=10, min_sequence_length=None, step_size=None):
        """Left-zero-padded ``(num_sequences, max_sequence_length)`` int32 matrix of
        each user's time-ordered items, one row per sliding window, newest window
        first (interactions.py:170-266).
        """
        if self.timestamps is None:
            raise ValueError('Cannot convert to sequences, timestamps not available.')
        dev = _device_of(self)
        if dev is not None:
            return self._to_sequence_device(max_sequence_length, min_sequence_length, step_size)
        if 0 in self.item_ids:
            raise ValueError('0 is used as an item id, conflicting with the sequence '
                             'padding value.')
        if step_size is None:
            step_size = max_sequence_length
        L = int(max_sequence_length)

        order = np.lexsort((self.timestamps, self.user_ids))
        users = self.user_ids[order]
        items = self.item_ids[order]
        uniq, first, counts = np.unique(users, return_index=True, return_counts=True)

        windows = np.ceil(counts / float(step_size)).astype(np.int64)
        total = int(windows.sum())
        owner = np.repeat(np.arange(len(uniq)), windows)             # user of each row
        rank = np.arange(total) - np.repeat(np.cumsum(windows) - windows, windows)
        end = counts[owner] - rank * step_size                        # window end (exclusive)
        src = end[:, None] - L + np.arange(L)[None, :]                # position in user's list
        valid = src >= 0
        flat = first[owner][:, None] + np.where(valid, src, 0)
        sequences = np.where(valid, items[flat], 0).astype(np.int32)
        sequence_users = uniq[owner].astype(np.int32)

        if min_sequence_length is not None:
            keep = sequences[:, -min_sequence_length] != 0
            sequences = sequences[keep]
            sequence_users = sequence_users[keep]

        return SequenceInteractions(sequences, user_ids=sequence_users, num_items=self.num_items)

    def _to_sequence_device(self, max_sequence_length, min_sequence_length, step_size):
        """``to_sequence`` of CUDA columns: a stable radix sort of (user, timestamp) and one
        kernel writing the windows; the same matrices as the host branch, as CUDA tensors."""
        from spotlight_b200 import prepare
        users, items, ts = self.user_ids, self.item_ids, self.timestamps
        if users.dtype not in (torch.int32, torch.int64) or items.dtype not in (torch.int32, torch.int64):
            raise TypeError('to_sequence on the device needs int32 or int64 user and item ids')
        if ts.dtype not in (torch.int32, torch.int64, torch.float32, torch.float64):
            raise TypeError('to_sequence on the device needs int32, int64, float32 or float64 timestamps, '
                            'got %s' % ts.dtype)
        if self.num_items >= 2 ** 31:
            raise ValueError('to_sequence on the device needs num_items < 2**31')
        n = len(users)
        if not 1 <= n < 2 ** 31:
            raise ValueError('to_sequence on the device needs 1 <= n < 2**31 interactions')
        if bool((items == 0).any()):
            raise ValueError('0 is used as an item id, conflicting with the sequence '
                             'padding value.')
        L = int(max_sequence_length)
        step = L if step_size is None else int(step_size)
        if L < 1 or step < 1 or (step_size is not None and step != step_size):
            raise ValueError('to_sequence on the device needs integer max_sequence_length >= 1 '
                             'and step_size >= 1')
        need = -1 if min_sequence_length is None else L - _column_index(min_sequence_length, L)
        with torch.cuda.device(users.device):
            sequences, sequence_users = prepare.sequence_rows(users.contiguous(), items.contiguous(),
                                                              ts.contiguous(), L, step, need)
        return SequenceInteractions(sequences, user_ids=sequence_users, num_items=self.num_items)


class SequenceInteractions(object):
    """Sequence matrix container (interactions.py:269-312)."""

    def __init__(self, sequences, user_ids=None, num_items=None):
        self.sequences = sequences
        self.user_ids = user_ids
        self.max_sequence_length = sequences.shape[1]
        self.num_items = sequences.max() + 1 if num_items is None else num_items

    def __repr__(self):
        num_sequences, sequence_length = self.sequences.shape
        return ('<Sequence interactions dataset ({num_sequences} sequences x '
                '{sequence_length} sequence length)>'
                .format(num_sequences=num_sequences, sequence_length=sequence_length))
