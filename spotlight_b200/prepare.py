"""Device data preparation over the C-ABI (csrc/prepare.cu, include/spotlight_b200.h P1).

``sequence_rows`` is the CUDA branch of ``Interactions.to_sequence``; ``user_split_order`` and
``gather`` serve the CUDA branches of ``spotlight_b200.cross_validation``.  Every call runs on the
current stream of the tensors' device; the host reads back only the sizes it needs to allocate
the next output (key ranges, numbers of users, rows and train interactions).
"""

import torch

from spotlight_b200 import _lib
from spotlight_b200.ops import _ptr, _stream

_TS_KIND = {torch.int32: 0, torch.int64: 1, torch.float32: 2, torch.float64: 3}
_MAX_N = (1 << 31) - 1


def _workspace(nbytes, dev):
    return torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=dev)


def gather(index, src):
    """``src[index]`` in ``src``'s dtype: int32 / int64 CUDA ``index``, a 4- or 8-byte CUDA column."""
    if src.element_size() not in (4, 8):
        raise ValueError('gather: columns must have 4- or 8-byte elements, got %s' % src.dtype)
    if index.dtype not in (torch.int32, torch.int64):
        raise ValueError('gather: index must be int32 or int64')
    index, src = index.contiguous(), src.contiguous()
    out = torch.empty(index.numel(), dtype=src.dtype, device=src.device)
    _lib.check(_lib.load().slb_gather_elements(_ptr(index), index.element_size(), index.numel(), _ptr(src),
                                               src.element_size(), _ptr(out), _stream()), 'gather_elements')
    return out


def user_split_order(user_ids, seed, mask):
    """Stable train/test partition of int32 CUDA ``user_ids``: position i is a test interaction iff
    ``mask[murmur3_32(user_ids[i], seed) % 100]``.  Returns (int32 order: the train positions
    ascending then the test positions ascending, number of train positions)."""
    n = user_ids.numel()
    if not 1 <= n <= _MAX_N:
        raise ValueError('user_based_train_test_split on the device needs 1 <= n < 2**31 interactions')
    lib = _lib.load()
    bits = sum(1 << r for r in range(100) if mask[r])
    uids = user_ids.contiguous()
    order = torch.empty(n, dtype=torch.int32, device=uids.device)
    num_train = torch.empty(1, dtype=torch.int32, device=uids.device)
    ws = _workspace(lib.slb_user_split_workspace_bytes(n), uids.device)
    _lib.check(lib.slb_user_split_order(_ptr(uids), n, int(seed), bits & (2 ** 64 - 1), bits >> 64, _ptr(order),
                                        _ptr(num_train), _ptr(ws), ws.numel(), _stream()), 'user_split_order')
    return order, int(num_train.item())


def sequence_rows(user_ids, item_ids, timestamps, max_len, step, need):
    """(sequences int32 (rows, max_len), sequence user ids int32 (rows,)) on the device: the windows
    of each user's interactions in (timestamp, original position) order, users ascending, newest
    window first, left-padded with 0; with ``need >= 1`` only windows ending at least ``need``
    items into the user's list are kept.  Inputs are contiguous CUDA tensors on one device."""
    n = user_ids.numel()
    dev = user_ids.device
    lib = _lib.load()
    ukey = torch.empty(n, dtype=torch.int64, device=dev)
    tkey = torch.empty(n, dtype=torch.int64, device=dev)
    rng = torch.empty(4, dtype=torch.int64, device=dev)
    _lib.check(lib.slb_sort_keys(_ptr(user_ids), user_ids.element_size(), _ptr(timestamps),
                                 _TS_KIND[timestamps.dtype], n, _ptr(ukey), _ptr(tkey), _ptr(rng), _stream()),
               'sort_keys')
    umin, umax, tmin, tmax = (v & (2 ** 64 - 1) for v in rng.tolist())       # uint64 keys
    order = torch.empty(n, dtype=torch.int32, device=dev)
    ws = _workspace(max(lib.slb_radix_order_workspace_bytes(n), lib.slb_sequence_windows_workspace_bytes(n)), dev)
    _lib.check(lib.slb_radix_order(_ptr(ukey), umin, (umax - umin).bit_length(), _ptr(tkey), tmin,
                                   (tmax - tmin).bit_length(), n, _ptr(order), _ptr(ws), ws.numel(), _stream()),
               'radix_order')
    del tkey
    starts = torch.empty(n + 1, dtype=torch.int32, device=dev)
    row_offs = torch.empty(n + 1, dtype=torch.int32, device=dev)
    num_users = torch.empty(1, dtype=torch.int32, device=dev)
    _lib.check(lib.slb_sequence_windows(_ptr(order), _ptr(ukey), n, step, need, _ptr(starts), _ptr(row_offs),
                                        _ptr(num_users), _ptr(ws), ws.numel(), _stream()), 'sequence_windows')
    U, rows = torch.cat([num_users, row_offs[n:]]).tolist()
    sequences = torch.empty((rows, max_len), dtype=torch.int32, device=dev)
    sequence_users = torch.empty(rows, dtype=torch.int32, device=dev)
    _lib.check(lib.slb_sequence_emit(_ptr(order), _ptr(user_ids), user_ids.element_size(), _ptr(item_ids),
                                     item_ids.element_size(), _ptr(starts), _ptr(row_offs), U, rows, max_len,
                                     step, _ptr(sequences), _ptr(sequence_users), _stream()), 'sequence_emit')
    return sequences, sequence_users
