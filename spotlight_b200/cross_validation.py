"""Shuffling and train/test splitting of ``Interactions`` with the reference's signatures,
defaults and ``random_state`` consumption (spotlight/cross_validation.py:12-176).

NumPy interactions give the reference's outputs byte for byte.  CUDA interactions stay on
their device and give the same arrays as CUDA tensors:

- ``shuffle_interactions`` / ``random_train_test_split`` take their permutation from the
  bit-exact device shuffle (csrc/shuffle.cu) for 2**17 <= n <= 2**29, otherwise from the host
  shuffle, and gather every column with ``slb_gather_elements``;
- ``user_based_train_test_split`` hashes the user ids and partitions every column stably on
  the device (``slb_user_split_order``).  The seed is drawn on the host as the reference draws
  it, and the float64 comparison ``h % 100 / 100.0 < test_percentage`` becomes a 100-entry
  mask built on the host, so the device does no float arithmetic.
"""

import numpy as np
import torch

from spotlight_b200.interactions import Interactions, _device_of
from spotlight_b200.rng import SHUFFLE_DEVICE_MAX, shuffled_order_device
from spotlight_b200.torch_utils import shuffled_order

DEVICE_SHUFFLE_MIN = 1 << 17        # as the models' fit(): both permutations are bit-exact


def _index_or_none(array, index):
    return None if array is None else array[index]


def _subset(interactions, index):
    """The interactions at ``index`` (an index array, a boolean mask or a slice)."""
    return Interactions(interactions.user_ids[index],
                        interactions.item_ids[index],
                        ratings=_index_or_none(interactions.ratings, index),
                        timestamps=_index_or_none(interactions.timestamps, index),
                        weights=_index_or_none(interactions.weights, index),
                        num_users=interactions.num_users,
                        num_items=interactions.num_items)


def _gathered(interactions, order):
    """``_subset(interactions, order)`` of CUDA interactions, one device gather per column."""
    from spotlight_b200.prepare import gather
    cols = {}
    for name in ('user_ids', 'item_ids', 'ratings', 'timestamps', 'weights'):
        col = getattr(interactions, name)
        cols[name] = None if col is None else gather(order, col)
    return Interactions(cols.pop('user_ids'), cols.pop('item_ids'), num_users=interactions.num_users,
                        num_items=interactions.num_items, **cols)


def _device_order(n, random_state, dev):
    """``random_state.shuffle(arange(n))`` as a CUDA tensor."""
    if DEVICE_SHUFFLE_MIN <= n <= SHUFFLE_DEVICE_MAX and random_state.get_state()[0] == 'MT19937':
        return shuffled_order_device(n, random_state, dev)
    return torch.from_numpy(shuffled_order(n, random_state)).to(dev)


def shuffle_interactions(interactions, random_state=None):
    """The interactions in the order of one ``random_state.shuffle`` of their positions
    (cross_validation.py:20-55)."""
    if random_state is None:
        random_state = np.random.RandomState()
    dev = _device_of(interactions)
    if dev is None:
        shuffle_indices = np.arange(len(interactions.user_ids))
        random_state.shuffle(shuffle_indices)
        return _subset(interactions, shuffle_indices)
    with torch.cuda.device(dev):
        return _gathered(interactions, _device_order(len(interactions.user_ids), random_state, dev))


def random_train_test_split(interactions, test_percentage=0.2, random_state=None):
    """(train, test): the first ``int((1.0 - test_percentage) * n)`` shuffled interactions and
    the rest (cross_validation.py:58-111)."""
    interactions = shuffle_interactions(interactions, random_state=random_state)
    cutoff = int((1.0 - test_percentage) * len(interactions))
    return (_subset(interactions, slice(None, cutoff)),
            _subset(interactions, slice(cutoff, None)))


def user_based_train_test_split(interactions, test_percentage=0.2, random_state=None):
    """(train, test) with every user's interactions on one side: a user is in the test set
    when ``murmurhash3_32(user_id, seed, positive=True) % 100 / 100.0 < test_percentage``,
    the seed drawn from ``random_state`` (cross_validation.py:114-176).  Both sides keep the
    interactions' original order.  User ids must be int32, as sklearn's hash requires."""
    if random_state is None:
        random_state = np.random.RandomState()
    seed = random_state.randint(np.iinfo(np.uint32).min, np.iinfo(np.uint32).max, dtype=np.int64)
    dev = _device_of(interactions)
    if dev is None:
        from sklearn.utils import murmurhash3_32
        in_test = (murmurhash3_32(interactions.user_ids, seed=seed, positive=True) % 100 / 100.0) < test_percentage
        return _subset(interactions, np.logical_not(in_test)), _subset(interactions, in_test)
    from spotlight_b200.prepare import user_split_order
    uids = interactions.user_ids
    if uids.dtype != torch.int32:
        raise TypeError('key.dtype should be int32, got %s' % str(uids.dtype).replace('torch.', ''))
    mask = [(r / 100.0) < test_percentage for r in range(100)]
    with torch.cuda.device(dev):
        order, num_train = user_split_order(uids, seed, mask)
        both = _gathered(interactions, order)
    return _subset(both, slice(None, num_train)), _subset(both, slice(num_train, None))
