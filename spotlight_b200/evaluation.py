"""Evaluation scoring on the device (reference: spotlight/evaluation.py:9-220).

``mrr_score``, ``precision_recall_score``, ``sequence_mrr_score`` and
``sequence_precision_recall_score`` keep the reference's signatures and results, but instead
of one ``predict`` + host ``rankdata`` / ``argsort`` per user or sequence (minutes to hours at
1M users or 1M items) they score a block of users (sequences) against all items at once --
one GEMM for dot-product models -- and rank every test target of the block with one pass of
``slb_rank_targets`` over each score row.  That kernel returns, per target, the average rank
(``rankdata`` of the negated scores: the MRR) and the stable position (where the target lands in
``argsort(-row, kind='stable')``: a hit at k iff position < k, for every k at once).

Known train items (``train=``) or the items of the input sequence (``exclude_preceding=True``)
are overwritten with ``-FLOAT_MAX`` in the block, exactly as the reference overwrites the negated
predictions with ``FLOAT_MAX``, so excluded targets are ranked with that score.

Ties: where exactly equal scores straddle the k boundary, precision/recall order them by
ascending item id (numpy's ``kind='stable'``); the reference's default ``argsort`` breaks such
ties in an unspecified order.
"""

import numpy as np
import torch

from spotlight_b200 import _lib, ops
from spotlight_b200.factorization.representations import BilinearNet
from spotlight_b200.layers import ScaledEmbedding
from spotlight_b200.sequence.representations import LSTMNet, _SeqNetBase

FLOAT_MAX = np.finfo(np.float32).max

_PAIRS_PER_CHUNK = 1 << 18      # (row, item) pairs per forward() call of the generic scorers


def _item_matrix(layer, num_items, dev):
    """(num_items, D) item vectors: the weight of a plain table, otherwise the layer's own
    forward over every id (for Bloom: the summed hashed rows)."""
    if type(layer) is ScaledEmbedding:
        return layer.weight
    return layer(torch.arange(num_items, device=dev)).reshape(num_items, -1)


def _generic_block(forward, reps, num_items, dev):
    """(len(reps), num_items) scores through the net's own pairwise forward, item chunk by item
    chunk: forward(rows of reps repeated per item, items (n, ...)) -> (n,)."""
    n = reps.shape[0]
    out = torch.empty(n, num_items, dtype=torch.float32, device=dev)
    chunk = max(1, _PAIRS_PER_CHUNK // max(n, 1))
    for lo in range(0, num_items, chunk):
        items = torch.arange(lo, min(num_items, lo + chunk), device=dev)
        c = items.numel()
        out[:, lo:lo + c] = forward(reps.repeat_interleave(c, 0), items.repeat(n)).reshape(n, c)
    return out


def _score_block(model, user_ids):
    """(len(user_ids), num_items) scores of factorization-model users against every item."""
    net = model._net
    num_items = model._num_items
    if hasattr(model._optimizer, 'flush'):
        model._optimizer.flush()
    net.train(False)
    with torch.no_grad():
        if not isinstance(net, BilinearNet):
            return _generic_block(net, user_ids, num_items, user_ids.device)
        dim = net.embedding_dim
        items = _item_matrix(net.item_embeddings, num_items, user_ids.device)
        u = net.user_embeddings(user_ids).reshape(-1, dim)
        out = u @ items.t()                                 # plain library GEMM (cuBLAS)
        out += net.user_biases(user_ids).reshape(-1, 1)
        out += net.item_biases.weight.reshape(1, -1)
    return out


def _score_sequences(model, sequences):
    """(len(sequences), num_items) next-item scores of a block of input sequences."""
    net = model._net
    num_items = model._num_items
    if hasattr(model._optimizer, 'flush'):
        model._optimizer.flush()
    net.train(False)
    with torch.no_grad():
        final = net.user_representation(sequences)[1]
        if isinstance(net, (_SeqNetBase, LSTMNet)) and final.dim() == 2:
            # the dot head of _SeqNetBase.forward for a 2-D representation, as one GEMM
            items = _item_matrix(net.item_embeddings, num_items, sequences.device)
            out = final @ items.t()
            out += net.item_biases.weight.reshape(1, -1)
            return out
        return _generic_block(lambda r, t: net(r, t.reshape(-1, 1)), final, num_items, sequences.device)


def _exclude(scores, rows, items):
    """Push (rows[j], items[j]) of the block to the bottom: the reference's FLOAT_MAX overwrite
    of the negated predictions."""
    if len(rows):
        dev = scores.device
        scores[torch.from_numpy(np.asarray(rows, dtype=np.int64)).to(dev),
               torch.from_numpy(np.asarray(items, dtype=np.int64)).to(dev)] = -float(FLOAT_MAX)


def _rank_targets(scores, row_ptr, targets, avg_rank=False, position=False):
    """slb_rank_targets over the block: targets of row r are targets[row_ptr[r]:row_ptr[r+1]].
    Returns (avg_rank float64 or None, position int64 or None) as NumPy arrays."""
    lib = _lib.load()
    dev = scores.device
    ops.require_cuda(scores)
    scores = scores.contiguous()
    rp = torch.from_numpy(np.ascontiguousarray(row_ptr, dtype=np.int64)).to(dev)
    tg = torch.from_numpy(np.ascontiguousarray(targets, dtype=np.int64)).to(dev)
    n = tg.numel()
    ar = torch.empty(n, dtype=torch.float32, device=dev) if avg_rank else None
    pos = torch.empty(n, dtype=torch.int64, device=dev) if position else None
    _lib.check(lib.slb_rank_targets(ops._ptr(scores), scores.shape[0], scores.shape[1], ops._ptr(rp),
                                    ops._ptr(tg), n, ops._ptr(ar), ops._ptr(pos), ops._stream()),
               'rank_targets')
    return (ar.double().cpu().numpy() if avg_rank else None,
            pos.cpu().numpy() if position else None)


def _check_items(ids, num_items):
    if len(ids) and (ids.min() < 0 or ids.max() >= num_items):
        raise ValueError('Item ids must lie in [0, %d), the model\'s number of items.' % num_items)


def _user_blocks(model, test, train, user_block):
    """Yield (first output row, score block, CSR test rows) for the users with test items."""
    test = test.tocsr()
    train = train.tocsr() if train is not None else None
    for m in (test, train):
        if m is not None:
            _check_items(m.indices, model._num_items)
    dev = next(model._net.parameters()).device
    users = np.nonzero(np.diff(test.indptr))[0]
    for lo in range(0, len(users), user_block):
        blk = users[lo:lo + user_block]
        scores = _score_block(model, torch.from_numpy(blk.astype(np.int64)).to(dev))
        if train is not None:
            tr = train[blk]
            _exclude(scores, np.repeat(np.arange(len(blk)), np.diff(tr.indptr)), tr.indices)
        yield lo, scores, test[blk]


def mrr_score(model, test, train=None, user_block=2048):
    """Mean reciprocal rank per user with test interactions (evaluation.py:9-56).

    One score per user with test items: the mean of 1 / average rank (``rankdata`` of the
    negated predictions) over the user's test items; train items, when given, are pushed to
    the bottom.  ``user_block`` users are scored per GEMM.
    """
    n_users = int((np.diff(test.tocsr().indptr) > 0).sum())
    out = np.empty(n_users, dtype=np.float64)
    for lo, scores, te in _user_blocks(model, test, train, user_block):
        ranks, _ = _rank_targets(scores, te.indptr, te.indices, avg_rank=True)
        n_per = np.diff(te.indptr)
        sums = np.add.reduceat(1.0 / ranks, te.indptr[:-1])
        out[lo:lo + len(n_per)] = sums / n_per
    return out


def _hits_at(position, row_ptr, ks, unique=None):
    """(n_rows, len(ks)) count of targets with position < k per row (only where ``unique``)."""
    n = len(row_ptr) - 1
    hits = np.zeros((n, len(ks)), dtype=np.int64)
    rows = np.repeat(np.arange(n), np.diff(row_ptr))
    for j, k in enumerate(ks):
        hit = position < k
        if unique is not None:
            hit &= unique
        hits[:, j] = np.bincount(rows[hit], minlength=n)
    return hits


def precision_recall_score(model, test, train=None, k=10, user_block=2048):
    """Precision@k and recall@k per user with test interactions (evaluation.py:154-220).

    ``k`` is an int or an array of ints; every k comes from one ranking pass.  precision =
    hits / min(k, num_items), recall = hits / the user's number of test items.  Shapes follow
    the reference's ``.squeeze()``: ``(n_users,)`` for a scalar k, ``(n_users, len(k))`` for an
    array.  Exact score ties across the k boundary are ordered by ascending item id (numpy's
    ``argsort(kind='stable')``); the reference's default argsort orders them arbitrarily.
    """
    ks = np.array([k]) if np.isscalar(k) else np.asarray(k)
    n_users = int((np.diff(test.tocsr().indptr) > 0).sum())
    hits = np.empty((n_users, len(ks)), dtype=np.int64)
    n_test = np.empty(n_users, dtype=np.int64)
    for lo, scores, te in _user_blocks(model, test, train, user_block):
        _, pos = _rank_targets(scores, te.indptr, te.indices, position=True)
        n = len(te.indptr) - 1
        hits[lo:lo + n] = _hits_at(pos, te.indptr, ks)
        n_test[lo:lo + n] = np.diff(te.indptr)
    precision = hits / np.minimum(ks, model._num_items).reshape(1, -1).astype(np.float64)
    recall = hits / n_test.reshape(-1, 1).astype(np.float64)
    return precision.squeeze(), recall.squeeze()


def _sequence_blocks(model, inputs, exclude_preceding, sequence_block):
    """Yield (first row, score block) over blocks of input sequences."""
    dev = next(model._net.parameters()).device
    for lo in range(0, len(inputs), sequence_block):
        blk = np.ascontiguousarray(inputs[lo:lo + sequence_block], dtype=np.int64)
        scores = _score_sequences(model, torch.from_numpy(blk).to(dev))
        if exclude_preceding:
            _exclude(scores, np.repeat(np.arange(len(blk)), blk.shape[1]), blk.reshape(-1))
        yield lo, scores


def sequence_mrr_score(model, test, exclude_preceding=False, sequence_block=256):
    """Reciprocal rank of the last item of every test sequence given the rest
    (evaluation.py:59-102).

    With ``exclude_preceding`` every item of the input prefix -- padding id 0 included, as in the
    reference -- is pushed to the bottom.  ``sequence_block`` sequences are scored at once.
    """
    _check_items(test.sequences.reshape(-1), model._num_items)
    sequences = test.sequences[:, :-1]
    targets = test.sequences[:, -1].astype(np.int64)
    out = np.empty(len(sequences), dtype=np.float64)
    for lo, scores in _sequence_blocks(model, sequences, exclude_preceding, sequence_block):
        n = scores.shape[0]
        ranks, _ = _rank_targets(scores, np.arange(n + 1), targets[lo:lo + n], avg_rank=True)
        out[lo:lo + n] = 1.0 / ranks
    return out


def sequence_precision_recall_score(model, test, k=10, exclude_preceding=False, sequence_block=256):
    """Precision@k and recall@k of the last k items of every test sequence given the rest
    (evaluation.py:105-151).

    Hits count the distinct target items (padding id 0 counts as an item) ranked in the top k;
    precision = hits / min(k, num_items), recall = hits / k.  ``k`` must be shorter than the
    sequences.  Exact score ties across the k boundary are ordered by ascending item id.
    """
    S = test.sequences.shape[1]
    if not 0 < k < S:
        raise ValueError('k = %d must be in [1, sequence length %d)' % (k, S))
    _check_items(test.sequences.reshape(-1), model._num_items)
    sequences = test.sequences[:, :-k]
    targets = np.sort(test.sequences[:, -k:].astype(np.int64), axis=1)
    unique = np.ones(targets.shape, dtype=bool)
    unique[:, 1:] = targets[:, 1:] != targets[:, :-1]
    hits = np.empty(len(sequences), dtype=np.int64)
    for lo, scores in _sequence_blocks(model, sequences, exclude_preceding, sequence_block):
        n = scores.shape[0]
        row_ptr = np.arange(n + 1) * k
        _, pos = _rank_targets(scores, row_ptr, targets[lo:lo + n].reshape(-1), position=True)
        hits[lo:lo + n] = _hits_at(pos, row_ptr, [k], unique[lo:lo + n].reshape(-1))[:, 0]
    return hits / float(min(k, model._num_items)), hits / float(k)


_RMSE_BLOCK = 1 << 22           # test pairs per predict + reduction launch


def rmse_score(model, test):
    """Root mean squared error of the model's predicted ratings on the test pairs
    (evaluation.py:223-244).

    The pairs are scored on the device in blocks through the model's prediction kernels
    (``exp`` / ``sigmoid`` applied for poisson / logistic models, as ``predict`` does); each
    block's mean squared error comes from the deterministic ``slb_rating_loss`` reduction and the
    blocks are combined in float64.  Returns a NumPy float32 like the reference.
    """
    n = len(test.user_ids)
    if test.ratings is None:
        raise TypeError("unsupported operand type(s) for -: 'NoneType' and 'float'")
    model._check_input(test.user_ids, test.item_ids)
    dev = next(model._net.parameters()).device
    predict_device = getattr(model, '_predict_device', None)
    total = 0.0
    for lo in range(0, n, _RMSE_BLOCK):
        hi = min(n, lo + _RMSE_BLOCK)
        users = torch.from_numpy(np.asarray(test.user_ids[lo:hi], dtype=np.int64)).to(dev)
        items = torch.from_numpy(np.asarray(test.item_ids[lo:hi], dtype=np.int64)).to(dev)
        ratings = torch.from_numpy(np.asarray(test.ratings[lo:hi], dtype=np.float32)).to(dev)
        if predict_device is not None:
            pred = predict_device(users, items)
        else:
            pred = torch.from_numpy(np.asarray(model.predict(test.user_ids[lo:hi], test.item_ids[lo:hi]),
                                               dtype=np.float32)).to(dev)
        mse, _ = ops.rating_loss(pred.reshape(-1).contiguous(), ratings, _lib.LOSS_KIND['regression'])
        total += float(mse) * (hi - lo)
    return np.float32(np.sqrt(total / n))
