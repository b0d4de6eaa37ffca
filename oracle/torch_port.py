"""The reference's fit() loop restated on stock torch CPU ops (oracle).

TEST INFRASTRUCTURE / TIMED CPU BASELINE ONLY -- never imported by
``spotlight_b200``.  The reference is pure Python over ATen and is not part of
this repository (bench.py uses it only when build() placed it in oracle/_ref),
so this module restates its hot
path with the *same* ATen ops in the same order, which gives the same
arithmetic and the same performance characteristics on the host cores:

* ``BilinearNet``       spotlight/factorization/representations.py:39-91
  (4x nn.Embedding, init layers.py:29-37 / 48-56)
* losses                spotlight/losses.py:40-50, 82-90, 115-124, 164-166
* the minibatch loop    spotlight/factorization/implicit.py:210-252, 254-275
  (host shuffle, host ``randint`` negatives, autograd backward,
  ``optimizer.step()``)

tests/test_oracle_port.py checks it against the golden fit trajectories of the
live reference (tests/golden/fit_*.npz).
"""

import numpy as np
import torch
import torch.nn as nn


class PortBilinearNet(nn.Module):
    def __init__(self, num_users, num_items, embedding_dim=32, sparse=False):
        super(PortBilinearNet, self).__init__()
        self.embedding_dim = embedding_dim
        self.user_embeddings = nn.Embedding(num_users, embedding_dim, sparse=sparse)
        self.item_embeddings = nn.Embedding(num_items, embedding_dim, sparse=sparse)
        self.user_biases = nn.Embedding(num_users, 1, sparse=sparse)
        self.item_biases = nn.Embedding(num_items, 1, sparse=sparse)
        with torch.no_grad():
            self.user_embeddings.weight.normal_(0, 1.0 / embedding_dim)
            self.item_embeddings.weight.normal_(0, 1.0 / embedding_dim)
            self.user_biases.weight.zero_()
            self.item_biases.weight.zero_()

    def forward(self, user_ids, item_ids):
        user_embedding = self.user_embeddings(user_ids).squeeze()
        item_embedding = self.item_embeddings(item_ids).squeeze()
        user_bias = self.user_biases(user_ids).squeeze()
        item_bias = self.item_biases(item_ids).squeeze()
        return (user_embedding * item_embedding).sum(1) + user_bias + item_bias


def _loss(kind, pos, neg):
    if kind == 'pointwise':
        return ((1.0 - torch.sigmoid(pos)) + torch.sigmoid(neg)).mean()
    if kind == 'bpr':
        return (1.0 - torch.sigmoid(pos - neg)).mean()
    if kind == 'adaptive_hinge':
        neg, _ = torch.max(neg, 0)
    return torch.clamp(neg - pos + 1.0, 0.0).mean()


def fit_steps(net, optimizer, users, items, num_items, batch_size, loss, random_state,
              n_neg=5, max_steps=None):
    """One epoch (or ``max_steps`` minibatches) of the reference loop.

    ``users`` / ``items``: already shuffled int64 arrays.  Returns the list of
    per-batch losses.
    """
    ut, it = torch.from_numpy(users), torch.from_numpy(items)
    losses = []
    for lo in range(0, len(users), batch_size):
        if max_steps is not None and len(losses) >= max_steps:
            break
        bu, bi = ut[lo:lo + batch_size], it[lo:lo + batch_size]
        pos = net(bu, bi)
        if loss == 'adaptive_hinge':
            B = bu.size(0)
            rep = bu.view(B, 1).expand(B, n_neg).reshape(B * n_neg)
            negs = random_state.randint(0, num_items, len(rep), dtype=np.int64)
            neg = net(rep, torch.from_numpy(negs)).view(n_neg, B)
        else:
            negs = random_state.randint(0, num_items, len(bu), dtype=np.int64)
            neg = net(bu, torch.from_numpy(negs))
        optimizer.zero_grad()
        lv = _loss(loss, pos, neg)
        losses.append(lv.item())
        lv.backward()
        optimizer.step()
    return losses


def fit(net, optimizer, user_ids, item_ids, num_items, batch_size, loss, random_state,
        n_iter=1, n_neg=5):
    """Full reference ``fit``: shuffle + epoch loop; returns epoch losses."""
    out = []
    user_ids = user_ids.astype(np.int64)
    item_ids = item_ids.astype(np.int64)
    for _ in range(n_iter):
        order = np.arange(len(user_ids))
        random_state.shuffle(order)
        losses = fit_steps(net, optimizer, user_ids[order], item_ids[order], num_items,
                           batch_size, loss, random_state, n_neg)
        out.append(sum(losses) / len(losses))
    return out
