"""Generate the explicit-feedback Bloom-layer golden vectors from the LIVE reference (build container only).

Run:  SPOTLIGHT_REFERENCE=<reference checkout> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_explicit_bloom.py

A standalone companion of make_golden_explicit.py (whose helpers it uses): it writes only the
fixtures below, so the existing fixtures are not regenerated.  The reference's ``BloomEmbedding``
hashes with scikit-learn's ``murmurhash3_32``.

* ``explicit_bloom_<loss>.npz``: one minibatch of the reference's ``ExplicitFactorizationModel``
  fit loop body (spotlight/factorization/explicit.py:223-234) on a ``BilinearNet`` whose user
  layer is a ``ScaledEmbedding`` and whose item layer is a ``BloomEmbedding(H = 3, padding_idx =
  0)``; ``explicit_bloom_both_regression.npz`` hashes both sides.  Each holds the state_dict, the
  minibatch (repeated users and items, the padding id 0 on both sides), the ratings, the
  predictions handed to the loss, the loss and every parameter's ``.grad``.
* ``fit_explicit_bloom_{sgd,adagrad}.npz``: two epochs of ``fit()`` (the last batch short) with
  a Bloom item layer under ``torch.optim.SGD`` / ``Adagrad`` without weight decay: initial and
  final state_dict, the RandomState key and position after the constructor and after fit, the
  epoch losses, ``predict`` for one user and ``rmse_score`` on a held-out set.
"""

import contextlib
import io
import os
import sys
import warnings

import numpy as np

sys.dont_write_bytecode = True
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import make_golden as mg  # noqa: E402
import make_golden_explicit as mge  # noqa: E402
import torch  # noqa: E402

from spotlight.evaluation import rmse_score  # noqa: E402
from spotlight.factorization.explicit import ExplicitFactorizationModel  # noqa: E402
from spotlight.factorization.representations import BilinearNet  # noqa: E402
from spotlight.interactions import Interactions  # noqa: E402
from spotlight.layers import BloomEmbedding, ScaledEmbedding  # noqa: E402

warnings.filterwarnings('ignore', message='size_average')

H, RATIO = 3, 0.5


def _net(num_users, num_items, dim, user_H, item_H, seed):
    torch.manual_seed(seed)
    user = (BloomEmbedding(num_users, dim, compression_ratio=RATIO, num_hash_functions=user_H) if user_H
            else ScaledEmbedding(num_users, dim))
    item = BloomEmbedding(num_items, dim, compression_ratio=RATIO, num_hash_functions=item_H)
    net = BilinearNet(num_users, num_items, dim, user_embedding_layer=user, item_embedding_layer=item)
    with torch.no_grad():   # zero-init biases would hide bias-gather bugs
        net.user_biases.weight.normal_(0, 0.1)
        net.item_biases.weight.normal_(0, 0.1)
    return net


def step_case(name, loss, user_H=0, num_users=23, num_items=31, dim=8, batch=40, seed=21):
    rs = np.random.RandomState(seed)
    users = rs.randint(0, num_users, batch).astype(np.int64)
    items = rs.randint(0, num_items, batch).astype(np.int64)
    users[:4] = [0, num_users - 1, users[5], users[5]]
    items[:4] = [0, num_items - 1, items[6], items[6]]
    ratings = mge._ratings(loss, rs, batch)
    inter = Interactions(users.astype(np.int32), items.astype(np.int32), ratings=ratings,
                         num_users=num_users, num_items=num_items)
    net = _net(num_users, num_items, dim, user_H, H, seed)
    model = ExplicitFactorizationModel(loss=loss, embedding_dim=dim, batch_size=batch, representation=net,
                                       random_state=np.random.RandomState(seed + 1))
    model._initialize(inter)
    out = dict(mg._state(net))
    # replay of the reference loop body, explicit.py:223-234
    predictions = net(torch.from_numpy(users), torch.from_numpy(items))
    if loss == 'poisson':
        predictions = torch.exp(predictions)
    model._optimizer.zero_grad()
    lv = model._loss_func(torch.from_numpy(ratings), predictions)
    lv.backward()
    out.update(mg._grads(net))
    out.update(users=users, items=items, ratings=ratings, pred=mg._np(predictions),
               loss=np.float32(lv.item()), loss_kind=np.array(loss), num_users=np.int64(num_users),
               num_items=np.int64(num_items), dim=np.int64(dim), user_H=np.int64(user_H), item_H=np.int64(H),
               bloom_ratio=np.float64(RATIO))
    np.savez_compressed(os.path.join(mg.HERE, name + '.npz'), **out)
    print(name, 'loss', lv.item())


def fit_case(name, loss, optimizer, num_users=40, num_items=300, dim=16, n_inter=1000, batch=128, seed=31):
    rs = np.random.RandomState(seed)
    users = rs.randint(0, num_users, n_inter).astype(np.int32)
    items = rs.randint(0, num_items, n_inter).astype(np.int32)
    ratings = mge._ratings(loss, rs, n_inter)
    inter = Interactions(users, items, ratings=ratings, num_users=num_users, num_items=num_items)
    lr = 0.05 if optimizer == 'sgd' else 0.1
    opt = (lambda p: torch.optim.SGD(p, lr=lr)) if optimizer == 'sgd' else \
        (lambda p: torch.optim.Adagrad(p, lr=lr))
    net = _net(num_users, num_items, dim, 0, H, seed)
    model = ExplicitFactorizationModel(loss=loss, embedding_dim=dim, batch_size=batch, n_iter=2,
                                       optimizer_func=opt, representation=net,
                                       random_state=np.random.RandomState(seed + 1))
    model._initialize(inter)
    out = {('init.' + k): mg._np(v) for k, v in model._net.state_dict().items()}
    st = model._random_state.get_state()
    out.update(rs0_key=st[1].copy(), rs0_pos=np.int64(st[2]))
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        model.fit(inter, verbose=True)
    losses = [float(line.split('loss')[1]) for line in buf.getvalue().strip().split('\n')]
    out.update({('final.' + k): mg._np(v) for k, v in model._net.state_dict().items()})
    out.update(mg._rs_state(model._random_state))
    test_u = rs.randint(0, num_users, 97).astype(np.int32)
    test_i = rs.randint(0, num_items, 97).astype(np.int32)
    test = Interactions(test_u, test_i, ratings=mge._ratings(loss, rs, 97), num_users=num_users,
                        num_items=num_items)
    out.update(users=users, items=items, ratings=ratings, epoch_losses=np.array(losses), loss_kind=np.array(loss),
               num_users=np.int64(num_users), num_items=np.int64(num_items), dim=np.int64(dim),
               batch=np.int64(batch), n_iter=np.int64(2), lr=np.float64(lr), optimizer=np.array(optimizer),
               bloom_H=np.int64(H), bloom_ratio=np.float64(RATIO),
               predict_user=np.int64(3), predict=model.predict(3).astype(np.float32),
               test_users=test_u, test_items=test_i, test_ratings=test.ratings,
               rmse=np.float32(rmse_score(model, test)))
    np.savez_compressed(os.path.join(mg.HERE, name + '.npz'), **out)
    print(name, 'epoch losses', losses, 'rmse', out['rmse'])


if __name__ == '__main__':
    for loss in ('regression', 'poisson', 'logistic'):
        step_case('explicit_bloom_' + loss, loss)
    step_case('explicit_bloom_both_regression', 'regression', user_H=2, seed=22)
    fit_case('fit_explicit_bloom_sgd', 'regression', 'sgd')
    fit_case('fit_explicit_bloom_adagrad', 'poisson', 'adagrad')
