"""Generate the explicit-feedback golden vectors from the LIVE reference (build container only).

Run:  SPOTLIGHT_REFERENCE=<reference checkout> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_explicit.py

A standalone companion of make_golden.py (whose helpers it uses): it writes only the six
explicit-feedback fixtures, so the existing fixtures are not regenerated.

* ``explicit_<loss>.npz``: one minibatch of the reference's ``ExplicitFactorizationModel`` fit
  loop body (spotlight/factorization/explicit.py:223-234) -- state_dict, the minibatch (with
  repeated users and items), ratings, the predictions handed to the loss, the loss and every
  parameter's ``.grad``.
* ``fit_explicit_<loss>.npz``: a small ``fit()`` -- epoch losses, initial and final state_dict,
  the ``RandomState`` position afterwards, ``predict`` and ``rmse_score`` outputs.
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
import torch  # noqa: E402

from spotlight.evaluation import rmse_score  # noqa: E402
from spotlight.factorization.explicit import ExplicitFactorizationModel  # noqa: E402
from spotlight.interactions import Interactions  # noqa: E402

warnings.filterwarnings('ignore', message='size_average')


def _ratings(loss, rs, n):
    if loss == 'regression':
        return rs.randint(1, 6, n).astype(np.float32)
    if loss == 'poisson':
        return rs.randint(0, 4, n).astype(np.float32)
    return rs.choice(np.array([-1.0, 0.0, 1.0], dtype=np.float32), n)


def step_case(name, loss, num_users=23, num_items=31, dim=8, batch=40, seed=21):
    rs = np.random.RandomState(seed)
    users = rs.randint(0, num_users, batch).astype(np.int64)
    items = rs.randint(0, num_items, batch).astype(np.int64)
    users[:4] = [0, num_users - 1, users[5], users[5]]
    items[:4] = [0, num_items - 1, items[6], items[6]]
    ratings = _ratings(loss, rs, batch)
    inter = Interactions(users.astype(np.int32), items.astype(np.int32), ratings=ratings,
                         num_users=num_users, num_items=num_items)
    model = ExplicitFactorizationModel(loss=loss, embedding_dim=dim, batch_size=batch,
                                       random_state=np.random.RandomState(seed + 1))
    model._initialize(inter)
    net = model._net
    with torch.no_grad():   # zero-init biases would hide bias-gather bugs
        g = torch.Generator().manual_seed(seed)
        net.user_biases.weight.copy_(torch.randn(net.user_biases.weight.shape, generator=g) * 0.1)
        net.item_biases.weight.copy_(torch.randn(net.item_biases.weight.shape, generator=g) * 0.1)
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
               loss=np.float32(lv.item()), num_users=np.int64(num_users),
               num_items=np.int64(num_items), dim=np.int64(dim))
    np.savez_compressed(os.path.join(mg.HERE, name + '.npz'), **out)
    print(name, 'loss', lv.item())


def fit_case(name, loss, optimizer, l2=0.0, num_users=30, num_items=40, dim=8, n_inter=500, batch=64,
             n_iter=3, seed=9):
    rs = np.random.RandomState(seed)
    users = rs.randint(0, num_users, n_inter).astype(np.int32)
    items = rs.randint(0, num_items, n_inter).astype(np.int32)
    ratings = _ratings(loss, rs, n_inter)
    inter = Interactions(users, items, ratings=ratings, num_users=num_users, num_items=num_items)
    if optimizer == 'sgd':
        opt = lambda p: torch.optim.SGD(p, lr=0.05)           # noqa: E731
        lr = 0.05
    elif optimizer == 'adagrad':
        opt = lambda p: torch.optim.Adagrad(p, lr=0.1)        # noqa: E731
        lr = 0.1
    else:
        opt, lr = None, 1e-2
    model = ExplicitFactorizationModel(loss=loss, embedding_dim=dim, batch_size=batch, n_iter=n_iter,
                                       l2=l2, learning_rate=lr, optimizer_func=opt,
                                       random_state=np.random.RandomState(seed))
    model._initialize(inter)
    out = {('init.' + k): mg._np(v) for k, v in model._net.state_dict().items()}
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        model.fit(inter, verbose=True)
    losses = [float(line.split('loss')[1]) for line in buf.getvalue().strip().split('\n')]
    out.update({('final.' + k): mg._np(v) for k, v in model._net.state_dict().items()})
    out.update(mg._rs_state(model._random_state))
    test_u = rs.randint(0, num_users, 97).astype(np.int32)
    test_i = rs.randint(0, num_items, 97).astype(np.int32)
    test = Interactions(test_u, test_i, ratings=_ratings(loss, rs, 97), num_users=num_users,
                        num_items=num_items)
    out.update(users=users, items=items, ratings=ratings, epoch_losses=np.array(losses),
               num_users=np.int64(num_users), num_items=np.int64(num_items), dim=np.int64(dim),
               batch=np.int64(batch), n_iter=np.int64(n_iter), seed=np.int64(seed), lr=np.float64(lr),
               l2=np.float64(l2), optimizer=np.array(optimizer),
               predict_user3=model.predict(3), predict_pairs=model.predict(test_u, test_i),
               test_users=test_u, test_items=test_i, test_ratings=test.ratings,
               rmse=np.float32(rmse_score(model, test)))
    np.savez_compressed(os.path.join(mg.HERE, name + '.npz'), **out)
    print(name, 'epoch losses', losses, 'rmse', out['rmse'])


if __name__ == '__main__':
    for loss in ('regression', 'poisson', 'logistic'):
        step_case('explicit_' + loss, loss)
    fit_case('fit_explicit_regression', 'regression', 'adam', l2=1e-3)
    fit_case('fit_explicit_poisson', 'poisson', 'sgd')
    fit_case('fit_explicit_logistic', 'logistic', 'adagrad')
