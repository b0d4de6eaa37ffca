"""Whole training steps on the generic autograd route, through the public model classes, against
the float64 oracles: the route every model takes outside the fused envelope (``embedding_dim``
not a multiple of 4, ``sparse=True``, padding rows, custom representations).

Each test first asserts ``model._route() == 'generic'``, so that a routing change cannot turn it
into a test of a fused step.  Steps run one minibatch at a time; after each, every parameter's
gradient is held at 1e-5 of the oracle's (evaluated at the weights the step started from) and the
SGD update at 1e-6 of the weights.
"""

import types

import numpy as np
import pytest
import torch

from conftest import assert_close
from oracle import explicit as oex
from oracle import mf as omf
from oracle import seq as oseq

pytestmark = pytest.mark.gpu

STEPS, B = 3, 64


def host(x):
    return x.detach().cpu().numpy().astype(np.float64)


def dense_grad(p):
    g = p.grad
    if g.is_sparse:
        g = g.coalesce().to_dense()
    return host(g)


def randomize(params, seed, zero_rows=()):
    torch.manual_seed(seed)
    with torch.no_grad():
        for p in params:
            p.copy_(torch.randn_like(p) * 0.5)
        for p, row in zero_rows:
            p[row].zero_()


def check_step(params, before, grads, lr, what):
    """Gradients at 1e-5 of the oracle's and w' = w - lr g at 1e-6 of the weights.  A gradient
    that is an exact 0 (bpr's user-bias pair gp + gn) is float32 rounding noise on either side:
    every table also gets an absolute 1e-6 of the step's largest gradient."""
    gmax = max(np.abs(g).max() for g in grads)
    for p, w0, g, nm in zip(params, before, grads, what):
        assert_close(dense_grad(p), g.reshape(w0.shape), 1e-5, atol=1e-6 * gmax, what='grad ' + nm)
        assert_close(host(p), w0 - lr * g.reshape(w0.shape), 1e-6, what='weights ' + nm)


def _implicit(loss, D, sparse, representation=None, U=50, I=60):
    from spotlight_b200.factorization.implicit import ImplicitFactorizationModel
    from spotlight_b200.interactions import Interactions
    rs = np.random.RandomState(D)
    n = STEPS * B
    users = rs.randint(0, U, n).astype(np.int64)
    items = rs.randint(0, I, n).astype(np.int64)
    if representation is not None:
        users[::7] = 3                              # the padding user in every minibatch
    lr = 0.2
    model = ImplicitFactorizationModel(loss=loss, embedding_dim=D, batch_size=B, n_iter=1, sparse=sparse,
                                       representation=representation, num_negative_samples=3,
                                       optimizer_func=lambda p: torch.optim.SGD(p, lr=lr), use_cuda=True,
                                       random_state=np.random.RandomState(11))
    model._initialize(Interactions(users.astype(np.int32), items.astype(np.int32), num_users=U, num_items=I))
    assert model._route() == 'generic'
    return model, users, items, lr


def _run_implicit(model, users, items, lr, loss, pad_user=None):
    net = model._net
    params = (net.user_embeddings.weight, net.item_embeddings.weight, net.user_biases.weight,
              net.item_biases.weight)
    randomize(params, 5, [(params[0], pad_user)] if pad_user is not None else ())
    n_neg, I = model._n_neg(), model._num_items
    # the negatives of the three steps, from the model's own RandomState
    model._random_state = np.random.RandomState(77)
    negs_dev = model._epoch_negatives(len(users))
    negs = np.random.RandomState(77).randint(0, I, len(users) * n_neg, dtype=np.int64)
    assert np.array_equal(negs_dev.cpu().numpy(), negs)
    ud, idv = torch.from_numpy(users).cuda(), torch.from_numpy(items).cuda()
    for s in range(STEPS):
        sl, nsl = slice(s * B, (s + 1) * B), slice(s * B * n_neg, (s + 1) * B * n_neg)
        before = [host(p) for p in params]
        got_loss = model._fit_epoch_autograd(ud[sl], idv[sl], negs_dev[nsl], 'generic')
        ref = omf.mf_step(*before, users[sl], items[sl], negs[nsl], loss, n_neg, np.float64)
        if pad_user is not None:
            ref['dWu'][pad_user] = 0.0
        assert_close(got_loss, float(ref['loss']), 1e-5, what='loss step %d' % s)
        check_step(params, before, [ref[k] for k in ('dWu', 'dWi', 'dbu', 'dbi')], lr, ('Wu', 'Wi', 'bu', 'bi'))
        if pad_user is not None:
            assert (host(params[0])[pad_user] == 0).all(), 'the padding row moved'
    return params


@pytest.mark.parametrize('sparse', [False, True], ids=['dense', 'sparse'])
@pytest.mark.parametrize('loss', ['pointwise', 'bpr', 'hinge', 'adaptive_hinge'])
@pytest.mark.parametrize('D', [6, 10])
def test_implicit_generic_steps(D, loss, sparse):
    """embedding_dim % 4 != 0 (scalar lookups at D and D = 1 for the biases), SGD; with
    ``sparse=True`` the COO gradient of every table, coalesced, is the dense float64 one."""
    model, users, items, lr = _implicit(loss, D, sparse)
    params = _run_implicit(model, users, items, lr, loss)
    if sparse:
        assert all(p.grad.is_sparse for p in params)


@pytest.mark.parametrize('loss', ['bpr', 'adaptive_hinge'])
def test_padding_user_layer(loss):
    """BilinearNet with a ScaledEmbedding(padding_idx=3) user layer (D = 8): the padding user is
    in every minibatch, its row gets no gradient and stays zero; its bias trains."""
    from spotlight_b200.factorization.representations import BilinearNet
    from spotlight_b200.layers import ScaledEmbedding
    rep = BilinearNet(50, 60, 8, user_embedding_layer=ScaledEmbedding(50, 8, padding_idx=3))
    model, users, items, lr = _implicit(loss, 8, False, representation=rep)
    params = _run_implicit(model, users, items, lr, loss, pad_user=3)
    assert (host(params[2])[3] != 0).all()


@pytest.mark.parametrize('loss', ['regression', 'poisson', 'logistic'])
def test_explicit_generic_steps(loss):
    from spotlight_b200.factorization.explicit import ExplicitFactorizationModel
    from spotlight_b200.interactions import Interactions
    U, I, D = 40, 70, 10
    rs = np.random.RandomState(21)
    n = STEPS * B
    users = rs.randint(0, U, n).astype(np.int64)
    items = rs.randint(0, I, n).astype(np.int64)
    ratings = (rs.choice([-1.0, 1.0], n) if loss == 'logistic' else rs.randint(0, 6, n)).astype(np.float32)
    lr = 0.1
    model = ExplicitFactorizationModel(loss=loss, embedding_dim=D, batch_size=B, n_iter=1,
                                       optimizer_func=lambda p: torch.optim.SGD(p, lr=lr), use_cuda=True,
                                       random_state=np.random.RandomState(3))
    model._initialize(Interactions(users.astype(np.int32), items.astype(np.int32), ratings=ratings,
                                   num_users=U, num_items=I))
    assert model._route() == 'generic'
    net = model._net
    params = (net.user_embeddings.weight, net.item_embeddings.weight, net.user_biases.weight,
              net.item_biases.weight)
    randomize(params, 6)
    ud, idv, rd = (torch.from_numpy(x).cuda() for x in (users, items, ratings))
    for s in range(STEPS):
        sl = slice(s * B, (s + 1) * B)
        before = [host(p) for p in params]
        got_loss = model._fit_epoch_autograd(ud[sl], idv[sl], rd[sl], 'generic')
        ref = oex.explicit_step(*before, users[sl], items[sl], ratings[sl], loss)
        assert_close(got_loss, ref['loss'], 1e-5, what='loss step %d' % s)
        check_step(params, before, [ref[k] for k in ('dWu', 'dWi', 'dbu', 'dbi')], lr, ('Wu', 'Wi', 'bu', 'bi'))


@pytest.mark.parametrize('loss', ['pointwise', 'bpr', 'hinge', 'adaptive_hinge'])
def test_pool_generic_steps(loss):
    """PoolNet at D = 6 (not fusable): the padding id 0 in the sequences, the padding row of the
    item table and of the item bias frozen at zero."""
    from spotlight_b200.sequence.implicit import ImplicitSequenceModel
    I, D, S = 80, 6, 7
    rs = np.random.RandomState(31)
    seqs = rs.randint(1, I, (STEPS * B, S)).astype(np.int64)
    seqs[rs.rand(*seqs.shape) < 0.25] = 0
    seqs[:, 0] = 0
    n_neg = 3 if loss == 'adaptive_hinge' else 1
    negs = rs.randint(0, I, (STEPS * B * n_neg, S)).astype(np.int64)
    lr = 0.3
    model = ImplicitSequenceModel(loss=loss, representation='pooling', embedding_dim=D, batch_size=B,
                                  num_negative_samples=n_neg, optimizer_func=lambda p: torch.optim.SGD(p, lr=lr),
                                  use_cuda=True, random_state=np.random.RandomState(4))
    model._initialize(types.SimpleNamespace(num_items=I))
    assert model._route() == 'generic'
    net = model._net
    params = (net.item_embeddings.weight, net.item_biases.weight)
    randomize(params, 7, [(params[0], 0), (params[1], 0)])
    for s in range(STEPS):
        batch = torch.from_numpy(seqs[s * B:(s + 1) * B]).cuda()
        # adaptive negatives: rows k * B + b of the step's (n * B, S) block
        bneg = negs[s * B * n_neg:(s + 1) * B * n_neg]
        before = [host(p) for p in params]
        model._optimizer.zero_grad()
        lval = model._generic_step(batch, torch.from_numpy(bneg).cuda(), n_neg)
        lval.backward()
        model._optimizer.step()
        ref = oseq.pool_step(before[0], before[1], seqs[s * B:(s + 1) * B], bneg, loss, n_neg, np.float64)
        assert_close(lval.item(), float(ref['loss']), 1e-5, what='loss step %d' % s)
        check_step(params, before, [ref['dE'], ref['dbias']], lr, ('E', 'bias'))
        assert (host(params[0])[0] == 0).all() and host(params[1])[0, 0] == 0, 'the padding row moved'
