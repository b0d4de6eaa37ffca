"""Explicit-feedback matrix factorization on the device: the fused rating step against the
float64 oracle (oracle/explicit.py) on every route, the live reference's fixtures
(tests/golden/explicit_*.npz, fit_explicit_*.npz), determinism, the configs[1] shape, the generic
route, prediction, ``rmse_score`` and the model's error behaviour.  Loss, scores and gradients
are held to 1e-5 of the tensor's max."""

import copy

import numpy as np
import pytest
import torch

from conftest import assert_close, load_golden
from oracle import explicit as oex

pytestmark = pytest.mark.gpu

LOSSES = ('regression', 'poisson', 'logistic')
DIMS = (4, 8, 12, 16, 32, 64, 100, 128, 256)


def _ratings(loss, rs, n):
    if loss == 'regression':
        return rs.randint(1, 6, n).astype(np.float32)
    if loss == 'poisson':
        return rs.randint(0, 4, n).astype(np.float32)
    return rs.choice(np.array([-1.0, 0.0, 1.0, 0.25], dtype=np.float32), n)


def _case(loss, U, I, D, B, seed, zipf=False):
    rs = np.random.RandomState(seed)
    Wu = (rs.randn(U, D) / np.sqrt(D)).astype(np.float32)
    Wi = (rs.randn(I, D) / np.sqrt(D)).astype(np.float32)
    bu = (rs.randn(U, 1) * 0.1).astype(np.float32)
    bi = (rs.randn(I, 1) * 0.1).astype(np.float32)
    if zipf:
        users = np.minimum(rs.zipf(1.6, B) - 1, U - 1).astype(np.int64)
        items = np.minimum(rs.zipf(1.4, B) - 1, I - 1).astype(np.int64)
    else:
        users = rs.randint(0, U, B).astype(np.int64)
        items = rs.randint(0, I, B).astype(np.int64)
        users[:4] = [0, U - 1, users[5], users[5]]
        items[:4] = [0, I - 1, items[6], items[6]]
    return dict(Wu=Wu, Wi=Wi, bu=bu, bi=bi, users=users, items=items, ratings=_ratings(loss, rs, B))


def _dev(c):
    return {k: torch.from_numpy(v).cuda() for k, v in c.items()}


def _dense_step(c, loss):
    from spotlight_b200 import _lib, ops
    t = _dev(c)
    return ops.mf_rating_train_step(t['Wu'], t['Wi'], t['bu'], t['bi'], t['users'], t['items'], t['ratings'],
                                    _lib.LOSS_KIND[loss], True)


def _check_dense(out, ref):
    assert_close(out[0].item(), ref['loss'], 1e-5, what='loss')
    assert_close(out[1].cpu().numpy(), ref['scores'], 1e-5, what='scores')
    for k, v in zip(('dWu', 'dWi', 'dbu', 'dbi'), out[2:]):
        assert_close(v.cpu().numpy(), ref[k], 1e-5, what=k)


@pytest.mark.parametrize('loss', LOSSES)
@pytest.mark.parametrize('D', DIMS)
def test_dense_step_matches_oracle(loss, D):
    c = _case(loss, 57, 83, D, 700, seed=D)
    ref = oex.explicit_step(c['Wu'], c['Wi'], c['bu'], c['bi'], c['users'], c['items'], c['ratings'], loss)
    _check_dense(_dense_step(c, loss), ref)


@pytest.mark.parametrize('loss', LOSSES)
def test_dense_step_large_batch_tiles(loss):
    """B above the small-batch threshold: 32-interaction tiles."""
    c = _case(loss, 20000, 5000, 64, 200000, seed=5)
    ref = oex.explicit_step(c['Wu'], c['Wi'], c['bu'], c['bi'], c['users'], c['items'], c['ratings'], loss)
    _check_dense(_dense_step(c, loss), ref)


PLANNED_DIMS = (8, 16, 32, 64, 128)      # the planned two-kernel step's one-term mode


def _inplace(c, loss, opt, lr, wd, states, planned=True):
    from spotlight_b200 import ops
    t = _dev(c)
    p = [t['Wu'], t['Wi'], t['bu'], t['bi']]
    st = [torch.from_numpy(s).cuda() for s in states] if states is not None else None
    l = ops.mf_train_step_inplace(*p, t['users'], t['items'], None, loss, opt, lr, st, wd, 1e-10,
                                  planned=planned, ratings=t['ratings'])
    return l.item(), [x.cpu().numpy() for x in p], ([x.cpu().numpy() for x in st] if st else None)


@pytest.mark.parametrize('loss', LOSSES)
@pytest.mark.parametrize('D', DIMS)
@pytest.mark.parametrize('opt,wd', [('sgd', 0.0), ('sgd', 0.05), ('adagrad', 0.0), ('adagrad', 0.05)])
@pytest.mark.parametrize('planned', [True, False])
def test_compact_fused_step_matches_oracle(loss, D, opt, wd, planned):
    """planned=True runs the planned two-kernel step at D in PLANNED_DIMS (first-generation
    compact kernels elsewhere); planned=False always the first-generation compact kernels."""
    from spotlight_b200 import _lib
    if not planned and D not in PLANNED_DIMS:
        pytest.skip('same kernels as planned=True at this D')
    c = _case(loss, 57, 83, D, 700, seed=3 * D)
    lr = 0.3
    states = [np.full_like(x, 0.01) for x in (c['Wu'], c['Wi'], c['bu'], c['bi'])] if opt == 'adagrad' else None
    kind = _lib.OPT_SGD if opt == 'sgd' else _lib.OPT_ADAGRAD
    l, params, st = _inplace(c, loss, kind, lr, wd, states, planned)
    ref_params = [x.astype(np.float64).copy() for x in (c['Wu'], c['Wi'], c['bu'], c['bi'])]
    ref_states = [s.astype(np.float64).copy() for s in states] if states else None
    ref = oex.fused_step(ref_params, c['users'], c['items'], c['ratings'], loss, opt, lr, wd, 1e-10, ref_states)
    assert_close(l, ref['loss'], 1e-5, what='loss')
    # compare the update (new - old): the parameters themselves would hide a wrong step
    for k, (a, e, w0) in enumerate(zip(params, ref_params, (c['Wu'], c['Wi'], c['bu'], c['bi']))):
        assert_close(a - w0, e - w0, 1e-5, atol=2e-7, what='delta %d' % k)
    if st:
        for k, (a, e) in enumerate(zip(st, ref_states)):
            assert_close(a, e, 1e-5, what='state %d' % k)


@pytest.mark.parametrize('loss', LOSSES)
def test_reference_step_fixture(loss):
    g = load_golden('explicit_' + loss)
    c = dict(Wu=g['sd.user_embeddings.weight'], Wi=g['sd.item_embeddings.weight'], bu=g['sd.user_biases.weight'],
             bi=g['sd.item_biases.weight'], users=g['users'], items=g['items'], ratings=g['ratings'])
    out = _dense_step(c, loss)
    assert_close(out[0].item(), g['loss'], 1e-5, what='loss')
    pred = out[1].cpu().numpy()
    assert_close(np.exp(pred) if loss == 'poisson' else pred, g['pred'], 1e-5, what='pred')
    for v, n in zip(out[2:], ('user_embeddings', 'item_embeddings', 'user_biases', 'item_biases')):
        assert_close(v.cpu().numpy(), g['grad.%s.weight' % n], 1e-5, what=n)


def _model(g, loss, optimizer_func, l2=0.0, lr=1e-2):
    from spotlight_b200.factorization.explicit import ExplicitFactorizationModel
    from spotlight_b200.interactions import Interactions
    inter = Interactions(g['users'], g['items'], ratings=g['ratings'], num_users=int(g['num_users']),
                         num_items=int(g['num_items']))
    model = ExplicitFactorizationModel(loss=loss, embedding_dim=int(g['dim']), batch_size=int(g['batch']),
                                       n_iter=int(g['n_iter']), l2=l2, learning_rate=lr,
                                       optimizer_func=optimizer_func, use_cuda=True,
                                       random_state=np.random.RandomState(int(g['seed'])))
    model._initialize(inter)
    model._net.load_state_dict({k[5:]: torch.from_numpy(v) for k, v in g.items() if k.startswith('init.')})
    return model, inter


def _fit_and_check(model, inter, g, loss, capsys, rtol):
    from spotlight_b200.evaluation import rmse_score
    from spotlight_b200.interactions import Interactions
    model.fit(inter, verbose=True)
    lines = [l for l in capsys.readouterr().out.strip().split('\n') if l.startswith('Epoch')]
    assert_close(np.array([float(l.split('loss')[1]) for l in lines]), g['epoch_losses'], 1e-5, what='losses')
    for k, v in model._net.state_dict().items():
        assert_close(v.cpu().numpy(), g['final.' + k], rtol, atol=1e-7, what=k)
    st = model._random_state.get_state()
    assert (st[1] == g['rs_key']).all() and st[2] == int(g['rs_pos'])
    assert_close(model.predict(3), g['predict_user3'], rtol, what='predict_user3')
    assert_close(model.predict(g['test_users'], g['test_items']), g['predict_pairs'], rtol, what='predict')
    test = Interactions(g['test_users'], g['test_items'], ratings=g['test_ratings'],
                        num_users=int(g['num_users']), num_items=int(g['num_items']))
    r = rmse_score(model, test)
    assert isinstance(r, np.float32)
    assert_close(r, g['rmse'], rtol, what='rmse')


@pytest.mark.parametrize('route', ['fused', 'epoch'])
def test_fit_poisson_sgd(route, capsys):
    from spotlight_b200 import optim
    g = load_golden('fit_explicit_poisson')
    func = optim.fused_sgd(lr=0.05) if route == 'epoch' else (lambda p: torch.optim.SGD(p, lr=0.05))
    model, inter = _model(g, 'poisson', func)
    assert model._route() == route
    _fit_and_check(model, inter, g, 'poisson', capsys, 1e-5)


@pytest.mark.parametrize('route', ['fused', 'epoch'])
def test_fit_logistic_adagrad(route, capsys):
    from spotlight_b200 import optim
    g = load_golden('fit_explicit_logistic')
    func = optim.fused_adagrad(lr=0.1) if route == 'epoch' else (lambda p: torch.optim.Adagrad(p, lr=0.1))
    model, inter = _model(g, 'logistic', func)
    assert model._route() == route
    # adagrad divides by sqrt(sum g^2): first-touch amplification (as test_model_gpu)
    _fit_and_check(model, inter, g, 'logistic', capsys, 1e-3)


@pytest.mark.parametrize('route', ['epoch', 'fused'])
def test_fit_regression_default_adam(route, capsys):
    """The default-constructed model (lazy-exact FusedAdam on the epoch pipeline) and stock
    torch.optim.Adam on the fused op, both against the reference's default-Adam trajectory."""
    from spotlight_b200.optim import FusedAdam
    g = load_golden('fit_explicit_regression')
    l2 = float(g['l2'])
    func = None if route == 'epoch' else (lambda p: torch.optim.Adam(p, lr=1e-2, weight_decay=l2))
    model, inter = _model(g, 'regression', func, l2=l2)
    assert isinstance(model._optimizer, FusedAdam) == (route == 'epoch')
    assert model._route() == route
    _fit_and_check(model, inter, g, 'regression', capsys, 2e-3)   # Adam: sign-level sensitivity


@pytest.mark.parametrize('loss', LOSSES)
def test_repeated_steps_bit_identical_with_hot_rows(loss):
    """Zipf-drawn batch: one item with > 128 members and a hot user (the long-segment kernels)."""
    c = _case(loss, 3000, 2000, 64, 20000, seed=17, zipf=True)
    assert np.bincount(c['items']).max() > 128 and np.bincount(c['users']).max() > 128
    a, b = _dense_step(c, loss), _dense_step(c, loss)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    ref = oex.explicit_step(c['Wu'], c['Wi'], c['bu'], c['bi'], c['users'], c['items'], c['ratings'], loss)
    _check_dense(a, ref)


@pytest.mark.parametrize('opt', ['sgd', 'adagrad'])
def test_epoch_equals_step_by_step(opt):
    """One slb_mf_fit_epoch call (the model's epoch route) equals per-step launches."""
    from spotlight_b200 import _lib, ops, optim
    from spotlight_b200.factorization.explicit import ExplicitFactorizationModel
    from spotlight_b200.interactions import Interactions
    rs = np.random.RandomState(2)
    U, I, n, B = 300, 200, 5000, 256
    inter = Interactions(rs.randint(0, U, n).astype(np.int32), rs.randint(0, I, n).astype(np.int32),
                         ratings=_ratings('regression', rs, n), num_users=U, num_items=I)
    func = optim.fused_sgd(lr=0.01) if opt == 'sgd' else optim.fused_adagrad(lr=0.05)
    model = ExplicitFactorizationModel(loss='regression', embedding_dim=32, n_iter=1, batch_size=B,
                                       optimizer_func=func, use_cuda=True, random_state=np.random.RandomState(4))
    model._initialize(inter)
    net = model._net
    params = [x.detach().clone() for x in (net.user_embeddings.weight, net.item_embeddings.weight,
                                           net.user_biases.weight, net.item_biases.weight)]
    states = [torch.zeros_like(p) for p in params] if opt == 'adagrad' else None
    rs_copy = np.random.RandomState()
    rs_copy.set_state(model._random_state.get_state())
    model.fit(inter)
    order = np.arange(n)
    rs_copy.shuffle(order)
    u = torch.from_numpy(inter.user_ids[order].astype(np.int64)).cuda()
    i = torch.from_numpy(inter.item_ids[order].astype(np.int64)).cuda()
    r = torch.from_numpy(inter.ratings[order]).cuda()
    kind = _lib.OPT_SGD if opt == 'sgd' else _lib.OPT_ADAGRAD
    lr = 0.01 if opt == 'sgd' else 0.05
    for lo in range(0, n, B):
        ops.mf_train_step_inplace(*params, u[lo:lo + B], i[lo:lo + B], None, 'regression', kind, lr, states,
                                  ratings=r[lo:lo + B])
    for a, b in zip(params, (net.user_embeddings.weight, net.item_embeddings.weight,
                             net.user_biases.weight, net.item_biases.weight)):
        assert torch.equal(a, b.detach())


@pytest.mark.parametrize('loss', LOSSES)
@pytest.mark.parametrize('D', PLANNED_DIMS)
@pytest.mark.parametrize('opt', ['sgd', 'adagrad'])
def test_planned_step_equals_first_generation_on_hot_rows(loss, D, opt):
    """Zipf-drawn batch with a hot item and a hot user (> 128 members: the hot-row sort and
    the *_long kernels): the planned step and the first-generation compact step give the same
    update, and the planned step's parameters and loss are bit-reproducible."""
    from spotlight_b200 import _lib
    c = _case(loss, 3000, 2000, D, 20000, seed=D + 1, zipf=True)
    assert np.bincount(c['items']).max() > 128 and np.bincount(c['users']).max() > 128
    kind = _lib.OPT_SGD if opt == 'sgd' else _lib.OPT_ADAGRAD
    states = [np.full_like(x, 0.01) for x in (c['Wu'], c['Wi'], c['bu'], c['bi'])] if opt == 'adagrad' else None
    lp, pp, sp = _inplace(c, loss, kind, 0.3, 0.01, states, planned=True)
    lp2, pp2, _ = _inplace(c, loss, kind, 0.3, 0.01, states, planned=True)
    lf, pf, sf = _inplace(c, loss, kind, 0.3, 0.01, states, planned=False)
    assert all(np.array_equal(a, b) for a, b in zip(pp, pp2))
    assert lp2 == lp, ('repeated loss', lp2, lp)
    assert_close(lp, lf, 1e-5, what='loss')
    for k, (a, b, w0) in enumerate(zip(pp, pf, (c['Wu'], c['Wi'], c['bu'], c['bi']))):
        assert_close(a - w0, b - w0, 1e-5, atol=2e-7, what='delta %d' % k)
    if sp:
        for k, (a, b) in enumerate(zip(sp, sf)):
            assert_close(a, b, 1e-5, what='state %d' % k)


@pytest.mark.parametrize('loss', LOSSES)
@pytest.mark.parametrize('D', DIMS)
def test_lazy_adam_equals_dense_adam(loss, D):
    """The default-constructed model (row-wise lazy-exact Adam on the first-generation compact
    step, whose pre-pass reads no negatives here) against stock torch.optim.Adam on the fused
    op's dense gradients, from the same weights and shuffles, with weight decay."""
    from spotlight_b200.factorization.explicit import ExplicitFactorizationModel
    from spotlight_b200.interactions import Interactions
    rs = np.random.RandomState(D)
    U, I, n = 400, 300, 2000
    inter = Interactions(rs.randint(0, U, n).astype(np.int32), rs.randint(0, I, n).astype(np.int32),
                         ratings=_ratings(loss, rs, n), num_users=U, num_items=I)
    models = []
    for func in (None, lambda p: torch.optim.Adam(p, lr=1e-2, weight_decay=1e-3)):
        m = ExplicitFactorizationModel(loss=loss, embedding_dim=D, n_iter=2, batch_size=128, l2=1e-3,
                                       optimizer_func=func, use_cuda=True, random_state=np.random.RandomState(3))
        m._initialize(inter)
        models.append(m)
    models[1]._net.load_state_dict(models[0]._net.state_dict())
    assert models[0]._route() == 'epoch' and models[1]._route() == 'fused'
    for m in models:
        m.fit(inter)
    # Adam normalises by |g|: fp32 evaluations of the same recurrence drift where a component is ~0
    for (k, a), (_, b) in zip(models[0]._net.state_dict().items(), models[1]._net.state_dict().items()):
        assert_close(a.cpu().numpy(), b.cpu().numpy(), 2e-3, atol=1e-7, what=k)


@pytest.mark.parametrize('route', ['epoch', 'fused'])
def test_float64_integer_ratings_train_as_float32(route):
    """Ratings reach the device as float32: an integer-valued float64 rating array trains to
    exactly the weights its float32 copy does (the reference would compute that loss in float64)."""
    from spotlight_b200 import optim
    from spotlight_b200.factorization.explicit import ExplicitFactorizationModel
    from spotlight_b200.interactions import Interactions
    rs = np.random.RandomState(12)
    U, I, n = 200, 150, 1500
    users, items = rs.randint(0, U, n).astype(np.int32), rs.randint(0, I, n).astype(np.int32)
    r32 = _ratings('regression', rs, n)
    states = []
    for r in (r32, r32.astype(np.float64)):
        func = optim.fused_sgd(lr=0.01) if route == 'epoch' else (lambda p: torch.optim.SGD(p, lr=0.01))
        m = ExplicitFactorizationModel(embedding_dim=16, n_iter=2, batch_size=128, optimizer_func=func, use_cuda=True,
                                       random_state=np.random.RandomState(5))
        m.fit(Interactions(users, items, ratings=r, num_users=U, num_items=I))
        assert m._route() == route
        states.append({k: v.cpu().numpy() for k, v in m._net.state_dict().items()})
    for k in states[0]:
        assert np.array_equal(states[0][k], states[1][k]), k


def test_configs1_shape_against_aten():
    """1M users x 100K items x 64, B = 524 288: one dense step against an fp32 ATen restatement."""
    from spotlight_b200 import _lib, ops
    g = torch.Generator(device='cuda').manual_seed(0)
    U, I, D, B = 1_000_000, 100_000, 64, 524_288
    Wu = torch.randn(U, D, device='cuda', generator=g) / 8
    Wi = torch.randn(I, D, device='cuda', generator=g) / 8
    bu = torch.randn(U, 1, device='cuda', generator=g) * 0.1
    bi = torch.randn(I, 1, device='cuda', generator=g) * 0.1
    users = torch.randint(0, U, (B,), device='cuda', generator=g)
    items = torch.randint(0, I, (B,), device='cuda', generator=g)
    ratings = torch.randint(1, 6, (B,), device='cuda', generator=g).float()
    out = ops.mf_rating_train_step(Wu, Wi, bu, bi, users, items, ratings, _lib.LOSS_KIND['regression'], True)
    s = (Wu[users] * Wi[items]).sum(1) + bu[users, 0] + bi[items, 0]
    gs = 2.0 * (s - ratings) / B
    ref = [((ratings - s) ** 2).mean(), s,
           torch.zeros_like(Wu).index_add_(0, users, gs[:, None] * Wi[items]),
           torch.zeros_like(Wi).index_add_(0, items, gs[:, None] * Wu[users]),
           torch.zeros_like(bu).index_add_(0, users, gs[:, None]),
           torch.zeros_like(bi).index_add_(0, items, gs[:, None])]
    for what, a, e in zip(('loss', 'scores', 'dWu', 'dWi', 'dbu', 'dbi'), out, ref):
        assert_close(a.cpu().numpy(), e.cpu().numpy(), 1e-5, what=what)


def _ref_loss(loss, r, p):
    if loss == 'regression':
        return ((r - p) ** 2).mean()
    if loss == 'poisson':
        return (p - r * torch.log(p)).mean()
    return torch.nn.functional.binary_cross_entropy_with_logits(p, torch.clamp(r, 0, 1))


@pytest.mark.parametrize('loss', LOSSES)
def test_standalone_losses_against_torch(loss):
    from spotlight_b200 import losses
    rs = np.random.RandomState(1)
    r = torch.from_numpy(_ratings(loss, rs, 1001)).cuda()
    x = torch.from_numpy(rs.randn(1001).astype(np.float32)).cuda()
    p1 = (x.exp() if loss == 'poisson' else x).clone().requires_grad_(True)
    p2 = p1.detach().clone().requires_grad_(True)
    l1 = getattr(losses, loss + '_loss')(r, p1)
    l2 = _ref_loss(loss, r, p2)
    l1.backward()
    l2.backward()
    assert_close(l1.item(), l2.item(), 1e-5, what='loss')
    assert_close(p1.grad.cpu().numpy(), p2.grad.cpu().numpy(), 1e-5, what='grad')
    with pytest.raises(ValueError):
        getattr(losses, loss + '_loss')(r.clone().requires_grad_(True), p1)


@pytest.mark.parametrize('loss', LOSSES)
@pytest.mark.parametrize('rep', ['bloom', 'custom'])
def test_generic_route_against_autograd(loss, rep):
    """A Bloom item layer and a custom representation train on the generic route: the same loop
    replayed with torch autograd on the restated losses gives the same weights."""
    from spotlight_b200.factorization.explicit import ExplicitFactorizationModel
    from spotlight_b200.factorization.representations import BilinearNet
    from spotlight_b200.interactions import Interactions
    from spotlight_b200.layers import BloomEmbedding
    rs = np.random.RandomState(8)
    U, I, n, B = 60, 90, 700, 128
    inter = Interactions(rs.randint(0, U, n).astype(np.int32), rs.randint(0, I, n).astype(np.int32),
                         ratings=_ratings(loss, rs, n), num_users=U, num_items=I)
    torch.manual_seed(0)
    if rep == 'bloom':
        net = BilinearNet(U, I, 16, item_embedding_layer=BloomEmbedding(I, 16, compression_ratio=0.5,
                                                                        num_hash_functions=2))
        bilinear = net
    else:
        class Custom(torch.nn.Module):
            def __init__(self):
                super().__init__()
                self.inner = BilinearNet(U, I, 16)

            def forward(self, user_ids, item_ids):
                return self.inner(user_ids, item_ids) * 0.5
        net = Custom()
        bilinear = net.inner
    with torch.no_grad():
        bilinear.user_biases.weight.normal_(0, 0.1)
    twin = copy.deepcopy(net).cuda()
    model = ExplicitFactorizationModel(loss=loss, n_iter=2, batch_size=B, representation=net, use_cuda=True,
                                       optimizer_func=lambda p: torch.optim.SGD(p, lr=0.05),
                                       random_state=np.random.RandomState(6))
    rs_copy = np.random.RandomState()
    rs_copy.set_state(model._random_state.get_state())
    model.fit(inter)
    assert model._route() == 'generic'
    opt = torch.optim.SGD(twin.parameters(), lr=0.05)
    for _ in range(2):
        order = np.arange(n)
        rs_copy.shuffle(order)
        u = torch.from_numpy(inter.user_ids[order].astype(np.int64)).cuda()
        i = torch.from_numpy(inter.item_ids[order].astype(np.int64)).cuda()
        r = torch.from_numpy(inter.ratings[order]).cuda()
        for lo in range(0, n, B):
            p = twin(u[lo:lo + B], i[lo:lo + B])
            if loss == 'poisson':
                p = torch.exp(p)
            opt.zero_grad()
            _ref_loss(loss, r[lo:lo + B], p).backward()
            opt.step()
    for (k, a), (_, b) in zip(model._net.state_dict().items(), twin.state_dict().items()):
        assert_close(a.cpu().numpy(), b.cpu().numpy(), 1e-5, atol=1e-7, what=k)


@pytest.mark.parametrize('loss', LOSSES)
def test_predict_forms_and_transform(loss):
    from spotlight_b200.factorization.explicit import ExplicitFactorizationModel
    from spotlight_b200.interactions import Interactions
    rs = np.random.RandomState(0)
    U, I = 20, 30
    inter = Interactions(rs.randint(0, U, 200).astype(np.int32), rs.randint(0, I, 200).astype(np.int32),
                         ratings=_ratings(loss, rs, 200), num_users=U, num_items=I)
    model = ExplicitFactorizationModel(loss=loss, n_iter=1, use_cuda=True, random_state=np.random.RandomState(1))
    model.fit(inter)
    net = model._net
    sd = {k: v.cpu().numpy().astype(np.float64) for k, v in net.state_dict().items()}

    def expect(u, i):
        s = (sd['user_embeddings.weight'][u] * sd['item_embeddings.weight'][i]).sum(-1) + \
            sd['user_biases.weight'][u, 0] + sd['item_biases.weight'][i, 0]
        return oex.transform(loss, s)

    all_items = model.predict(3)
    assert all_items.dtype == np.float32 and all_items.shape == (I,)
    assert_close(all_items, expect(np.full(I, 3), np.arange(I)), 1e-5)
    some = np.array([0, 5, 29])
    assert_close(model.predict(3, some), expect(np.full(3, 3), some), 1e-5)
    us = np.array([1, 2, 19])
    assert_close(model.predict(us, some), expect(us, some), 1e-5)


def test_rmse_score_blocks_against_numpy(monkeypatch):
    from spotlight_b200 import evaluation
    from spotlight_b200.factorization.explicit import ExplicitFactorizationModel
    from spotlight_b200.interactions import Interactions
    rs = np.random.RandomState(0)
    U, I, n = 50, 70, 3000
    inter = Interactions(rs.randint(0, U, n).astype(np.int32), rs.randint(0, I, n).astype(np.int32),
                         ratings=_ratings('regression', rs, n), num_users=U, num_items=I)
    model = ExplicitFactorizationModel(n_iter=2, use_cuda=True, random_state=np.random.RandomState(1))
    model.fit(inter)
    expect = np.sqrt(((inter.ratings.astype(np.float64) -
                       model.predict(inter.user_ids, inter.item_ids)) ** 2).mean())
    monkeypatch.setattr(evaluation, '_RMSE_BLOCK', 1000)
    assert_close(evaluation.rmse_score(model, inter), expect, 1e-5)


def test_errors_and_pickling(tmp_path):
    from spotlight_b200.factorization.explicit import ExplicitFactorizationModel
    from spotlight_b200.interactions import Interactions
    rs = np.random.RandomState(0)
    U, I, n = 20, 30, 300
    users, items = rs.randint(0, U, n).astype(np.int32), rs.randint(0, I, n).astype(np.int32)
    ratings = _ratings('regression', rs, n)
    inter = Interactions(users, items, ratings=ratings, num_users=U, num_items=I)

    with pytest.raises(RuntimeError):
        ExplicitFactorizationModel(use_cuda=False).fit(inter)
    with pytest.raises(TypeError):
        ExplicitFactorizationModel(n_iter=1, use_cuda=True).fit(Interactions(users, items, num_users=U,
                                                                             num_items=I))
    bad = users.copy()
    bad[3] = -1
    with pytest.raises(IndexError):
        ExplicitFactorizationModel(n_iter=1, use_cuda=True).fit(
            Interactions(bad, items, ratings=ratings, num_users=U, num_items=I))
    nan = ratings.copy()
    nan[0] = np.nan
    with pytest.raises(ValueError):
        ExplicitFactorizationModel(n_iter=1, use_cuda=True).fit(
            Interactions(users, items, ratings=nan, num_users=U, num_items=I))

    model = ExplicitFactorizationModel(n_iter=1, use_cuda=True, random_state=np.random.RandomState(2))
    model.fit(inter)
    with pytest.raises(ValueError):
        model.predict(U)
    with pytest.raises(ValueError):
        model.predict(0, np.array([I]))
    big = users.copy()
    big[0] = U
    with pytest.raises(ValueError):
        model.fit(Interactions(big, items, ratings=ratings, num_users=U + 1, num_items=I))

    path = str(tmp_path / 'model.pt')
    torch.save(model, path)
    loaded = torch.load(path, weights_only=False)
    assert np.array_equal(loaded.predict(users, items), model.predict(users, items))
    loaded.fit(inter)                      # training resumes from the pickled state


def test_implicit_default_adam_model_resumes_after_pickling(tmp_path):
    """FusedAdam keeps its step count through torch.save / torch.load, so a pickled default-Adam
    model (implicit or explicit) resumes fit() exactly where an unpickled one does."""
    from spotlight_b200.factorization.implicit import ImplicitFactorizationModel
    from spotlight_b200.interactions import Interactions
    rs = np.random.RandomState(0)
    inter = Interactions(rs.randint(0, 50, 800).astype(np.int32), rs.randint(0, 60, 800).astype(np.int32),
                         num_users=50, num_items=60)
    model = ImplicitFactorizationModel(loss='bpr', embedding_dim=8, n_iter=1, use_cuda=True,
                                       random_state=np.random.RandomState(1))
    model.fit(inter)
    path = str(tmp_path / 'implicit.pt')
    torch.save(model, path)
    loaded = torch.load(path, weights_only=False)
    assert loaded._optimizer.steps_taken == model._optimizer.steps_taken > 0
    model.fit(inter)
    loaded.fit(inter)
    for (k, a), (_, b) in zip(model._net.state_dict().items(), loaded._net.state_dict().items()):
        assert torch.equal(a, b), k
