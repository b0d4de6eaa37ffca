"""NCCL / device tests of the sharded hashed-table (Bloom) model with Adagrad and lazy-exact Adam.

* The users-only mode of slb_mf_bloom_train_step (through ops.mf_bloom_step_pairs) against the float64
  oracle (oracle.bloom.step plus oracle.adam.LazyAdamTable): D in {16, 64, 128}, H in {1, 4}, pointwise,
  bpr and hinge, Adagrad and Adam, on Zipf batches with a hot user and a hot item id.
* slb_bias_sparse_adam against LazyAdamTable (repeated ids, padding pairs, ids several steps behind),
  and replicas with different catch-up histories ending bit-identical.
* World-1 fit() (world 2 as well when two GPUs are visible) of a BilinearNet with a BloomEmbedding item
  layer, three losses x {fused_adagrad, fused_adam}, against the single-GPU ImplicitFactorizationModel
  on the same net from the same seed, and mrr_score of the gathered net against the single-GPU model's.
"""

import copy
import os
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT, assert_close
from oracle import bloom as ob
from oracle.adam import LazyAdamTable

sys.path.insert(0, os.path.join(ROOT, 'tests'))
pytestmark = pytest.mark.gpu

import sharded_common as sc                                  # noqa: E402
from test_sharded_seq_adam_cpu import _check_adam              # noqa: E402

DEV = 'cuda:0'
LR, WD, BETAS, EPS = 1e-2, 1e-2, (0.9, 0.999), 1e-8


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _zipf_batch(rs, B, U, N):
    """Zipf users and items, with user 3 and item id 7 hot (a fifth of the batch each)."""
    users = (rs.zipf(1.3, B) - 1) % U
    items = (rs.zipf(1.3, B) - 1) % (N - 1) + 1
    users[rs.rand(B) < 0.2] = 3
    items[rs.rand(B) < 0.2] = 7
    negs = rs.randint(0, N, B)
    return users.astype(np.int64), items.astype(np.int64), negs.astype(np.int64)


def _case(D, H, seed):
    rs = np.random.RandomState(seed)
    U, N, M, B = 150, 3000, 400, 700
    Wu = (rs.randn(U, D) * 0.3).astype(np.float32)
    Wi = (rs.randn(M, D) * 0.3).astype(np.float32)
    Wi[0] = 0
    bu = (rs.randn(U, 1) * 0.1).astype(np.float32)
    bi = (rs.randn(N, 1) * 0.1).astype(np.float32)
    users, items, negs = _zipf_batch(rs, B, U, N)
    return rs, dict(Wu=Wu, Wi=Wi, bu=bu, bi=bi, users=users, items=items, negs=negs, H=H, norm=3 * B)


def _seeds(H):
    from spotlight_b200.layers import SEEDS
    return [int(x) for x in SEEDS[:H]]


def _ref(c, Wu, bu, bi, loss):
    return ob.step([Wu, c['Wi'].astype(np.float64), bu, bi], c['users'], c['items'], c['negs'], loss, 0, c['H'], -1,
                   0, norm=c['norm'])


def _pair_sums(ids, g, n):
    ids, g = ids.cpu().numpy(), g.cpu().numpy().astype(np.float64)
    out = np.zeros(n)
    live = ids >= 0
    np.add.at(out, ids[live], g[live])
    return out


@pytest.mark.parametrize('D', [16, 64, 128])
@pytest.mark.parametrize('H', [1, 4])
@pytest.mark.parametrize('loss', ['pointwise', 'bpr', 'hinge'])
def test_users_only_adagrad(D, H, loss):
    """Adagrad on the user rows and biases in place; dense dWi and item-bias pairs handed out."""
    from spotlight_b200 import _lib, ops
    rs, c = _case(D, H, seed=D + H)
    sWu0 = rs.uniform(0.5, 1.5, c['Wu'].shape).astype(np.float32) * 1e-6
    sbu0 = rs.uniform(0.5, 1.5, c['bu'].shape).astype(np.float32) * 1e-4
    Wu, bu, sWu, sbu = t(c['Wu']), t(c['bu']), t(sWu0), t(sbu0)
    dWi = torch.zeros((c['Wi'].shape[0], D), device=DEV)
    lval, dWu, dW, up, (ii, gi) = ops.mf_bloom_step_pairs(
        Wu, t(c['Wi']), bu, t(c['bi']), t(c['users']), t(c['items']), t(c['negs']), loss, _seeds(H), 0,
        norm_batch=c['norm'], users_only=dict(opt=_lib.OPT_ADAGRAD, lr=0.05, eps=1e-10, states=(sWu, sbu.reshape(-1))),
        dWi=dWi)
    assert dWu is None and up is None and dW is dWi
    ref = _ref(c, c['Wu'].astype(np.float64), c['bu'].astype(np.float64), c['bi'].astype(np.float64), loss)
    assert_close(lval.item(), ref['loss'], 1e-5, what='loss')
    assert_close(dWi.cpu().numpy(), ref['dWi'], 1e-5, what='dWi')
    assert_close(_pair_sums(ii, gi, len(c['bi'])), ref['dbi'].reshape(-1), 1e-5, atol=1e-12, what='item-bias pairs')
    for got, w0, s0, g, nm in ((Wu, c['Wu'], sWu0, ref['dWu'], 'Wu'), (bu, c['bu'], sbu0, ref['dbu'], 'bu')):
        s = s0.astype(np.float64) + g * g
        want = w0 - 0.05 * g / (np.sqrt(s) + 1e-10)
        sc_ = {'Wu': sWu, 'bu': sbu}[nm]
        assert_close(got.cpu().numpy(), want, 1e-5, what=nm)
        assert_close(sc_.cpu().numpy(), s, 1e-5, what='s' + nm)


def _adam_tabs(rs, c, T):
    """LazyAdamTables of Wu, bu (sharing last) and bi at steps taken T - 1: seeded moments and rows
    0, 1, 2 and 4 steps behind."""
    kw = dict(lr=LR, betas=BETAS, eps=EPS, weight_decay=WD)
    tabs = [LazyAdamTable(c[k], **kw) for k in ('Wu', 'bu', 'bi')]
    last_u = np.maximum(T - 1 - rs.choice([0, 1, 2, 4], len(c['Wu'])), 0)
    last_b = np.maximum(T - 1 - rs.choice([0, 1, 2, 4], len(c['bi'])), 0)
    for tab, last in zip(tabs, (last_u, last_u, last_b)):
        tab.m = rs.randn(*tab.w.shape) * 1e-3
        tab.v = rs.uniform(0.5, 1.5, tab.w.shape) * 1e-6
        tab.m, tab.v = tab.m.astype(np.float32).astype(np.float64), tab.v.astype(np.float32).astype(np.float64)
        tab.last = last.copy()
    return tabs


@pytest.mark.parametrize('D', [16, 64, 128])
@pytest.mark.parametrize('H', [1, 4])
@pytest.mark.parametrize('loss', ['pointwise', 'bpr', 'hinge'])
def test_users_only_adam(D, H, loss):
    """Step T: the referenced user rows, user biases and item-bias ids caught up through T - 1, then
    step T on the touched user rows and biases; the item biases are only caught up."""
    from spotlight_b200 import _lib, ops
    from spotlight_b200.optim import FusedAdam
    rs, c = _case(D, H, seed=10 * D + H)
    T = 6
    tabs = _adam_tabs(rs, c, T)
    f = lambda x: t(x.astype(np.float32))             # noqa: E731
    Wu, mWu, vWu = f(tabs[0].w), f(tabs[0].m), f(tabs[0].v)
    bu, mbu, vbu = f(tabs[1].w), f(tabs[1].m), f(tabs[1].v)
    bi, mbi, vbi = f(tabs[2].w), f(tabs[2].m), f(tabs[2].v)
    last_u, last_bi = t(tabs[0].last.astype(np.int32)), t(tabs[2].last.astype(np.int32))
    opt = FusedAdam([torch.zeros(1, device=DEV)], lr=LR, betas=BETAS, eps=EPS, weight_decay=WD)
    dWi = torch.zeros((c['Wi'].shape[0], D), device=DEV)
    uo = dict(opt=_lib.OPT_ADAM, lr=LR, eps=EPS, weight_decay=WD, beta1=BETAS[0], beta2=BETAS[1],
              sched=opt.schedule(T, torch.device(DEV)), step=T,
              states=((mWu, vWu, last_u), (mbu, vbu), (mbi, vbi, last_bi)))
    lval, _, _, _, (ii, gi) = ops.mf_bloom_step_pairs(
        Wu, t(c['Wi']), bu, bi, t(c['users']), t(c['items']), t(c['negs']), loss, _seeds(H), 0,
        norm_batch=c['norm'], users_only=uo, dWi=dWi)
    # the oracle: catch-up, forward / backward, step T on the touched user rows and biases
    tabs[0].catch_up(c['users'], T - 1)
    tabs[1].catch_up(c['users'], T - 1)
    tabs[2].catch_up(np.r_[c['items'], c['negs']], T - 1)
    ref = _ref(c, tabs[0].w, tabs[1].w, tabs[2].w, loss)
    rows = np.flatnonzero(ref['touched'][0])
    assert np.array_equal(rows, np.flatnonzero(ref['touched'][2]))
    tabs[0].apply(rows, ref['dWu'][rows], T)
    tabs[1].apply(rows, ref['dbu'][rows], T)
    assert_close(lval.item(), ref['loss'], 1e-5, what='loss')
    assert_close(dWi.cpu().numpy(), ref['dWi'], 1e-5, what='dWi')
    assert_close(_pair_sums(ii, gi, len(c['bi'])), ref['dbi'].reshape(-1), 1e-5, atol=1e-12, what='item-bias pairs')
    for got, tab, nm in ((Wu, tabs[0], 'Wu'), (bu, tabs[1], 'bu'), (bi, tabs[2], 'bi')):
        assert_close(got.cpu().numpy(), tab.w, 1e-5, what=nm)
    for got, tab, nm in ((mWu, tabs[0], 'mWu'), (mbu, tabs[1], 'mbu'), (mbi, tabs[2], 'mbi')):
        assert_close(got.cpu().numpy(), tab.m, 1e-5, what=nm)
    for got, tab, nm in ((vWu, tabs[0], 'vWu'), (vbu, tabs[1], 'vbu'), (vbi, tabs[2], 'vbi')):
        assert_close(got.cpu().numpy(), tab.v, 1e-5, what=nm)
    assert np.array_equal(last_u.cpu().numpy(), tabs[0].last)
    assert np.array_equal(last_bi.cpu().numpy(), tabs[2].last)


def test_users_only_rejections():
    """Adaptive hinge and the missing item-bias pairs fail with SLB_EINVAL and a message."""
    from spotlight_b200 import _lib, ops
    _, c = _case(16, 2, seed=1)
    sWu, sbu = torch.zeros((len(c['Wu']), 16), device=DEV), torch.zeros(len(c['bu']), device=DEV)
    uo = dict(opt=_lib.OPT_ADAGRAD, lr=0.05, eps=1e-10, states=(sWu, sbu))
    negs = np.r_[c['negs'], c['negs']]
    with pytest.raises(Exception, match='users-only mode takes the pointwise, bpr and hinge'):
        ops.mf_bloom_step_pairs(t(c['Wu']), t(c['Wi']), t(c['bu']), t(c['bi']), t(c['users']), t(c['items']),
                                t(negs[:len(c['users'])]), 'adaptive_hinge', _seeds(2), 0, users_only=uo)


def test_bias_sparse_adam():
    """Repeated ids summed in pair order, padding pairs (0, 0) and skipped ids (-1), ids up to five
    steps behind; a replica that another kernel caught up through T - 1 first ends bit-identical."""
    from spotlight_b200 import _lib, ops
    from spotlight_b200.optim import FusedAdam
    lib = _lib.load()
    rs = np.random.RandomState(4)
    N, n, T = 5000, 3000, 7
    ids = rs.randint(0, N, n)
    ids[rs.rand(n) < 0.1] = 11                         # a hot id
    g = (rs.randn(n) * 1e-3).astype(np.float32)
    ids[-200:], g[-200:] = 0, 0.0                      # all-gather padding
    ids[:50] = -1                                      # pairs that touch nothing
    tab = LazyAdamTable(rs.randn(N, 1) * 0.1, lr=LR, betas=BETAS, eps=EPS, weight_decay=WD)
    tab.w = tab.w.astype(np.float32).astype(np.float64)
    tab.m = (rs.randn(N, 1) * 1e-3).astype(np.float32).astype(np.float64)
    tab.v = (rs.uniform(0.5, 1.5, (N, 1)) * 1e-6).astype(np.float32).astype(np.float64)
    tab.last = np.maximum(T - 1 - rs.randint(0, 6, N), 0)
    opt = FusedAdam([torch.zeros(1, device=DEV)], lr=LR, betas=BETAS, eps=EPS, weight_decay=WD)
    sched = opt.schedule(T, torch.device(DEV))
    f = lambda x: t(x.astype(np.float32))             # noqa: E731
    reps = []
    for caught_up in (False, True):
        b, m, v, last = f(tab.w), f(tab.m), f(tab.v), t(tab.last.astype(np.int32))
        if caught_up:                                  # every id replayed through T - 1 by the flush kernel
            _lib.check(lib.slb_adam_flush_table(ops._ptr(b), ops._ptr(m), ops._ptr(v), ops._ptr(last), N, 1,
                                                ops._ptr(sched), T - 1, BETAS[0], BETAS[1], 1 - BETAS[0],
                                                1 - BETAS[1], EPS, WD, ops._stream()), 'flush')
        ops.bias_sparse_adam(t(ids), t(g), b, m, v, last, sched, T, BETAS[0], BETAS[1], EPS, WD)
        reps.append((b, m, v, last))
    live = ids >= 0
    sums = np.zeros(N)
    np.add.at(sums, ids[live], g[live].astype(np.float64))
    rows = np.unique(ids[live])
    tab.catch_up(rows, T - 1)
    tab.apply(rows, sums[rows].reshape(-1, 1), T)
    b, m, v, last = reps[0]
    assert_close(b.cpu().numpy(), tab.w, 1e-5, what='bias')
    assert_close(m.cpu().numpy(), tab.m, 1e-5, what='exp_avg')
    assert_close(v.cpu().numpy(), tab.v, 1e-5, what='exp_avg_sq')
    assert np.array_equal(last.cpu().numpy(), tab.last)
    for b, m, v, last in reps:                         # flush both replicas through T + 2
        sched2 = opt.schedule(T + 2, torch.device(DEV))
        _lib.check(lib.slb_adam_flush_table(ops._ptr(b), ops._ptr(m), ops._ptr(v), ops._ptr(last), N, 1,
                                            ops._ptr(sched2), T + 2, BETAS[0], BETAS[1], 1 - BETAS[0], 1 - BETAS[1],
                                            EPS, WD, ops._stream()), 'flush')
    for x, y in zip(reps[0], reps[1]):
        assert torch.equal(x, y)


def test_adam_dense_table():
    """slb_adam_dense_table: every row replays its pending steps and takes step T, zero rows included."""
    from spotlight_b200 import _lib, ops
    from spotlight_b200.optim import FusedAdam
    rs = np.random.RandomState(5)
    rows, D, T = 333, 12, 5
    tab = LazyAdamTable((rs.randn(rows, D) * 0.3).astype(np.float32), lr=LR, betas=BETAS, eps=EPS, weight_decay=WD)
    tab.m = (rs.randn(rows, D) * 1e-3).astype(np.float32).astype(np.float64)
    tab.v = (rs.uniform(0.5, 1.5, (rows, D)) * 1e-6).astype(np.float32).astype(np.float64)
    tab.last = np.maximum(T - 1 - rs.randint(0, 4, rows), 0)
    G = (rs.randn(rows, D) * 1e-3).astype(np.float32)
    G[rs.rand(rows) < 0.3] = 0
    f = lambda x: t(x.astype(np.float32))             # noqa: E731
    W, m, v, last, Gd = f(tab.w), f(tab.m), f(tab.v), t(tab.last.astype(np.int32)), t(G)
    opt = FusedAdam([torch.zeros(1, device=DEV)], lr=LR, betas=BETAS, eps=EPS, weight_decay=WD)
    sched = opt.schedule(T, torch.device(DEV))
    lib = _lib.load()
    _lib.check(lib.slb_adam_dense_table(ops._ptr(W), ops._ptr(m), ops._ptr(v), ops._ptr(last), ops._ptr(Gd), rows,
                                        D, ops._ptr(sched), T, BETAS[0], BETAS[1],
                                        1 - BETAS[0], 1 - BETAS[1], EPS, WD, ops._stream()), 'adam_dense_table')
    every = np.arange(rows)
    tab.catch_up(every, T - 1)
    tab.apply(every, G.astype(np.float64), T)
    assert_close(W.cpu().numpy(), tab.w, 1e-5, what='W')
    assert_close(m.cpu().numpy(), tab.m, 1e-5, what='exp_avg')
    assert np.array_equal(last.cpu().numpy(), np.full(rows, T))
    assert lib.slb_adam_dense_table(None, None, None, None, None, 0, D, None, T, 0.9, 0.999, 0.1, 0.001, EPS, WD,
                                    ops._stream()) == 0
    assert lib.slb_adam_dense_table(ops._ptr(W), None, None, None, None, rows, D, None, T, 0.9, 0.999, 0.1, 0.001,
                                    EPS, WD, ops._stream()) != 0


# ------------------------------------------------------------------ fit()

FIT = dict(U=120, I=3000, D=16, H=3, B=256, n=1900, n_iter=2, seed=21)
LOSSES = ['pointwise', 'bpr', 'hinge']
OPTS = ['adagrad', 'adam']
WORLDS = [1] + ([2] if torch.cuda.is_available() and torch.cuda.device_count() >= 2 else [])


def _opt(name):
    from spotlight_b200 import optim
    return optim.fused_adagrad(lr=0.05) if name == 'adagrad' else optim.fused_adam(lr=LR, weight_decay=1e-3)


def _net():
    from spotlight_b200.factorization.representations import BilinearNet
    from spotlight_b200.layers import BloomEmbedding
    torch.manual_seed(3)
    net = BilinearNet(FIT['U'], FIT['I'], FIT['D'],
                      item_embedding_layer=BloomEmbedding(FIT['I'], FIT['D'], compression_ratio=0.1,
                                                          num_hash_functions=FIT['H']))
    with torch.no_grad():
        net.user_biases.weight.normal_(0, 0.1)
        net.item_biases.weight.normal_(0, 0.1)
    return net


def _data():
    rs = np.random.RandomState(8)
    return (rs.randint(0, FIT['U'], FIT['n']).astype(np.int32),
            rs.randint(1, FIT['I'], FIT['n']).astype(np.int32))


def _tables(net):
    return [p.detach().cpu().numpy() for p in (net.user_embeddings.weight, net.item_embeddings.embeddings.weight,
                                               net.user_biases.weight, net.item_biases.weight)]


def _fit_job(rank, world, dev, loss, opt):
    from spotlight_b200.interactions import Interactions
    from spotlight_b200.sharded import ShardedImplicitFactorizationModel
    users, items = _data()
    rs = np.random.RandomState(FIT['seed'])
    model = ShardedImplicitFactorizationModel(FIT['U'], FIT['I'], rank, world, dev, loss=loss, n_iter=FIT['n_iter'],
                                              batch_size=FIT['B'], random_state=rs, optimizer_func=_opt(opt),
                                              representation=_net())
    model.fit(Interactions(users, items, num_users=FIT['U'], num_items=FIT['I']))
    net = model.gathered_net()
    return _tables(net), model.epoch_losses, rs.get_state(), net.cpu()


_RES, _SINGLE = {}, {}


def _results(world):
    if world not in _RES:
        _RES[world] = sc.run_world(_fit_jobs, world, backend='nccl', timeout=900)
    return _RES[world]


def _fit_jobs(rank, world, dev):
    return {(loss, opt): _fit_job(rank, world, dev, loss, opt) for loss in LOSSES for opt in OPTS}


def _single(loss, opt):
    if (loss, opt) not in _SINGLE:
        from spotlight_b200.factorization.implicit import ImplicitFactorizationModel
        from spotlight_b200.interactions import Interactions
        users, items = _data()
        inter = Interactions(users, items, num_users=FIT['U'], num_items=FIT['I'])
        rs = np.random.RandomState(FIT['seed'])
        one = ImplicitFactorizationModel(loss=loss, embedding_dim=FIT['D'], n_iter=FIT['n_iter'], batch_size=FIT['B'],
                                         use_cuda=True, random_state=rs, representation=_net(),
                                         optimizer_func=_opt(opt))
        losses = []
        orig = one._fit_epoch_bloom_fused

        def traced(*a, **kw):
            out = orig(*a, **kw)
            losses.append(out)
            return out
        one._fit_epoch_bloom_fused = traced
        one.fit(inter)
        assert len(losses) == FIT['n_iter'], 'the single-GPU fit did not take the fused Bloom route'
        _SINGLE[loss, opt] = (_tables(one._net), losses, rs.get_state(), one, inter)
    return _SINGLE[loss, opt]


@pytest.mark.parametrize('world', WORLDS)
@pytest.mark.parametrize('opt', OPTS)
@pytest.mark.parametrize('loss', LOSSES)
def test_sharded_bloom_fit_equals_single_gpu_fit(world, loss, opt):
    """fit() of the sharded Bloom model (two epochs, a short last minibatch) against the single-GPU
    fused Bloom fit on the same net from the same seed: epoch losses, the four tables, the final
    RandomState, and mrr_score of gathered_net() against the single-GPU model's."""
    from spotlight_b200.evaluation import mrr_score
    got, losses, state, net = _results(world)[0][loss, opt]
    ref, want_losses, want_state, one, inter = _single(loss, opt)
    assert_close(np.array(losses), np.array(want_losses, dtype=np.float64), 2e-5, what='epoch losses')
    lr = LR if opt == 'adam' else 0.05
    for a, b, nm in zip(got, ref, ('Wu', 'Wi', 'bu', 'bi')):
        _check_adam(a, b.reshape(a.shape).astype(np.float64), lr, nm, rtol=1e-4)
    assert np.array_equal(state[1], want_state[1]) and state[2] == want_state[2]
    twin = copy.copy(one)
    twin._net = net.to(DEV)
    assert_close(mrr_score(twin, inter), mrr_score(one, inter), 1e-4, what='mrr')
