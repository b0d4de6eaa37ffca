"""World-size-2 and 3 gloo tests of the sharded hashed-table (Bloom) model on CPU, with a NumPy backend
that runs the users-only local step and the owners' and replicas' lazy-exact Adam in float64
(oracle.adam.LazyAdamTable): ShardedBloomMF steps under pointwise, bpr and hinge against a
single-process float64 step with dense Adam on all four tables of the concatenated minibatch, and
ShardedImplicitFactorizationModel(representation=<Bloom net>).fit() against a float64 replay of the
reference's stream under Adagrad and Adam.  Also the optimizer and representation selection."""

import os
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT, assert_close

sys.path.insert(0, os.path.join(ROOT, 'tests'))

import sharded_common as sc                                  # noqa: E402
from oracle import bloom as ob                               # noqa: E402
from oracle import mf as omf                                 # noqa: E402
from oracle.adam import LazyAdamTable                        # noqa: E402
from test_sharded_seq_adam_cpu import DenseAdam, _check_adam   # noqa: E402

LR = 1e-2


class F32AdamTable(LazyAdamTable):
    """LazyAdamTable whose every step (replayed or real) rounds the row, exp_avg and exp_avg_sq to
    float32, as the kernels' step-by-step replay does: a replica then ends the same whichever call
    caught an id up."""

    def _step(self, rows, t, g):
        super(F32AdamTable, self)._step(rows, t, g)
        for x in (self.w, self.m, self.v):
            x[rows] = x[rows].astype(np.float32)


class BloomAdamBackend(sc.NumpyBackend):
    """NumpyBackend plus the users-only hashed step and lazy-exact Adam in float64 on the float32
    tensors of BloomShardState (stored back as float32 after every call)."""

    @staticmethod
    def _kw(st):
        hp = st.opt.fused_hparams()
        return dict(lr=hp['lr'], betas=(hp['beta1'], hp['beta2']), eps=hp['eps'], weight_decay=hp['weight_decay'])

    def _tab(self, st, w, m, v, last):
        tab = F32AdamTable(w.numpy().reshape(m.shape), **self._kw(st))
        tab.m, tab.v = m.numpy().astype(np.float64), v.numpy().astype(np.float64)
        tab.last = last.numpy().astype(np.int64)
        return tab

    @staticmethod
    def _store(tab, w, m, v, last):
        for dst, src in ((w, tab.w), (m, tab.m), (v, tab.v)):
            dst.copy_(torch.from_numpy(src.reshape(dst.shape).astype(np.float32)))
        if last is not None:
            last.copy_(torch.from_numpy(tab.last.astype(np.int32)))

    def _tables(self, st):
        return [self._tab(st, st.Wu, st.mWu, st.vWu, st.last_u), self._tab(st, st.bu2, st.mbu, st.vbu, st.last_u),
                self._tab(st, st.bi2, st.mbi, st.vbi, st.last_bi)]

    def _store_all(self, st, tabs):
        self._store(tabs[0], st.Wu, st.mWu, st.vWu, st.last_u)
        assert np.array_equal(tabs[0].last, tabs[1].last)
        self._store(tabs[1], st.bu2, st.mbu, st.vbu, None)
        self._store(tabs[2], st.bi2, st.mbi, st.vbi, st.last_bi)

    def bloom_local_step(self, st, W_full, users_local, items, negs, loss, global_batch, t=None):
        if t is None:
            return super(BloomAdamBackend, self).bloom_local_step(st, W_full, users_local, items, negs, loss,
                                                                  global_batch)
        u, i, n = users_local.numpy(), items.numpy(), negs.numpy()
        tabs = self._tables(st)
        tabs[0].catch_up(u, t - 1)
        tabs[1].catch_up(u, t - 1)
        tabs[2].catch_up(np.r_[i, n], t - 1)
        H = len(st.item_seeds)
        ref = ob.step([tabs[0].w, W_full.numpy().astype(np.float64), tabs[1].w, tabs[2].w], u, i, n, loss, 0, H, -1,
                      0, norm=global_batch)
        rows = np.flatnonzero(ref['touched'][0])
        tabs[0].apply(rows, ref['dWu'][rows], t)
        tabs[1].apply(rows, ref['dbu'][rows], t)
        self._store_all(st, tabs)
        ids = np.flatnonzero(ref['touched'][3])
        pairs = (torch.from_numpy(ids.astype(np.int64)),
                 torch.from_numpy(ref['dbi'].reshape(-1)[ids].astype(np.float32)))
        return (torch.tensor(float(ref['loss']), dtype=torch.float32), None,
                torch.from_numpy(ref['dWi'].astype(np.float32)), None, pairs)

    def bloom_adam_dense(self, st, g_shard, t):
        tab = self._tab(st, st.Wi, st.mWi, st.vWi, st.last_i)
        rows = np.arange(tab.w.shape[0])
        tab.catch_up(rows, t - 1)
        tab.apply(rows, g_shard.numpy().astype(np.float64), t)
        self._store(tab, st.Wi, st.mWi, st.vWi, st.last_i)

    def bloom_bias_adam(self, st, ids, g, t):
        ids, g = ids.numpy(), g.numpy().astype(np.float64)
        live = ids >= 0
        sums = np.zeros(st.bi.numel())
        np.add.at(sums, ids[live], g[live])
        rows = np.unique(ids[live])
        tab = self._tab(st, st.bi2, st.mbi, st.vbi, st.last_bi)
        tab.catch_up(rows, t - 1)
        tab.apply(rows, sums[rows].reshape(-1, 1), t)
        self._store(tab, st.bi2, st.mbi, st.vbi, st.last_bi)

    def owner_adam_flush(self, st):
        T = st.opt.steps_taken
        if T < 1:
            return
        if st.Wu.shape[0]:
            tabs = self._tables(st)
            for tab in tabs[:2]:
                tab.flush(T)
            self._store(tabs[0], st.Wu, st.mWu, st.vWu, st.last_u)
            self._store(tabs[1], st.bu2, st.mbu, st.vbu, None)
        for w, m, v, last in ((st.Wi, st.mWi, st.vWi, st.last_i), (st.bi2, st.mbi, st.vbi, st.last_bi)):
            tab = self._tab(st, w, m, v, last)
            tab.flush(T)
            self._store(tab, w, m, v, last)


# ------------------------------------------------------------------ ShardedBloomMF steps

STEP = dict(seed=41, U=23, N=61, M=17, D=8, H=3)
SIZES = (12, 3, 10, 2)       # minibatch sizes; the second holds rank 0's users only
SHARED_ID = 5                # an item id every rank's members use: its hashed rows are touched everywhere
ONLY_PAD = 60                # an item-bias id no interaction touches (the padding pairs step id 0 only)


def _step_problem():
    c = STEP
    rs = np.random.RandomState(c['seed'])
    Wu = (rs.randn(c['U'], c['D']) * 0.3).astype(np.float32)
    Wi = (rs.randn(c['M'], c['D']) * 0.3).astype(np.float32)
    Wi[0] = 0
    bu = (rs.randn(c['U'], 1) * 0.1).astype(np.float32)
    bi = (rs.randn(c['N'], 1) * 0.1).astype(np.float32)
    batches = []
    for k, B in enumerate(SIZES):
        # users below 9 only (rank 0's range at worlds 2 and 3; the last rank owns none of 19..22)
        hi = 9 if k == 1 else 19
        users = rs.randint(0, hi, B).astype(np.int64)
        items = rs.randint(1, ONLY_PAD, B).astype(np.int64)
        items[0] = SHARED_ID
        negs = rs.randint(0, ONLY_PAD, B).astype(np.int64)
        batches.append((users, items, negs))
    return (Wu, Wi, bu, bi), batches


def _step_job(rank, world, dev, loss, wd):
    from spotlight_b200.optim import fused_adam
    from spotlight_b200.sharded import BloomShardState, ShardedBloomMF, ShardPlan
    params, batches = _step_problem()
    c = STEP
    plan = ShardPlan(c['U'] + 4, c['N'], world)          # 4 trailing users no interaction names
    init = [torch.from_numpy(p) for p in params]
    init[0] = torch.cat([init[0], torch.zeros(4, c['D'])])
    init[2] = torch.cat([init[2], torch.zeros(4, 1)])
    st = BloomShardState(plan, rank, c['D'], dev, c['N'], c['M'], c['H'], init=init,
                         optimizer_func=fused_adam(lr=LR, weight_decay=wd))
    model = ShardedBloomMF(plan, st, rank, BloomAdamBackend())
    losses = []
    for users, items, negs in batches:
        mine = plan.user_owner(users) == rank
        f = lambda x: torch.from_numpy(x[mine])        # noqa: E731
        losses.append(float(model.step(f(users), f(items), f(negs), loss, len(users))))
    BloomAdamBackend().owner_adam_flush(st)
    out = [sc.gather_rows(st.Wu, plan.uchunk, c['U']), sc.gather_rows(st.Wi, st.mchunk, c['M']),
           sc.gather_rows(st.bu.reshape(-1, 1), plan.uchunk, c['U'])]
    return out, st.bi.reshape(-1, 1).numpy().copy(), losses, st.opt.steps_taken


def _dense_adam_steps(params, batches, loss, wd, H):
    P = [p.astype(np.float64) for p in params]
    opt = DenseAdam(LR, wd)
    losses = []
    for users, items, negs in batches:
        r = omf.mf_bloom_step(P[0], P[1], P[2], P[3], users, items, negs, loss, H, 0, np.float64)
        losses.append(float(r['loss']))
        opt(P, [r['dWu'], r['dWi'], r['dbu'], r['dbi']])
    return P, losses


@pytest.mark.parametrize('world', [2, 3])
@pytest.mark.parametrize('loss', ['pointwise', 'bpr', 'hinge'])
@pytest.mark.parametrize('wd', [0.0, 1e-2])
def test_sharded_bloom_adam_step_matches_dense_adam(world, loss, wd):
    """Four Adam steps (a rank without members in the second minibatch and with members in the next,
    user rows no interaction names, a hashed row every rank touches, an item-bias id only the flush moves), then
    the flush, against dense Adam on the concatenated minibatches; the item-bias replicas are bitwise
    equal across ranks."""
    res = sc.run_world(_step_job, world, (loss, wd))
    params, batches = _step_problem()
    ref, ref_losses = _dense_adam_steps(params, batches, loss, wd, STEP['H'])
    got, bi, losses, steps = res[0]
    assert steps == len(SIZES)
    assert_close(np.array(losses), np.array(ref_losses), 1e-5, what='losses')
    for a, b, nm in zip(got + [bi], ref, ('Wu', 'Wi', 'bu', 'bi')):
        _check_adam(a, b, LR, nm)
    for r in range(1, world):
        assert np.array_equal(res[r][1], bi), 'item-bias replica of rank %d differs' % r


# ------------------------------------------------------------------ fit()

FIT = dict(U=19, N=80, D=8, H=2, ratio=0.25, B=16, n=70, n_iter=2, seed=13)


def _fit_net():
    from spotlight_b200.factorization.representations import BilinearNet
    from spotlight_b200.layers import BloomEmbedding
    torch.manual_seed(5)
    net = BilinearNet(FIT['U'], FIT['N'], FIT['D'],
                      item_embedding_layer=BloomEmbedding(FIT['N'], FIT['D'], compression_ratio=FIT['ratio'],
                                                          num_hash_functions=FIT['H']))
    with torch.no_grad():
        net.user_biases.weight.normal_(0, 0.1)
        net.item_biases.weight.normal_(0, 0.1)
    return net


def _fit_data():
    rs = np.random.RandomState(2)
    return rs.randint(0, FIT['U'], FIT['n']).astype(np.int32), rs.randint(1, FIT['N'], FIT['n']).astype(np.int32)


def _opt(name):
    from spotlight_b200 import optim
    return optim.fused_adagrad(lr=0.05) if name == 'adagrad' else optim.fused_adam(lr=LR, weight_decay=1e-3)


def _fit_job(rank, world, dev, loss, opt):
    from spotlight_b200.interactions import Interactions
    from spotlight_b200.sharded import ShardedImplicitFactorizationModel
    users, items = _fit_data()
    rs = np.random.RandomState(FIT['seed'])
    model = ShardedImplicitFactorizationModel(FIT['U'], FIT['N'], rank, world, dev, backend=BloomAdamBackend(),
                                              loss=loss, n_iter=FIT['n_iter'], batch_size=FIT['B'], random_state=rs,
                                              optimizer_func=_opt(opt), representation=_fit_net())
    inter = Interactions(users, items, num_users=FIT['U'], num_items=FIT['N'])
    model.fit(inter)
    model.fit(inter)                                   # resumes the step count and the moments
    net = model.gathered_net()
    tabs = [p.detach().numpy().copy() for p in (net.user_embeddings.weight, net.item_embeddings.embeddings.weight,
                                                net.user_biases.weight)]
    return tabs, model.state.bi.reshape(-1, 1).numpy().copy(), model.epoch_losses, rs.get_state()


def _replay(loss, opt):
    """The reference's stream (ctor draw, then per epoch the permutation and one sample_items per
    minibatch) over both fit() calls, float64, dense Adam or Adagrad on all four tables."""
    users, items = _fit_data()
    net = _fit_net()
    P = [p.detach().numpy().astype(np.float64) for p in (net.user_embeddings.weight,
                                                         net.item_embeddings.embeddings.weight,
                                                         net.user_biases.weight, net.item_biases.weight)]
    epochs, rs = sc.reference_epochs(FIT['seed'], users, items, FIT['N'], FIT['B'], 2 * FIT['n_iter'])
    adam = DenseAdam(LR, 1e-3)
    S = [np.zeros_like(p) for p in P]
    losses = []
    for batches in epochs:
        el = []
        for u, i, n in batches:
            r = omf.mf_bloom_step(P[0], P[1], P[2], P[3], u, i, n, loss, FIT['H'], 0, np.float64)
            el.append(float(r['loss']))
            grads = [r['dWu'], r['dWi'], r['dbu'], r['dbi']]
            if opt == 'adam':
                adam(P, grads)
            else:
                for k, g in enumerate(grads):
                    S[k] += g * g
                    P[k] -= 0.05 * g / (np.sqrt(S[k]) + 1e-10)
        losses.append(np.mean(el))
    return P, losses, rs


@pytest.mark.parametrize('opt', ['adagrad', 'adam'])
@pytest.mark.parametrize('loss', ['pointwise', 'bpr', 'hinge'])
def test_sharded_bloom_fit_matches_reference_stream(loss, opt):
    """Two resumed fit() calls at world 2 (a short last minibatch) against the float64 replay: tables,
    epoch losses, the final RandomState, and item-bias replicas bitwise equal across ranks."""
    res = sc.run_world(_fit_job, 2, (loss, opt))
    ref, ref_losses, rs = _replay(loss, opt)
    tabs, bi, losses, state = res[0]
    assert_close(np.array(losses), np.array(ref_losses), 1e-5, what='epoch losses')
    lr = LR if opt == 'adam' else 0.05
    for a, b, nm in zip(tabs + [bi], ref, ('Wu', 'Wi', 'bu', 'bi')):
        _check_adam(a, b, lr, nm, rtol=1e-4)
    want = rs.get_state()
    assert np.array_equal(state[1], want[1]) and state[2] == want[2]
    assert np.array_equal(res[1][1], bi)


# ------------------------------------------------------------------ selection

def _state(optimizer_func):
    from spotlight_b200.sharded import BloomShardState, ShardPlan
    return BloomShardState(ShardPlan(10, 50, 2), 0, 8, 'cpu', 50, 12, 2, optimizer_func=optimizer_func)


def test_optimizer_selection():
    from spotlight_b200 import optim
    from spotlight_b200.optim import FusedAdam
    st = _state(None)
    assert st.opt is None and st.sWu is not None and (st.lr, st.eps) == (0.05, 1e-10)
    st = _state(optim.fused_adagrad(lr=0.3, eps=1e-6))
    assert st.opt is None and (st.lr, st.eps) == (0.3, 1e-6)
    st = _state(optim.fused_adam(lr=1e-3, weight_decay=1e-2))
    assert isinstance(st.opt, FusedAdam) and st.sWu is None
    lazy = {id(p): s.get('lazy') for p, s in st.opt.state.items()}
    assert lazy == {id(st.Wu): 'pair', id(st.bu2): 'pair', id(st.Wi): 'own', id(st.bi2): 'own'}
    for bad in (optim.fused_adagrad(lr=0.1, weight_decay=1e-3), optim.fused_sgd(lr=0.1),
                lambda params: torch.optim.Adam(params)):
        with pytest.raises(ValueError, match='fused_adagrad without weight decay or optim.fused_adam'):
            _state(bad)


def test_representation_selection():
    from spotlight_b200.factorization.representations import BilinearNet
    from spotlight_b200.layers import BloomEmbedding
    from spotlight_b200.sharded import ShardedImplicitFactorizationModel

    def model(net, **kw):
        return ShardedImplicitFactorizationModel(20, 50, 0, 1, 'cpu', backend=BloomAdamBackend(), representation=net,
                                                 **kw)

    def bloom(n=50, **kw):
        return BloomEmbedding(n, 8, compression_ratio=0.3, num_hash_functions=2, **kw)

    m = model(BilinearNet(20, 50, 8, item_embedding_layer=bloom()))
    assert m.state.M == 15 and m.state.Wu.shape == (20, 8)
    cases = [
        (dict(loss='adaptive_hinge'), BilinearNet(20, 50, 8, item_embedding_layer=bloom()), 'adaptive hinge'),
        (dict(exchange='a2a'), BilinearNet(20, 50, 8, item_embedding_layer=bloom()), 'whole'),
        ({}, BilinearNet(20, 50, 8, user_embedding_layer=BloomEmbedding(20, 8), item_embedding_layer=bloom()),
         'plain user layer'),
        ({}, BilinearNet(20, 50, 8, item_embedding_layer=bloom(), sparse=True), 'dense gradients'),
        ({}, BilinearNet(20, 50, 8, item_embedding_layer=bloom(n=60)), 'item ids'),
        ({}, BilinearNet(20, 50, 8), 'BloomEmbedding'),
        ({}, BilinearNet(20, 50, 8, item_embedding_layer=bloom(padding_idx=None)), 'BloomEmbedding'),
    ]
    for kw, net, msg in cases:
        with pytest.raises(ValueError, match=msg):
            model(net, **kw)
    with pytest.raises(NotImplementedError):            # the layer itself refuses bag=True
        bloom(bag=True)
