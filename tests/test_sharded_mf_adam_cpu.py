"""World-size-2 and 3 gloo tests of sharded factorization training with row-wise lazy-exact Adam
(``optimizer_func=fused_adam``) on CPU, with a NumPy backend that runs the users-only local step
and the owner-side Adam in float64 (oracle.adam.LazyAdamTable): ShardedMF steps under pointwise,
bpr and hinge over both exchanges and a mix of them against the single-process lazy scheme
(oracle.adam.lazy_mf_step) on the concatenated minibatch, and
ShardedImplicitFactorizationModel.fit() for all four losses against a float64 dense-Adam replay of
the reference's stream.  Also the optimizer selection and the resource usage of the new kernels."""

import os
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT, assert_close

sys.path.insert(0, os.path.join(ROOT, 'tests'))

import sharded_common as sc                                  # noqa: E402
from oracle import mf as omf                                 # noqa: E402
from oracle.adam import LazyAdamTable, lazy_mf_step, mf_terms  # noqa: E402
from test_sharded_seq_adam_cpu import DenseAdam, _check_adam   # noqa: E402

LR = 1e-2


class AdamMFBackend(sc.NumpyBackend):
    """NumpyBackend plus lazy-exact Adam in float64 on the float32 shards and state tensors of
    ShardState: the users-only local step, the owner-side catch-up and update, the whole-shard
    catch-up and dense step, and the flush."""

    @staticmethod
    def _pair(st, users):
        if users:
            return (st.Wu, st.mWu, st.vWu), (st.bu2, st.mbu, st.vbu), st.last_u
        return (st.Wi, st.mWi, st.vWi), (st.bi2, st.mbi, st.vbi), st.last

    def _tables(self, st, users):
        hp = st.opt.fused_hparams()
        kw = dict(lr=hp['lr'], betas=(hp['beta1'], hp['beta2']), eps=hp['eps'], weight_decay=hp['weight_decay'])
        emb, bias, last = self._pair(st, users)
        tabs = []
        for w, m, v in (emb, bias):
            tab = LazyAdamTable(w.numpy(), **kw)
            tab.m = m.numpy().astype(np.float64).reshape(tab.w.shape)
            tab.v = v.numpy().astype(np.float64).reshape(tab.w.shape)
            tab.last = last.numpy().astype(np.int64)                # the row and its bias share `last`
            tabs.append(tab)
        return tabs

    def _store(self, st, users, tabs):
        emb, bias, last = self._pair(st, users)
        for tab, tensors in zip(tabs, (emb, bias)):
            for dst, src in zip(tensors, (tab.w, tab.m, tab.v)):
                dst.copy_(torch.from_numpy(src.reshape(dst.shape).astype(np.float32)))
        assert np.array_equal(tabs[0].last, tabs[1].last)
        last.copy_(torch.from_numpy(tabs[0].last.astype(np.int32)))

    def local_step(self, st, cache_rows, cache_bias, n_cache, users_local, pos_idx, neg_idx, loss,
                   global_batch, n_neg=1, t=None):
        if t is None:
            return super(AdamMFBackend, self).local_step(st, cache_rows, cache_bias, n_cache, users_local, pos_idx,
                                                         neg_idx, loss, global_batch, n_neg)
        u = users_local.numpy()
        tabs = self._tables(st, True)
        for tab in tabs:                                         # the prepass: referenced user rows
            tab.catch_up(u, t - 1)
        P = [tabs[0].w, cache_rows.numpy().astype(np.float64), tabs[1].w,
             cache_bias.numpy().astype(np.float64).reshape(-1, 1)]
        ref = mf_terms(P, u, pos_idx.numpy(), neg_idx.numpy(), loss, n_neg)
        scale = len(u) / float(global_batch)
        rows = np.flatnonzero(omf.touched(P[0].shape[0], ref['terms'][0], ref['terms'][2]))
        tabs[0].apply(rows, ref['dWu'][rows] * scale, t)
        tabs[1].apply(rows, ref['dbu'].reshape(-1, 1)[rows] * scale, t)
        self._store(st, True, tabs)
        return (torch.tensor(float(ref['loss']) * scale, dtype=torch.float32),
                torch.from_numpy((ref['dWi'] * scale).astype(np.float32))[:n_cache],
                torch.from_numpy((ref['dbi'].reshape(-1) * scale).astype(np.float32))[:n_cache])

    def owner_adam_catch_up(self, st, local_ids, t):
        ids = local_ids.numpy()
        if len(ids):
            tabs = self._tables(st, False)
            for tab in tabs:
                tab.catch_up(ids, t - 1)
            self._store(st, False, tabs)

    def owner_adam_update(self, st, local_ids, g_rows, g_bias, t):
        ids = local_ids.numpy()
        if not len(ids):
            return
        rows = np.unique(ids)
        slot = np.searchsorted(rows, ids)
        dW = np.zeros((len(rows), st.Wi.shape[1]))
        db = np.zeros((len(rows), 1))
        np.add.at(dW, slot, g_rows.numpy().astype(np.float64))           # position (= rank) order
        np.add.at(db, slot, g_bias.numpy().reshape(-1, 1).astype(np.float64))
        tabs = self._tables(st, False)
        tabs[0].apply(rows, dW, t)
        tabs[1].apply(rows, db, t)
        self._store(st, False, tabs)

    def _flush(self, st, users, upto):
        if upto >= 1 and self._pair(st, users)[0][0].shape[0]:
            tabs = self._tables(st, users)
            for tab in tabs:
                tab.flush(upto)
            self._store(st, users, tabs)

    def owner_adam_catch_up_shard(self, st, upto):
        self._flush(st, False, upto)

    def user_adam_catch_up(self, st, user_ids, t):
        tabs = self._tables(st, True)
        for tab in tabs:
            tab.catch_up(user_ids.numpy(), t - 1)
        self._store(st, True, tabs)

    def adam_dense(self, st, users, g, g_bias, t):
        tabs = self._tables(st, users)
        rows = np.arange(tabs[0].w.shape[0])
        for tab, grad in zip(tabs, (g.numpy(), g_bias.numpy().reshape(-1, 1))):
            tab.catch_up(rows, t - 1)
            tab.apply(rows, grad.astype(np.float64), t)
        self._store(st, users, tabs)

    def owner_adam_flush(self, st):
        for users in (True, False):
            self._flush(st, users, st.opt.steps_taken)


# ------------------------------------------------------------------ ShardedMF steps

STEP = dict(seed=31, U=23, I=41, D=8)
SIZES = (12, 3, 10, 2)       # minibatch sizes; the second holds rank 0's users only
SHARED = 5                   # an item every rank with members requests
ROUTES = {'a2a': ('a2a',) * 4, 'dense': ('dense',) * 4, 'mix': ('a2a', 'dense', 'a2a', 'a2a')}
N_ADA = 3                    # adaptive hinge: negatives per interaction


def step_batches(U, I, n_neg=1):
    """Items and negatives come from [0, 14) and [28, I): [14, 28) -- the whole item range of rank 1
    at world 3 -- is never drawn, so only the flush moves those rows.  ``n_neg`` negatives per
    interaction, flat: the n-block of interaction b is negs[b * n_neg:(b + 1) * n_neg]."""
    rs = np.random.RandomState(STEP['seed'] + 2)
    pool = np.r_[0:14, 28:I] if I > 28 else np.arange(I)
    out = []
    for k, B in enumerate(SIZES):
        users = rs.randint(0, min(U, 3) if k == 1 else U, B).astype(np.int64)
        items = rs.choice(pool, B).astype(np.int64)
        items[::3] = min(SHARED, I - 1)
        out.append((users, items, rs.choice(pool, B * n_neg).astype(np.int64)))
    return out


def step_params(U, I):
    return [p.astype(np.float32) for p in sc.make_margin_params(STEP['seed'], U, I, STEP['D'])]


def lazy_trajectory(U, I, loss, wd):
    """Single process: the float64 lazy scheme on the whole minibatches, then the flush."""
    kw = dict(lr=LR, weight_decay=wd)
    tabs = [LazyAdamTable(p, **kw) for p in step_params(U, I)]
    losses = []
    n_neg = N_ADA if loss == 'adaptive_hinge' else 1
    for t, (users, items, negs) in enumerate(step_batches(U, I, n_neg), 1):
        losses.append(float(lazy_mf_step(tabs, users, items, negs, loss, t, n_neg)['loss']))
    for tab in tabs:
        tab.flush(len(SIZES))
    return [tab.w for tab in tabs], losses


STEP_JOBS = [(loss, route, wd, 23, 41) for loss in ('pointwise', 'bpr', 'hinge') for route in ROUTES
             for wd in (0.0, 1e-2)]
STEP_JOBS += [('adaptive_hinge', 'adaptive', wd, 23, 41) for wd in (0.0, 1e-2)]
STEP_JOBS += [('bpr', 'mix', 1e-2, 2, 4),     # at world 3: rank 2 owns no users and an empty item range
              ('adaptive_hinge', 'adaptive', 1e-2, 2, 4)]


def _step_job(rank, world, loss, route, wd, U, I):
    from spotlight_b200.optim import fused_adam
    from spotlight_b200.sharded import ShardedMF, ShardPlan, ShardState
    plan = ShardPlan(U, I, world)
    st = ShardState(plan, rank, STEP['D'], 'cpu', init=[torch.from_numpy(p) for p in step_params(U, I)],
                    optimizer_func=fused_adam(lr=LR, weight_decay=wd))
    be = AdamMFBackend()
    model = ShardedMF(plan, st, rank, be)
    losses = []
    if loss == 'adaptive_hinge':
        # ShardedMF.step_adaptive with the reference's pairing: a member's n-block of negatives, its
        # position in the minibatch and the minibatch's users
        for users, items, negs in step_batches(U, I, N_ADA):
            mine = plan.user_owner(users) == rank
            block = negs.reshape(len(users), N_ADA)[mine].reshape(-1)
            losses.append(float(model.step_adaptive(
                torch.from_numpy(users[mine]), torch.from_numpy(items[mine]), torch.from_numpy(block),
                torch.from_numpy(np.flatnonzero(mine)), torch.from_numpy(users), N_ADA)))
        be.owner_adam_flush(st)
        return (sc.gather_tables(st, plan, U, I), losses, st.last.numpy().copy(), st.last_u.numpy().copy(),
                st.opt.steps_taken)
    for (users, items, negs), exchange in zip(step_batches(U, I), ROUTES[route]):
        mine = plan.user_owner(users) == rank
        t = lambda x: torch.from_numpy(x[mine])          # noqa: E731
        losses.append(float(model.step(t(users), t(items), t(negs), loss, len(users), exchange)))
    be.owner_adam_flush(st)
    return (sc.gather_tables(st, plan, U, I), losses, st.last.numpy().copy(), st.last_u.numpy().copy(),
            st.opt.steps_taken)


def _step_jobs(rank, world, dev):
    return {job: _step_job(rank, world, *job) for job in STEP_JOBS}


_CACHE = {}


def _step_results(world):
    if world not in _CACHE:
        _CACHE[world] = sc.run_world(_step_jobs, world)
    return _CACHE[world]


@pytest.mark.parametrize('world', [2, 3])
@pytest.mark.parametrize('loss,route,wd,U,I', STEP_JOBS)
def test_sharded_mf_adam_step_matches_lazy_scheme(world, loss, route, wd, U, I):
    """Four steps with minibatches of 12, 3, 10 and 2 interactions (the second holds rank 0's users
    only, the last leaves a rank without members), an item a third of every minibatch uses (requested
    by every rank with members) and an item range no minibatch draws, over the a2a exchange, the
    dense one or a2a -> dense -> a2a, or ShardedMF.step_adaptive with three negatives per interaction
    (after the second minibatch the other ranks' user shards are a step behind when they are next
    scored and stepped); after the flush the gathered tables equal the float64 lazy
    scheme on the whole minibatches, and every row of every rank is current for the step count."""
    if I == 4 and world != 3:
        pytest.skip('the empty user and item ranges arise at world 3')
    res = _step_results(world)
    got, losses = res[0][loss, route, wd, U, I][:2]
    ref, ref_losses = lazy_trajectory(U, I, loss, wd)
    assert_close(np.array(losses), np.array(ref_losses), 1e-5, what='losses')
    for a, b, nm in zip(got, ref, ('Wu', 'Wi', 'bu', 'bi')):
        _check_adam(a, b, LR, nm)
    for r in range(world):
        _, rl, last, last_u, steps = res[r][loss, route, wd, U, I]
        assert rl == losses and steps == len(SIZES)
        assert (last == steps).all() and (last_u == steps).all()
    if I == 4:
        assert res[2][loss, route, wd, U, I][3].size == 0           # rank 2 owns no users
    if I == 41 and wd > 0:
        assert not np.array_equal(got[1][14:28], step_params(U, I)[1][14:28])    # moved by the flush alone


# ------------------------------------------------------------------ ShardedImplicitFactorizationModel.fit

FIT = dict(seed=17, U=30, I=25, D=8, n=150, B=32, n_iter=2)
# 'auto' at world 2: the full minibatches of 32 take the dense exchange (2 * 16 >= 25 items), the last
# one of 22 the a2a exchange
FIT_JOBS = [('pointwise', 'a2a'), ('bpr', 'dense'), ('bpr', 'auto'), ('hinge', 'a2a'), ('adaptive_hinge', 'a2a')]
WD = 1e-3


def _fit_problem():
    params = [p.astype(np.float32) for p in sc.make_margin_params(FIT['seed'], FIT['U'], FIT['I'], FIT['D'])]
    rs = np.random.RandomState(FIT['seed'] + 1)
    users = rs.randint(0, FIT['U'], FIT['n']).astype(np.int32)
    items = rs.randint(0, FIT['I'], FIT['n']).astype(np.int32)
    return params, users, items


def _fit_job(rank, world, loss, exchange, splits):
    from spotlight_b200.interactions import Interactions
    from spotlight_b200.optim import fused_adam
    from spotlight_b200.sharded import ShardedImplicitFactorizationModel
    params, users, items = _fit_problem()
    rs = np.random.RandomState(FIT['seed'])
    model = ShardedImplicitFactorizationModel(
        FIT['U'], FIT['I'], rank, world, 'cpu', backend=AdamMFBackend(), loss=loss, embedding_dim=FIT['D'],
        n_iter=FIT['n_iter'] // splits, batch_size=FIT['B'], random_state=rs, exchange=exchange,
        init=[torch.from_numpy(p) for p in params], num_negative_samples=3,
        optimizer_func=fused_adam(lr=LR, weight_decay=WD))
    routes = []
    for name in ('step_a2a', 'step_dense'):          # record the exchange each step takes
        def traced(*args, _f=getattr(model.mf, name), _name=name, **kw):
            routes.append(_name)
            return _f(*args, **kw)
        setattr(model.mf, name, traced)
    inter = Interactions(users, items, num_users=FIT['U'], num_items=FIT['I'])
    for _ in range(splits):
        model.fit(inter)
    return (sc.gather_tables(model.state, model.plan, FIT['U'], FIT['I']), model.epoch_losses, rs.get_state(),
            model.state.opt.steps_taken, routes)


def _fit_jobs(rank, world, dev):
    return {(loss, ex, splits): _fit_job(rank, world, loss, ex, splits) for loss, ex in FIT_JOBS for splits in (1, 2)}


_FIT = {}


def _replay(loss, n_neg, store=None):
    """The single-process fit(): reference_epochs' minibatches stepped whole through the float64
    oracle, and dense Adam (weight decay included) on all four tables."""
    params, users, items = _fit_problem()
    epochs, rs = sc.reference_epochs(FIT['seed'], users, items, FIT['I'], FIT['B'], FIT['n_iter'], n_neg)
    P = [p.astype(np.float64) for p in params]
    adam = DenseAdam(LR, WD)
    epoch_losses = []
    for batches in epochs:
        losses = []
        for u, i, ng in batches:
            r = omf.mf_step(P[0], P[1], P[2], P[3], u, i, ng, loss, n_neg, np.float64)
            losses.append(float(r['loss']))
            adam(P, [r['dWu'], r['dWi'], r['dbu'], r['dbi']], store=store)
        epoch_losses.append(float(np.mean(losses)))
    return P, epoch_losses, rs, adam.t


@pytest.mark.parametrize('loss,exchange', FIT_JOBS)
def test_sharded_mf_fit_adam_is_the_single_process_fit(loss, exchange):
    """fit() at world 2 with fused_adam(weight_decay=1e-3) over two epochs of 150 interactions in
    minibatches of 32 (the last has 22) against the single-process replay of the reference's stream
    with dense float64 Adam; and two fit(n_iter=1) calls, which resume the step count, the moments
    and `last`.  Under exchange='auto' the full minibatches take the dense exchange and the short last one
    the a2a exchange.  Epoch losses, the four tables, the step count and every rank's final RandomState."""
    n_neg = 3 if loss == 'adaptive_hinge' else 1
    # float32 parameter storage for adaptive hinge, whose argmax over negatives turns the gap between
    # float64 and float32 storage into different active terms (test_sharded_seq_adam_cpu)
    store = np.float32 if loss == 'adaptive_hinge' else None
    if not _FIT:
        _FIT.update(sc.run_world(_fit_jobs, 2))
    ref, ref_losses, rs, steps = _replay(loss, n_neg, store)
    want = rs.get_state()
    for splits in (1, 2):
        for r in range(2):
            got, losses, state, taken, routes = _FIT[r][loss, exchange, splits]
            if exchange == 'auto':                  # a short last minibatch switched the route
                per_epoch = ['step_dense'] * (FIT['n'] // FIT['B']) + ['step_a2a']
                assert routes == per_epoch * FIT['n_iter'], routes
            assert_close(np.array(losses), np.array(ref_losses), 1e-5, what='epoch losses')
            for a, b, nm in zip(got, ref, ('Wu', 'Wi', 'bu', 'bi')):
                _check_adam(a, b.reshape(a.shape), LR, nm)
            assert np.array_equal(state[1], want[1]) and state[2] == want[2]
            assert taken == steps == FIT['n_iter'] * -(-FIT['n'] // FIT['B'])


# ------------------------------------------------------------------ optimizer selection

def test_sharded_mf_model_optimizer_selection():
    """None keeps the row-wise Adagrad state at learning_rate; fused_adagrad without weight decay is
    Adagrad with its hyper-parameters; fused_adam builds a FusedAdam over the two (table, bias view)
    pairs -- the item pair alone on a rank that owns no users; torch.optim.Adam, fused_sgd and
    fused_adagrad with weight decay are rejected."""
    from spotlight_b200.optim import FusedAdam, fused_adagrad, fused_adam, fused_sgd
    from spotlight_b200.sharded import ShardedImplicitFactorizationModel

    def make(func, U=12, rank=0, world=1):
        return ShardedImplicitFactorizationModel(U, 20, rank, world, 'cpu', backend=AdamMFBackend(), embedding_dim=8,
                                                 learning_rate=0.03, optimizer_func=func)

    st = make(None).state
    assert st.opt is None and (st.lr, st.eps) == (0.03, 1e-10)
    assert st.sWu.shape == st.Wu.shape and st.sbi.shape == st.bi.shape and not st.sWi.any()
    st = make(fused_adagrad(lr=0.2, eps=1e-6)).state
    assert st.opt is None and (st.lr, st.eps) == (0.2, 1e-6) and st.sWi.shape == st.Wi.shape
    st = make(fused_adam(lr=1e-3, weight_decay=1e-4)).state
    assert isinstance(st.opt, FusedAdam) and st.sWu is None and st.sWi is None
    params = st.opt.param_groups[0]['params']
    assert len(params) == 4 and params[0] is st.Wu and params[1] is st.bu2 and params[2] is st.Wi
    assert params[3] is st.bi2 and st.bi2.data_ptr() == st.bi.data_ptr() and st.bu2.shape == (12, 1)
    assert st.mWu.shape == st.Wu.shape and st.last_u.shape == (12,) and st.mbi.shape == (20, 1)
    assert st.last.shape == (20,) and not st.last.any()
    st = make(fused_adam(), U=2, rank=2, world=3).state           # no users on rank 2
    assert st.Wu.shape[0] == 0 and st.opt.param_groups[0]['params'] == [st.Wi, st.bi2]
    for func in (lambda p: torch.optim.Adam(p, lr=1e-3), fused_sgd(lr=0.1), fused_adagrad(lr=0.1, weight_decay=1e-3)):
        with pytest.raises(ValueError, match='fused_adam'):
            make(func)


# ------------------------------------------------------------------ resource usage

def test_mf_adam_shard_kernels_do_not_spill():
    """Every instantiation of the users-only Adam prepass and step and of the dense Adam step (lanes
    per row 1 .. 32) has no stack frame and no local memory in the built library."""
    from test_mf_resource_usage_cpu import _find, _usage
    usage = _usage()
    for name in ('mf_adam_users_prepass_kernel', 'mf_adam_users_kernel', 'adam_dense_kernel'):
        for lpr in (1, 2, 4, 8, 16, 32):
            r = _find(usage, '%d%sILi%dEE' % (len(name), name, lpr))
            assert r['STACK'] == 0 and r['LOCAL'] == 0, '%s<%d> spills: %s' % (name, lpr, r)
