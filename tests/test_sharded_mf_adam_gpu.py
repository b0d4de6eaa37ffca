"""NCCL / device tests of sharded factorization training with row-wise lazy-exact Adam.

* The users-only Adam mode of slb_mf_train_step (mf_adam_users_prepass_kernel,
  mf_bwd_*_kernel<.., 1> into dense dWi / dbi, mf_adam_users_kernel), through
  GpuBackend.local_step, against oracle.adam restricted to the user tables, on oracle/mf_adam_cases.py
  cases (t0 = 1 and 1000, rows current, behind, far behind and never touched).
* slb_adam_dense against LazyAdamTable, and the C-ABI rejections of both entries.
* World-1 fit() (world 2 as well when two GPUs are visible) for all four losses, both exchanges and
  exchange='auto' switching between them under fused_adam against the single-GPU fused_adam fit from
  the same seed and weights.
"""

import contextlib
import ctypes
import io
import os
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT, assert_close
from oracle import mf as omf
from oracle import mf_adam_cases as mac
from oracle.adam import LazyAdamTable, mf_terms

sys.path.insert(0, os.path.join(ROOT, 'tests'))
pytestmark = pytest.mark.gpu

import sharded_common as sc                                 # noqa: E402
from test_mf_adam_oracle_gpu import LR, _check_param          # noqa: E402
from test_sharded_seq_adam_cpu import _check_adam             # noqa: E402

DEV = 'cuda:0'


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------ users-only Adam mode

USERS_CASES = [(4, 'pointwise', 1, 0.0, 1000), (8, 'bpr', 1, 0.1, 1), (16, 'hinge', 1, 0.1, 1000),
               (64, 'pointwise', 1, 0.0, 1), (128, 'bpr', 1, 0.1, 1000), (260, 'adaptive_hinge', 2, 0.1, 1000)]


def _user_state(case, wd, t0):
    """A world-1 ShardState under fused_adam at steps taken t0 - 1 with the case's seeded user state,
    and the float64 user tables (Wu, bu) with the same state."""
    from spotlight_b200.optim import fused_adam
    from spotlight_b200.sharded import ShardPlan, ShardState
    state = mac.seed_state(case, t0, seed=case['D'] + t0)
    plan = ShardPlan(case['U'], case['I'], 1)
    st = ShardState(plan, 0, case['D'], DEV, init=[t(case[k]) for k in mac.TABLES],
                    optimizer_func=fused_adam(lr=LR, weight_decay=wd))
    st.opt.advance(t0 - 1)
    for dst, k in (((st.mWu, st.vWu, st.last_u), 0), ((st.mbu, st.vbu, None), 2)):
        m, v, last = state[k]
        dst[0].copy_(t(m).reshape(dst[0].shape))
        dst[1].copy_(t(v).reshape(dst[1].shape))
        if dst[2] is not None:
            dst[2].copy_(t(last))
    tabs = mac.tables(case, LR, wd, state)
    return st, tabs[0], tabs[2]


@pytest.mark.parametrize('D,loss,n,wd,t0', USERS_CASES)
def test_users_only_adam_step(D, loss, n, wd, t0):
    """Three steps of GpuBackend.local_step (the item table as the row cache, norm_batch = 2B): per
    step the loss share, the user rows and their moments against the scheme, last_u exactly, the dense
    item gradient, and rows neither read nor stepped bit-identical.  The case's item tables never
    move (their owners would step them)."""
    from spotlight_b200.sharded import GpuBackend
    case = mac.small_case(D, loss, n, _sms())
    st, Wu, bu = _user_state(case, wd, t0)
    be = GpuBackend(DEV)
    Wi, bi = case['Wi'].astype(np.float64), case['bi'].astype(np.float64).reshape(-1, 1)
    cache_W, cache_b = t(case['Wi']), t(case['bi'].reshape(-1))
    for step, (u, i, j, _) in enumerate(mac.batches(case, 3, seed=t0), t0):
        before = st.Wu.cpu().numpy().copy()
        last_before = Wu.last.copy()
        for tab in (Wu, bu):
            tab.catch_up(u, step - 1)
        ref = mf_terms([Wu.w, Wi, bu.w, bi], u, i, j, loss, case['n_neg'])
        rows = np.flatnonzero(omf.touched(case['U'], ref['terms'][0], ref['terms'][2]))
        Wu.apply(rows, 0.5 * ref['dWu'][rows], step)
        bu.apply(rows, 0.5 * ref['dbu'].reshape(-1, 1)[rows], step)
        B = len(u)
        share, dWi, dbi = be.local_step(st, cache_W, cache_b, case['I'], t(u), t(i), t(j), loss, 2 * B,
                                        case['n_neg'], t=step)
        st.opt.advance(1)
        what = 'step %d' % step
        assert_close(share.item(), 0.5 * ref['loss'], 1e-5, what=what + ' loss')
        assert (st.last_u.cpu().numpy() == Wu.last).all(), what + ' last_u'
        for dev, tab, nm in (((st.Wu, st.mWu, st.vWu), Wu, 'Wu'), ((st.bu2, st.mbu, st.vbu), bu, 'bu')):
            assert_close(dev[1].cpu().numpy().reshape(tab.m.shape), tab.m, 2e-5, atol=1e-12, what=nm + ' exp_avg')
            assert_close(dev[2].cpu().numpy().reshape(tab.v.shape), tab.v, 2e-5, atol=1e-20, what=nm + ' exp_avg_sq')
            _check_param(dev[0], tab, '%s %s' % (what, nm))
        assert_close(dWi.cpu().numpy(), 0.5 * ref['dWi'], 2e-5, atol=1e-9, what=what + ' dWi')
        assert_close(dbi.cpu().numpy(), 0.5 * ref['dbi'].reshape(-1), 2e-5, atol=1e-9, what=what + ' dbi')
        still = Wu.last == last_before
        assert (st.Wu.cpu().numpy()[still] == before[still]).all(), what + ': a row neither read nor stepped moved'
    assert (st.Wi.cpu().numpy() == case['Wi']).all() and (st.last.cpu().numpy() == 0).all()


# ------------------------------------------------------------------ slb_adam_dense

def _dense_case(D, rows, T, wd, seed=0):
    rs = np.random.RandomState(seed + D)
    W = rs.randn(rows, D).astype(np.float32) * 0.3
    b = rs.randn(rows, 1).astype(np.float32) * 0.1
    G = (rs.randn(rows, D) * 1e-2).astype(np.float32)
    gb = (rs.randn(rows, 1) * 1e-2).astype(np.float32)
    G[::5], gb[::5] = 0.0, 0.0                                     # zero-gradient rows still take the step
    group = rs.randint(0, 4, rows)                                 # current, behind, far behind, never touched
    last = np.select([group == 0, group == 1, group == 2], [T - 1, T - 2, rs.randint(1, 20, rows)], 0)
    tabs = []
    for w, g in ((W, G), (b, gb)):
        tab = LazyAdamTable(w, lr=1e-2, weight_decay=wd)
        tab.m = (rs.randn(*w.shape) * 1e-3).astype(np.float32).astype(np.float64)
        tab.v = (rs.uniform(0.25, 1.0, w.shape) * 1e-6).astype(np.float32).astype(np.float64)
        tab.m[group == 3], tab.v[group == 3] = 0.0, 0.0
        tab.last = last.astype(np.int64)
        tabs.append(tab)
    return tabs, G, gb


def _dense_call(tabs, G, gb, T, wd, rows=None):
    from spotlight_b200 import _lib, ops
    from spotlight_b200.optim import FusedAdam
    dev = [[t(x.astype(np.float32)) for x in (tab.w, tab.m, tab.v)] for tab in tabs]
    last = t(tabs[0].last.astype(np.int32))
    sched = FusedAdam([torch.zeros(1)], lr=1e-2).schedule(T, torch.device(DEV))
    g, g_b = t(G), t(gb.reshape(-1))
    n = tabs[0].w.shape[0] if rows is None else rows
    rc = _lib.load().slb_adam_dense(*[ops._ptr(x) for x in dev[0] + dev[1]], ops._ptr(last), ops._ptr(g),
                                    ops._ptr(g_b), n, tabs[0].w.shape[1], ops._ptr(sched), T,
                                    0.9, 0.999, 1.0 - 0.9, 1.0 - 0.999, 1e-8, wd, ops._stream())
    torch.cuda.synchronize()
    return rc, dev, last


@pytest.mark.parametrize('D', [1, 3, 64, 128])
@pytest.mark.parametrize('wd', [0.0, 1e-2])
def test_adam_dense(D, wd):
    """Every row replays its missed steps through T - 1 (rows current, one behind, far behind and never
    touched), then takes step T with its gradient row (every fifth row all zero): the table, its bias,
    their moments against LazyAdamTable, and last = T everywhere."""
    T = 1000
    tabs, G, gb = _dense_case(D, 300, T, wd)
    rc, dev, last = _dense_call(tabs, G, gb, T, wd)
    assert rc == 0
    rows = np.arange(300)
    for tab, g in zip(tabs, (G, gb)):
        tab.catch_up(rows, T - 1)
        tab.apply(rows, g.astype(np.float64), T)
    for (w, m, v), tab, nm in zip(dev, tabs, ('W', 'b')):
        assert_close(m.cpu().numpy(), tab.m, 2e-5, atol=1e-12, what=nm + ' exp_avg')
        assert_close(v.cpu().numpy(), tab.v, 2e-5, atol=1e-20, what=nm + ' exp_avg_sq')
        assert_close(w.cpu().numpy(), tab.w, 2e-6, what=nm)
    assert (last.cpu().numpy() == T).all()


def test_adam_dense_rows_zero_and_rejections():
    """rows = 0 changes nothing; null pointers and bad sizes are rejected with the library's error, and
    so is a users-only Adam step without its user state or with compact gradients."""
    from spotlight_b200 import _lib, ops
    tabs, G, gb = _dense_case(8, 10, 50, 0.0)
    rc, dev, last = _dense_call(tabs, G, gb, 50, 0.0, rows=0)
    assert rc == 0 and (dev[0][0].cpu().numpy() == tabs[0].w.astype(np.float32)).all()
    assert (last.cpu().numpy() == tabs[0].last).all()
    lib = _lib.load()
    x = t(np.zeros((10, 8), np.float32))
    p = ops._ptr(x)
    args = lambda ptr, rows, dim, step: [ptr] + [p] * 6 + [p, p, rows, dim, p, step, 0.9, 0.999, 0.1, 0.001,  # noqa: E731
                                                           1e-8, 0.0, ops._stream()]
    assert lib.slb_adam_dense(*args(None, 10, 8, 5)) != 0 and b'null' in lib.slb_last_error()
    for rows, dim, step in ((-1, 8, 5), (10, 0, 5), (10, 8, 0), (10, 8, 1 << 31)):
        assert lib.slb_adam_dense(*args(p, rows, dim, step)) != 0 and b'bad sizes' in lib.slb_last_error()
    # the users-only mode of slb_mf_train_step
    from spotlight_b200.optim import fused_adam
    from spotlight_b200.sharded import ShardPlan, ShardState
    st = ShardState(ShardPlan(10, 10, 1), 0, 8, DEV, optimizer_func=fused_adam())
    ids = t(np.arange(4, dtype=np.int64))
    a = ops.mf_step_args(st.Wu, st.Wi, st.bu, st.bi, ids, ids, ids, 'bpr', 1)
    a.opt, a.opt_users_only, a.grad_mode = _lib.OPT_ADAM, 1, _lib.GRAD_DENSE
    loss_out = torch.zeros(1, device=DEV)
    a.loss_out = loss_out.data_ptr()
    dW, db = torch.zeros_like(st.Wi), torch.zeros_like(st.bi)
    a.dWi, a.dbi = dW.data_ptr(), db.data_ptr()
    ws = ops.workspace('adam_reject', lib.slb_mf_step_workspace_bytes(4, 1, a.loss, 10, 10), torch.device(DEV))
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    assert lib.slb_mf_train_step(ctypes.byref(a), ops._stream()) != 0       # no user state, no schedule
    assert b'users-only Adam' in lib.slb_last_error()
    a.state_Wu, a.state_bu, a.state2_Wu, a.state2_bu = st.mWu.data_ptr(), st.mbu.data_ptr(), st.vWu.data_ptr(), \
        st.vbu.data_ptr()
    a.last_u, a.adam_sched, a.adam_step = st.last_u.data_ptr(), st.opt.schedule(1, torch.device(DEV)).data_ptr(), 1
    a.grad_mode = _lib.GRAD_COMPACT
    assert lib.slb_mf_train_step(ctypes.byref(a), ops._stream()) != 0       # compact gradients
    a.grad_mode = _lib.GRAD_DENSE
    assert lib.slb_mf_train_step(ctypes.byref(a), ops._stream()) == 0       # the item state may be NULL
    torch.cuda.synchronize()


# ------------------------------------------------------------------ fit() against the single-GPU fit

# n = 14 B + 300: under exchange='auto' the full minibatches take the dense exchange (2 B / world >= I),
# the last one the a2a exchange (2 * 300 / world < I)
FIT = dict(seed=41, U=3000, I=800, D=32, n=14 * 4096 + 300, B=4096, n_iter=2)
FIT_JOBS = [('pointwise', 'a2a'), ('pointwise', 'dense'), ('bpr', 'a2a'), ('bpr', 'dense'), ('bpr', 'auto'),
            ('hinge', 'a2a'), ('hinge', 'dense'), ('adaptive_hinge', 'a2a')]
FIT_OPT = dict(lr=1e-2, weight_decay=1e-3)
WORLDS = [1] + ([2] if torch.cuda.is_available() and torch.cuda.device_count() >= 2 else [])


def _fit_problem():
    rs = np.random.RandomState(8)
    params, _ = sc.make_problem(6, FIT['U'], FIT['I'], FIT['D'], 8, 0)
    params = tuple(p * 0.3 for p in params)
    return params, rs.randint(0, FIT['U'], FIT['n']).astype(np.int32), rs.randint(0, FIT['I'], FIT['n']).astype(np.int32)


def _fit_job(rank, world, dev, loss, exchange):
    from spotlight_b200.interactions import Interactions
    from spotlight_b200.optim import fused_adam
    from spotlight_b200.sharded import ShardedImplicitFactorizationModel
    params, users, items = _fit_problem()
    rs = np.random.RandomState(FIT['seed'])
    model = ShardedImplicitFactorizationModel(
        FIT['U'], FIT['I'], rank, world, dev, loss=loss, embedding_dim=FIT['D'], n_iter=FIT['n_iter'],
        batch_size=FIT['B'], random_state=rs, exchange=exchange, init=[torch.from_numpy(p) for p in params],
        num_negative_samples=4, optimizer_func=fused_adam(**FIT_OPT))
    routes = []
    for name in ('step_a2a', 'step_dense'):          # record the exchange each step takes
        def traced(*args, _f=getattr(model.mf, name), _name=name, **kw):
            routes.append(_name)
            return _f(*args, **kw)
        setattr(model.mf, name, traced)
    model.fit(Interactions(users, items, num_users=FIT['U'], num_items=FIT['I']))
    st = model.state
    lasts = [int(x.min()) for x in (st.last, st.last_u) if x.numel()] + [int(x.max()) for x in (st.last, st.last_u)
                                                                        if x.numel()]
    return (sc.gather_tables(st, model.plan, FIT['U'], FIT['I']), model.epoch_losses, rs.get_state(),
            st.opt.steps_taken, lasts, routes)


def _fit_jobs(rank, world, dev):
    return {job: _fit_job(rank, world, dev, *job) for job in FIT_JOBS}


_RES, _SINGLE = {}, {}


def _results(world):
    if world not in _RES:
        _RES[world] = sc.run_world(_fit_jobs, world, backend='nccl', timeout=900)
    return _RES[world]


def _single_gpu_fit(loss):
    if loss not in _SINGLE:
        from spotlight_b200.factorization.implicit import ImplicitFactorizationModel
        from spotlight_b200.interactions import Interactions
        from spotlight_b200.optim import fused_adam
        params, users, items = _fit_problem()
        inter = Interactions(users, items, num_users=FIT['U'], num_items=FIT['I'])
        rs = np.random.RandomState(FIT['seed'])
        one = ImplicitFactorizationModel(loss=loss, embedding_dim=FIT['D'], n_iter=FIT['n_iter'], batch_size=FIT['B'],
                                         use_cuda=True, random_state=rs, num_negative_samples=4,
                                         optimizer_func=fused_adam(**FIT_OPT))
        one._initialize(inter)
        net = one._net
        with torch.no_grad():
            for prm, val in zip((net.user_embeddings.weight, net.item_embeddings.weight, net.user_biases.weight,
                                 net.item_biases.weight), params):
                prm.copy_(torch.from_numpy(val).to(prm.device).reshape(prm.shape))
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            one.fit(inter, verbose=True)
        losses = [float(line.split('loss')[1]) for line in buf.getvalue().splitlines() if line.startswith('Epoch')]
        tabs = [p.detach().cpu().numpy() for p in (net.user_embeddings.weight, net.item_embeddings.weight,
                                                   net.user_biases.weight, net.item_biases.weight)]
        _SINGLE[loss] = (tabs, losses, rs.get_state(), one._optimizer.steps_taken)
    return _SINGLE[loss]


@pytest.mark.parametrize('world', WORLDS)
@pytest.mark.parametrize('loss,exchange', FIT_JOBS)
def test_sharded_mf_fit_adam_equals_single_gpu_fit(world, loss, exchange):
    """fit() with fused_adam(lr=1e-2, weight_decay=1e-3) through the sharded route (users-only Adam
    step, owner catch-up and Adam, or the whole-shard catch-up and dense Adam step, the flush) against
    ImplicitFactorizationModel(fused_adam) from the same seed and weights: epoch losses, the four
    tables (the dense-Adam tolerances of test_sharded_seq_adam_cpu, in units of lr), the RandomState
    position, the step count and every row current for it.  Adaptive hinge as
    test_sharded_fit_equals_single_gpu_fit checks it: its trajectory is chaotic at the row level."""
    got, losses, state, steps, lasts, routes = _results(world)[0][loss, exchange]
    if exchange == 'auto':                          # the short last minibatch switched the route
        assert routes == (['step_dense'] * (FIT['n'] // FIT['B']) + ['step_a2a']) * FIT['n_iter'], routes
    ref, want_losses, want_state, want_steps = _single_gpu_fit(loss)
    loss_tol = 1e-4 if (loss == 'adaptive_hinge' and world > 1) else 2e-5
    assert_close(np.array(losses), np.array(want_losses), loss_tol, what='epoch losses')
    for a, b, nm in zip(got, ref, ('Wu', 'Wi', 'bu', 'bi')):
        if loss == 'adaptive_hinge':
            floor = {'Wu': 0.8, 'Wi': 0.3}.get(nm)
            assert np.isfinite(a).all()
            if floor is not None:
                assert np.corrcoef(a.reshape(-1), b.reshape(-1))[0, 1] > floor, nm
        else:
            _check_adam(a, b.reshape(a.shape).astype(np.float64), FIT_OPT['lr'], nm, rtol=1e-4)
    assert np.array_equal(state[1], want_state[1]) and state[2] == want_state[2]
    assert steps == want_steps and set(lasts) == {steps}
