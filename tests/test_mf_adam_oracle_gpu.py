"""Lazy-exact Adam on the first-generation MF step -- the default optimizer of
ImplicitFactorizationModel() and ExplicitFactorizationModel() -- against the float64 scheme of
oracle/adam.py (lazy_mf_step, LazyAdamTable).

The step runs through the production route, model._fit_epoch_pipeline: mf_adam_prepass_kernel<L>,
the forward (mf_fwd_tile_kernel, mf_fwd_kernel<L> for adaptive hinge), the segment index, the mode-0
compact backward (mf_bwd_tile_kernel<L, 0, TI, EX>, mf_bwd_long_kernel<L, 0> for hot rows) and
mf_adam_apply_kernel<L>; fit() ends with adam_flush_kernel<L>.  Cases come from
oracle/mf_adam_cases.py: every member-list length class, hot rows, Adam state at a start step t0 of 1
or 1000 with rows current, one step behind, far behind and never touched.

Tolerances as tests/test_mf_bloom_adam_gpu.py: the loss at 1e-5, `last` exactly, the moments at 2e-5
of their scale, the parameters at 5 % of one step where the first moment is above 1e-3 of its
maximum, half a step where it is between 1e-5 and 1e-3 of it, within one step's bound elsewhere
(m / sqrt(v) turns last-bit gradient differences on near-zero components into fractions of a step).
"""

import os
import re

import numpy as np
import pytest
import torch

from conftest import assert_close
from oracle import mf_adam_cases as mac
from oracle.adam import LazyAdamTable, lazy_mf_step

pytestmark = pytest.mark.gpu

LR = 1e-3
STEPS = 4
TABLES = mac.TABLES
DIMS = mac.DIMS


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to('cuda:0')


def _check_param(dev, tab, what):
    w, m = dev.detach().cpu().numpy().astype(np.float64).reshape(tab.w.shape), tab.m
    scale = np.abs(m).max()
    quiet = np.abs(m) < 1e-3 * scale
    noise = np.abs(m) < 1e-5 * scale
    err = np.abs(w - tab.w)
    tol = 2e-6 * np.abs(tab.w).max()
    assert err[~quiet].max(initial=0.0) <= 0.05 * LR + tol, '%s: %.3e' % (what, err[~quiet].max())
    assert err[quiet & ~noise].max(initial=0.0) <= 0.5 * LR + tol, '%s (small moments): %.3e' % (
        what, err[quiet & ~noise].max(initial=0.0))
    assert err.max() <= 2.1 * LR, '%s moved by more than an Adam step' % what
    return err[~quiet].max(initial=0.0)


def _model(case, wd, t0, state):
    """A default-optimizer model holding the case's tables, with FusedAdam at steps taken t0 - 1 and
    the seeded state; returns (model, params, states)."""
    from spotlight_b200.factorization.explicit import ExplicitFactorizationModel
    from spotlight_b200.factorization.implicit import ImplicitFactorizationModel
    from spotlight_b200.interactions import Interactions
    from spotlight_b200.optim import FusedAdam
    kw = dict(embedding_dim=case['D'], batch_size=len(case['users']), l2=wd, learning_rate=LR, use_cuda=True,
              random_state=np.random.RandomState(0))
    if case['loss'] in mac.EXPLICIT:
        m = ExplicitFactorizationModel(loss=case['loss'], **kw)
    else:
        m = ImplicitFactorizationModel(loss=case['loss'], num_negative_samples=case['n_neg'], **kw)
    m._initialize(Interactions(np.zeros(1, np.int32), np.zeros(1, np.int32), num_users=case['U'],
                               num_items=case['I']))
    net, opt = m._net, m._optimizer
    assert isinstance(opt, FusedAdam) and m._route() == 'epoch'
    P = (net.user_embeddings.weight, net.item_embeddings.weight, net.user_biases.weight, net.item_biases.weight)
    opt.advance(t0 - 1)
    S = [opt.fused_states(p) for p in P]
    with torch.no_grad():
        for p, k in zip(P, TABLES):
            p.copy_(t(case[k]).reshape(p.shape))
        for (m_, v_, last), (sm, sv, sl) in zip(S, state):
            m_.copy_(t(sm).reshape(m_.shape))
            v_.copy_(t(sv).reshape(v_.shape))
            last.copy_(t(sl))
    return m, P, S


def _step(model, u, i, j, r):
    """One optimizer step through the epoch pipeline (batch_size = the batch)."""
    model._batch_size = len(u)
    third = t(r) if j is None else t(j)
    return model._fit_epoch_pipeline(t(u), t(i), third)


def _lasts(S):
    """The device `last` of each of the four tables: a bias has its embedding's."""
    lu, li = S[0][2].cpu().numpy(), S[1][2].cpu().numpy()
    return lu, li, lu, li


def _check_state(P, S, tabs, what):
    lasts = _lasts(S)
    worst = 0.0
    for k, (tab, p, (m, v, _), nm) in enumerate(zip(tabs, P, S, TABLES)):
        assert (lasts[k] == tab.last).all(), '%s %s last: %d rows differ' % (what, nm, (lasts[k] != tab.last).sum())
        # the floors are ~1e-7 of a moment: bpr's user-bias gradient gp + gn is 0 in float64, fp32 leaves
        # a residue of ~1e-13 (measured 4.5e-14 in exp_avg)
        assert_close(m.cpu().numpy().reshape(tab.m.shape), tab.m, 2e-5, atol=1e-12, what='%s %s exp_avg' % (what, nm))
        assert_close(v.cpu().numpy().reshape(tab.v.shape), tab.v, 2e-5, atol=1e-20, what='%s %s exp_avg_sq' % (what, nm))
        worst = max(worst, _check_param(p, tab, '%s %s' % (what, nm)))
    return worst


def run_steps(case, wd, t0, record=None):
    """STEPS consecutive steps from t0 against the scheme, every check after every step, then fit()'s
    flush (adam_flush_kernel) against the scheme's."""
    state = mac.seed_state(case, t0, seed=case['D'] + t0)
    model, P, S = _model(case, wd, t0, state)
    tabs = mac.tables(case, LR, wd, state)
    worst, read_only = 0.0, 0
    for step, (u, i, j, r) in enumerate(mac.batches(case, STEPS, seed=t0), t0):
        before = [p.detach().cpu().numpy().copy() for p in P]
        last_before = [tab.last.copy() for tab in tabs]
        ref = lazy_mf_step(tabs, u, i, j, case['loss'], step, case['n_neg'], r)
        loss = _step(model, u, i, j, r)
        what = 'step %d' % step
        assert_close(loss, ref['loss'], 1e-5, what=what + ' loss')
        worst = max(worst, _check_state(P, S, tabs, what))
        for k, (tab, nm) in enumerate(zip(tabs, TABLES)):
            still = tab.last == last_before[k]
            now = P[k].detach().cpu().numpy()
            assert (now[still] == before[k][still]).all(), '%s %s: a row neither read nor stepped changed' % (what, nm)
        refs = (u, i if j is None else np.r_[i, j])
        for side, touched in enumerate((ref['touched_u'], ref['touched_i'])):
            rows = np.setdiff1d(refs[side], np.flatnonzero(touched))
            assert (_lasts(S)[side][rows] == step - 1).all(), '%s: a row read but not stepped is not at t - 1' % what
            read_only += len(rows)
    assert any((tab.last < t0 + STEPS - 2).any() for tab in tabs), 'no row missed several steps'
    if case['loss'] in ('hinge', 'adaptive_hinge'):
        assert read_only > 0, 'no row was read without being stepped'
    opt = model._optimizer
    assert opt.steps_taken == t0 - 1 + STEPS
    opt.flush()
    for tab in tabs:
        tab.flush(opt.steps_taken)
    worst = max(worst, _check_state(P, S, tabs, 'flushed'))
    assert all((last == opt.steps_taken).all() for last in _lasts(S))
    if record is not None:
        record('param_err_over_lr', worst / LR)


# ------------------------------------------------------------------ matrix
# oracle/mf_adam_cases.py: every D twice with small batches (8-interaction forward tiles, 8-segment
# backward tiles), the losses cycling, wd and t0 alternating; then large batches (2B above the backward
# threshold: 32-segment tiles) and one above the forward threshold (32-interaction forward tiles).
SMALL, LARGE = mac.SMALL, mac.LARGE


def _ids(e):
    return '%d-%s%d-wd%g-t%d' % e


@pytest.mark.parametrize('D,loss,n,wd,t0', SMALL, ids=[_ids(e) for e in SMALL])
def test_small_batch(D, loss, n, wd, t0, record_property):
    case = mac.small_case(D, loss, n, sms())
    assert 2 * len(case['users']) < mac.bwd_small_limit(sms())
    run_steps(case, wd, t0, record_property)


@pytest.mark.parametrize('D,loss,n,wd,t0', LARGE, ids=[_ids(e) for e in LARGE])
def test_large_batch(D, loss, n, wd, t0, record_property):
    case = mac.large_case(D, loss, n, sms())
    assert 2 * len(case['users']) >= mac.bwd_small_limit(sms())
    assert len(case['users']) < mac.fwd_small_limit(sms())
    run_steps(case, wd, t0, record_property)


def test_large_forward_tiles(record_property):
    """B above the forward-tile threshold: mf_fwd_tile_kernel with 32-interaction tiles."""
    case = mac.make_case(16, mac.fwd_small_limit(sms()) + 1001, 'bpr', 1, seed=29, sms=sms())
    run_steps(case, 0.1, 1000, record_property)


# ------------------------------------------------------------------ the epoch pipeline
EPOCH = [(32, 'bpr', 1, 0.1, 1000), (24, 'adaptive_hinge', 5, 0.0, 1000), (12, 'poisson', 1, 0.1, 1)]


@pytest.mark.parametrize('D,loss,n,wd,t0', EPOCH, ids=[_ids(e) for e in EPOCH])
def test_epoch_equals_single_steps(D, loss, n, wd, t0):
    """One slb_mf_fit_epoch call over n = k B + r interactions (a short last batch; step k takes
    adam_step + k) equals k + 1 single-step calls bit for bit, and the scheme."""
    case = mac.make_case(D, 3001 + D, loss, n, seed=D + 3, sms=sms())
    state = mac.seed_state(case, t0, seed=D)
    Bs = 700
    N = len(case['users'])
    k, r = divmod(N, Bs)
    assert k >= 3 and r > 0
    neg = None if case['negs'] is None else case['negs'].reshape(case['n_neg'], N)
    batches = []
    for lo in range(0, N, Bs):
        sl = slice(lo, min(N, lo + Bs))
        batches.append((case['users'][sl], case['items'][sl], None if neg is None else neg[:, sl].reshape(-1),
                        None if case['negs'] is not None else case['ratings'][sl]))
    whole, P1, S1 = _model(case, wd, t0, state)
    whole._batch_size = Bs
    if neg is None:
        whole._fit_epoch_pipeline(t(case['users']), t(case['items']), t(case['ratings']))
    else:
        # the epoch's negatives as the pipeline takes them: batch by batch, each in its (n, B') layout
        whole._fit_epoch_pipeline(t(case['users']), t(case['items']), t(np.concatenate([b[2] for b in batches])))
    single, P2, S2 = _model(case, wd, t0, state)
    for u, i, j, rr in batches:
        _step(single, u, i, j, rr)
    assert whole._optimizer.steps_taken == single._optimizer.steps_taken == t0 - 1 + k + 1
    for x, y, nm in zip(P1, P2, TABLES):
        assert torch.equal(x, y), nm
    for a, b in zip(S1, S2):
        for x, y in zip(a, b):
            assert torch.equal(x, y)
    tabs = mac.tables(case, LR, wd, state)
    for step, (u, i, j, rr) in enumerate(batches, t0):
        lazy_mf_step(tabs, u, i, j, loss, step, case['n_neg'], rr)
    _check_state(P1, S1, tabs, 'epoch')


# ------------------------------------------------------------------ flush
# fp32 against float64 over catch-ups of 1 .. 2000 steps, measured on an H100 SXM (700 W power limit),
# largest over D = 4, 24, 260 and wd = 0, 1e-2, relative to the table's scale: on elements the float64
# flush leaves at least ten steps (10 lr) from 0, w 1.2e-6, exp_avg 2.2e-6, exp_avg_sq 2.0e-5 (v is
# multiplied by beta2 in fp32 at every replayed step).  With weight decay, Adam's normalised step walks
# many elements to 0, where they oscillate by about one step; there fp32 and float64 fall out of phase:
# w up to 0.58 lr apart, exp_avg 3.7e-5 of its scale.
FLUSH_RTOL = {'w': 2e-5, 'exp_avg': 2e-5, 'exp_avg_sq': 1e-4}
NEAR_ZERO_RTOL = {'w': 1.0, 'exp_avg': 1e-3, 'exp_avg_sq': 1e-4}       # w: in units of lr, one step


def _flush_case(D, wd, T=2000, rows=3000, seed=0):
    rs = np.random.RandomState(seed)
    W = rs.randn(rows, D) * 0.3
    b = rs.randn(rows, 1) * 0.1
    g = 1e-3
    group = rs.randint(0, 4, rows)
    last = np.select([group == 0, group == 1, group == 2], [T, T - 1, rs.randint(1, T - 1, rows)], 0)
    tabs = []
    for p in (W, b):
        tab = LazyAdamTable(p, lr=LR, weight_decay=wd)
        tab.m = np.where((group == 3)[:, None], 0.0, rs.randn(*p.shape) * 0.5 * g)
        tab.v = np.where((group == 3)[:, None], 0.0, g * g * rs.uniform(0.25, 1.0, p.shape))
        tab.last = last.astype(np.int64)
        tabs.append(tab)
    return tabs, group


@pytest.mark.parametrize('wd', [0.0, 1e-2])
@pytest.mark.parametrize('D', [4, 24, 260])
def test_flush_long_gaps(D, wd, record_property):
    """slb_adam_flush on its own: rows current, one step behind, 1 .. 2000 steps behind and never
    touched, against LazyAdamTable.flush in float64.  Afterwards last == t everywhere; untouched rows
    (m = v = 0) with wd = 0 stay bit-identical."""
    from spotlight_b200 import _lib, ops
    from spotlight_b200.optim import FusedAdam
    T = 2000
    tabs, group = _flush_case(D, wd, T, seed=D)
    dev = [t(x.astype(np.float32)) for tab in tabs for x in (tab.w, tab.m, tab.v)]
    last = t(tabs[0].last.astype(np.int32))
    W0 = dev[0].cpu().numpy().copy()
    W32 = [tab.w.astype(np.float32).astype(np.float64) for tab in tabs]
    for tab, w in zip(tabs, W32):          # the scheme starts from the same fp32 values
        tab.w, tab.m, tab.v = w, tab.m.astype(np.float32).astype(np.float64), tab.v.astype(np.float32).astype(np.float64)
    opt = FusedAdam([torch.nn.Parameter(torch.zeros(1))], lr=LR, weight_decay=wd)
    sched = opt.schedule(T, torch.device('cuda:0'))
    lib = _lib.load()
    _lib.check(lib.slb_adam_flush(*[ops._ptr(x) for x in dev], ops._ptr(last), tabs[0].w.shape[0], D, ops._ptr(sched),
                                  T, 0.9, 0.999, 1.0 - 0.9, 1.0 - 0.999, 1e-8, wd, ops._stream()), 'adam_flush')
    for tab in tabs:
        tab.flush(T)
    assert (last.cpu().numpy() == T).all()
    measured = {}
    for k, (tab, nm) in enumerate(zip(tabs, ('W', 'b'))):
        # elements the float64 flush leaves at least ten steps away from 0 follow a smooth trajectory;
        # the others (weight decay walked them to 0, where Adam's normalised step oscillates) are
        # held to a fraction of a step
        far = np.abs(tab.w) >= 10 * LR
        w, m, v = (x.cpu().numpy().astype(np.float64).reshape(tab.w.shape) for x in dev[3 * k:3 * k + 3])
        for got, want, what in ((w, tab.w, 'w'), (m, tab.m, 'exp_avg'), (v, tab.v, 'exp_avg_sq')):
            err, scale = np.abs(got - want), np.abs(want).max()
            measured['%s_%s_far' % (nm, what)] = err[far].max(initial=0.0) / scale
            measured['%s_%s_all' % (nm, what)] = err.max() / scale
            assert err[far].max(initial=0.0) <= FLUSH_RTOL[what] * scale, '%s %s: %.3e' % (nm, what, err[far].max())
            bound = NEAR_ZERO_RTOL[what] * (LR if what == 'w' else scale)
            assert err.max() <= bound, '%s %s near 0: %.3e' % (nm, what, err.max())
        measured['%s_w_all_over_lr' % nm] = np.abs(w - tab.w).max() / LR
    if wd == 0:
        never = group == 3
        assert (dev[0].cpu().numpy()[never] == W0[never]).all()
    for key, val in measured.items():
        record_property(key, float(val))


# ------------------------------------------------------------------ resume
def _fit_model(n_iter, inter, init):
    from spotlight_b200.factorization.implicit import ImplicitFactorizationModel
    m = ImplicitFactorizationModel(loss='bpr', embedding_dim=32, n_iter=n_iter, batch_size=128, l2=1e-3,
                                   use_cuda=True, random_state=np.random.RandomState(11))
    m._initialize(inter)
    m._net.load_state_dict(init)
    return m


def _interactions(U=4000, I=900, n=6000, seed=3):
    from spotlight_b200.interactions import Interactions
    rs = np.random.RandomState(seed)
    return Interactions(rs.randint(0, U, n).astype(np.int32), rs.randint(0, I, n).astype(np.int32),
                        num_users=U, num_items=I)


def test_resume_after_pickle_equals_uninterrupted_fit(tmp_path):
    """fit() one epoch, torch.save / torch.load, fit() one more: the same tables and Adam state, bit for
    bit, as one two-epoch fit().  The first fit()'s flush replays exactly the element steps the second
    epoch's prepass would have replayed."""
    inter = _interactions()
    ref = _fit_model(2, inter, _init_state(inter))
    ref.fit(inter)
    a = _fit_model(1, inter, _init_state(inter))
    a.fit(inter)
    path = str(tmp_path / 'model.pt')
    torch.save(a, path)
    b = torch.load(path, weights_only=False)
    b.fit(inter)
    assert b._optimizer.steps_taken == ref._optimizer.steps_taken
    for (k, x), (_, y) in zip(ref._net.state_dict().items(), b._net.state_dict().items()):
        assert torch.equal(x, y), k
    for p, q in zip(ref._net.parameters(), b._net.parameters()):
        s0, s1 = ref._optimizer.state[p], b._optimizer.state[q]
        for key in ('exp_avg', 'exp_avg_sq', 'last'):
            assert torch.equal(s0[key], s1[key]), key


def _init_state(inter):
    from spotlight_b200.factorization.representations import BilinearNet
    torch.manual_seed(5)
    net = BilinearNet(inter.num_users, inter.num_items, 32)
    with torch.no_grad():
        net.user_biases.weight.normal_(0, 0.1)
        net.item_biases.weight.normal_(0, 0.1)
    return net.state_dict()


# ------------------------------------------------------------------ hyperparameter changes
@pytest.mark.parametrize('change', ['lr', 'lr+wd'])
def test_hyperparameter_change_between_fits(change):
    """fit(), then a new lr (and weight decay) in param_groups, then fit() again: the default lazy Adam
    against torch.optim.Adam on the fused route given the same change, from the same weights and
    RandomState.  The steps rows missed before the change are replayed with the values they were
    taken under, those after it with the new ones, as dense Adam took them."""
    from spotlight_b200.factorization.implicit import ImplicitFactorizationModel
    inter = _interactions()
    models = []
    for func in (None, lambda p: torch.optim.Adam(p, lr=1e-2, weight_decay=1e-4)):
        m = ImplicitFactorizationModel(loss='bpr', embedding_dim=32, n_iter=2, batch_size=128, l2=1e-4,
                                       optimizer_func=func, use_cuda=True, random_state=np.random.RandomState(11))
        m._initialize(inter)
        models.append(m)
    models[1]._net.load_state_dict(models[0]._net.state_dict())
    assert models[0]._route() == 'epoch' and models[1]._route() == 'fused'
    for m in models:
        m.fit(inter)
        g = m._optimizer.param_groups[0]
        g['lr'] = 3e-3
        if change == 'lr+wd':
            g['weight_decay'] = 1e-3
        m.fit(inter)
    # test_model_gpu.test_lazy_adam_equals_dense_adam's tolerances
    for (k, a), (_, b) in zip(models[0]._net.state_dict().items(), models[1]._net.state_dict().items()):
        assert_close(a.cpu().numpy(), b.cpu().numpy(), 5e-4, atol=1e-7, what=k)
    st0 = models[0]._optimizer.state[models[0]._net.user_embeddings.weight]
    st1 = models[1]._optimizer.state[models[1]._net.user_embeddings.weight]
    assert_close(st0['exp_avg'].cpu().numpy(), st1['exp_avg'].cpu().numpy(), 2e-3, atol=1e-9, what='exp_avg')
    assert_close(st0['exp_avg_sq'].cpu().numpy(), st1['exp_avg_sq'].cpu().numpy(), 2e-3, atol=1e-12,
                 what='exp_avg_sq')


# ------------------------------------------------------------------ every variant runs
def _profiled_kernel_names():
    """Kernel names, as torch.profiler records them, of one Adam step of a small and a large batch
    (bpr) and of an adaptive hinge batch at every D, each followed by a flush."""
    from torch.profiler import ProfilerActivity, profile
    runs = []
    for D in DIMS:
        for B, loss, n in ((3001 + D, 'bpr', 1), (mac.bwd_small_limit(sms()) // 2 + 1001, 'bpr', 1),
                           (3001 + D, 'adaptive_hinge', 2)):
            case = mac.make_case(D, B, loss, n, seed=D, sms=sms())
            model, _, _ = _model(case, 0.0, 2, mac.seed_state(case, 2, seed=D))
            runs.append((model, case))
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for model, case in runs + runs:       # the profiler can lose a session's first launches
            _step(model, case['users'], case['items'], case['negs'], case.get('ratings'))
            model._optimizer.flush()
        torch.cuda.synchronize()
    return sorted({ev.name.replace(' ', '') for ev in prof.events()
                   if ev.device_type == torch.autograd.DeviceType.CUDA})


def test_profiler_sees_every_variant():
    """Every LPR's prepass, apply and flush kernels, both backward tile sizes with the right EX, the
    mode-0 hot-row kernel and adaptive hinge's forward run.  The profiling runs in a child process, so
    its profiler session does not share this process's CUPTI state with the other suites' profiler
    tests."""
    import json
    import subprocess
    import sys
    from oracle.mf_cases import lpr_for_dim
    here = os.path.dirname(os.path.abspath(__file__))
    code = ('import json, sys; sys.path.insert(0, %r); sys.path.insert(0, %r); '
            'import test_mf_adam_oracle_gpu as m; print(json.dumps(m._profiled_kernel_names()))'
            % (os.path.dirname(here), here))
    out = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, cwd=os.path.dirname(here),
                         timeout=900)
    assert out.returncode == 0, out.stderr[-4000:]
    names = json.loads(out.stdout.strip().split('\n')[-1])
    want = []
    for D in DIMS:
        L = lpr_for_dim(D)
        ex = '(true|\\(bool\\)1|1)' if L >= 8 and D == 4 * L else '(false|\\(bool\\)0|0)'
        want += ['mf_adam_prepass_kernel<%d>' % L, 'mf_adam_apply_kernel<%d>' % L, 'adam_flush_kernel<%d>' % L,
                 'mf_bwd_tile_kernel<%d,0,8,%s>' % (L, ex), 'mf_bwd_tile_kernel<%d,0,32,%s>' % (L, ex),
                 'mf_bwd_long_kernel<%d,0>' % L, 'mf_fwd_kernel<%d>' % L]
    mine = [n for n in names if 'mf_' in n or 'adam' in n]
    for w in sorted(set(want)):
        assert any(re.search(w, n) for n in names), (w, mine)
