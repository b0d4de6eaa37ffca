"""Lazy-exact Adam in the fused hashed-table MF step (csrc/mf.cu slb_mf_bloom_train_step under
SLB_OPT_ADAM: mf_bloom_adam_prepass_kernel, the mode-0 backward in compact mode,
mf_bloom_adam_apply_kernel and bias_adam_apply_kernel) against the float64 scheme of
tests/bloom_adam_common.py and against torch.optim.Adam.

Tolerances as tests/test_seq_adam_gpu.py: moments at 2e-5 of their scale; parameters at 5 % of one
step where the first moment is above 1e-3 of its maximum, at half a step where it is between 1e-5 and
1e-3, and within one step's bound on the rest (m / sqrt(v) turns last-bit gradient differences on
near-zero components into fractions of a step)."""

import numpy as np
import pytest
import torch

from bloom_adam_common import lazy_step, make_tables, read_rows
from conftest import assert_close
from oracle import bloom_cases as bc
from oracle.murmur import SEEDS

pytestmark = pytest.mark.gpu

LR = 1e-3
STEPS = 4
TABLES = ('Wu', 'Wi', 'bu', 'bi')


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to('cuda:0')


def _check_param(dev, tab, what):
    w, m = dev.cpu().numpy().astype(np.float64).reshape(tab.w.shape), tab.m
    scale = np.abs(m).max()
    quiet = np.abs(m) < 1e-3 * scale
    noise = np.abs(m) < 1e-5 * scale
    err = np.abs(w - tab.w)
    tol = 2e-6 * np.abs(tab.w).max()
    assert err[~quiet].max(initial=0.0) <= 0.05 * LR + tol, '%s: %.3e' % (what, err[~quiet].max())
    assert err[quiet & ~noise].max(initial=0.0) <= 0.5 * LR + tol, '%s (small moments): %.3e' % (
        what, err[quiet & ~noise].max(initial=0.0))
    assert err.max() <= 2.1 * LR, '%s moved by more than an Adam step' % what


def _batches(case, seed=0):
    """Step 1 is the whole case (hot rows beyond the sort cap, bucket twins, the padding id); later
    steps take a random eighth of it, so rows miss steps between touches."""
    B, n = len(case['users']), case['n_neg']
    rs = np.random.RandomState(seed)
    out = [(case['users'], case['items'], case['negs'])]
    for _ in range(STEPS - 1):
        idx = np.sort(rs.choice(B, B // 8, replace=False))
        negs = case['negs'][rs.permutation(len(case['negs']))[:len(idx) * n]]
        out.append((case['users'][idx], case['items'][idx], negs))
    return out


def _state(P):
    """Four (exp_avg, exp_avg_sq, last) triples of zeros for the GPU tables P."""
    return [(torch.zeros_like(p), torch.zeros_like(p), torch.zeros(p.shape[0], dtype=torch.int32, device=p.device))
            for p in P]


def _sched(upto):
    from spotlight_b200.optim import FusedAdam
    return FusedAdam([torch.nn.Parameter(torch.zeros(1))], lr=LR).schedule(upto, torch.device('cuda:0'))


def _gpu_step(P, S, case, u, i, j, step, wd, sched):
    from spotlight_b200 import _lib, ops
    return ops.mf_bloom_train_step_inplace(
        *P, t(u), t(i), t(j), case['loss'], case['n_neg'], list(SEEDS[:case['Hu']]), list(SEEDS[:case['Hi']]),
        case['pad_u'], case['pad_i'], _lib.OPT_ADAM, LR, states=S, weight_decay=wd, eps=1e-8,
        adam=dict(beta1=0.9, beta2=0.999, sched=sched, step=step)).item()


def _flush(P, S, steps, wd, sched):
    from spotlight_b200 import _lib, ops
    lib = _lib.load()
    for p, (m, v, last) in zip(P, S):
        _lib.check(lib.slb_adam_flush_table(ops._ptr(p), ops._ptr(m), ops._ptr(v), ops._ptr(last), p.shape[0],
                                            p[0].numel(), ops._ptr(sched), steps, 0.9, 0.999, 1.0 - 0.9,
                                            1.0 - 0.999, 1e-8, wd, ops._stream()), 'adam_flush_table')


# (D, loss, n_neg, Hu, Hi, pad): every LPR, every loss, the hash pairs (0,1) (0,4) (2,3) (3,0) (0,24),
# padding 0 / 3 / none
ENTRIES = [(4, 'pointwise', 1, 0, 1, 0), (12, 'bpr', 1, 0, 4, 3), (32, 'hinge', 1, 2, 3, -1),
           (64, 'adaptive_hinge', 2, 3, 0, 0), (100, 'adaptive_hinge', 5, 0, 24, 3), (128, 'bpr', 1, 2, 3, 0),
           (256, 'hinge', 1, 0, 4, -1)]
PARITY = [e + (wd,) for e in ENTRIES for wd in (0.0, 0.1)]


@pytest.mark.parametrize('D,loss,n,Hu,Hi,pad,wd', PARITY, ids=['%d-%s%d-%d,%d-pad%d-wd%g' % e for e in PARITY])
def test_step_parity(D, loss, n, Hu, Hi, pad, wd):
    """Four consecutive steps against the float64 scheme: after each the loss, every table and its
    moments, `last` exactly, and every entry the step neither read nor stepped bit-identical; after a
    flush, all four tables and moments against the scheme's flush (float64 dense Adam,
    tests/test_mf_bloom_adam_oracle_cpu.py)."""
    seed = 501 + 10 * D + Hu + Hi
    case = bc.case_for(D, loss, n, Hu, Hi, pad, seed + (seed % 5 == 0))    # seed % 5 == 0: a 3M-id case
    assert len(case['hot_items']) > 0
    tabs = make_tables(bc.tables64(case), LR, wd)
    P = [t(case[k].copy()) for k in TABLES]
    S = _state(P)
    sched = _sched(STEPS)
    for step, (u, i, j) in enumerate(_batches(case), 1):
        before = [p.cpu().numpy().copy() for p in P]
        last_before = [tab.last.copy() for tab in tabs]
        ref = lazy_step(tabs, case, u, i, j, step)
        loss_gpu = _gpu_step(P, S, case, u, i, j, step, wd, sched)
        what = 'step %d' % step
        assert_close(loss_gpu, ref['loss'], 1e-5, what=what + ' loss')
        for k, (tab, p, (m, v, last), nm) in enumerate(zip(tabs, P, S, TABLES)):
            assert (last.cpu().numpy() == tab.last).all(), '%s %s last' % (what, nm)
            assert_close(m.cpu().numpy().reshape(tab.m.shape), tab.m, 2e-5, what='%s %s exp_avg' % (what, nm))
            assert_close(v.cpu().numpy().reshape(tab.v.shape), tab.v, 2e-5, what='%s %s exp_avg_sq' % (what, nm))
            _check_param(p, tab, '%s %s' % (what, nm))
            still = tab.last == last_before[k]
            assert (p.cpu().numpy()[still] == before[k][still]).all(), '%s %s: an entry not read changed' % (what, nm)
    assert any((tab.last < STEPS - 1).any() for tab in tabs), 'no entry missed several steps'
    _flush(P, S, STEPS, wd, sched)
    for tab, p, (m, v, last), nm in zip(tabs, P, S, TABLES):
        tab.flush(STEPS)
        assert (last.cpu().numpy() == STEPS).all()
        assert_close(m.cpu().numpy().reshape(tab.m.shape), tab.m, 2e-5, what='flushed %s exp_avg' % nm)
        _check_param(p, tab, 'flushed ' + nm)


def test_read_rows_cover_the_padding_row():
    """The prepass reads the padding row of a hashed table like any other (the case has the padding
    id among its users and items)."""
    case = bc.case_for(32, 'bpr', 1, 2, 3, 0, 611)
    ru, ri, _, _ = read_rows(case, case['Wu'].shape[0], case['Wi'].shape[0], case['users'], case['items'],
                             case['negs'])
    assert (ru == 0).any() and (ri == 0).any()


def test_bit_reproducible():
    case = bc.case_for(64, 'adaptive_hinge', 2, 2, 3, 0, 711)
    sched = _sched(STEPS)
    outs = []
    for _ in range(2):
        P = [t(case[k].copy()) for k in TABLES]
        S = _state(P)
        losses = [_gpu_step(P, S, case, u, i, j, s, 0.1, sched) for s, (u, i, j) in enumerate(_batches(case), 1)]
        outs.append((losses, [x.cpu().numpy() for x in P + [y for s in S for y in s]]))
    assert outs[0][0] == outs[1][0]
    for a, b in zip(outs[0][1], outs[1][1]):
        assert (a == b).all()


def test_c_abi_rejections_leave_tables_untouched():
    """Adam with a rating loss, without a state pointer, `last` or schedule, with adam_step < 1, and
    in dense mode: each refused with a clear message before any launch."""
    import ctypes
    from spotlight_b200 import _lib, ops
    case = bc.case_for(16, 'bpr', 1, 0, 3, 0, 811)
    P = [t(case[k].copy()) for k in TABLES]
    S = _state(P)
    sched = _sched(4)
    users, items, negs = t(case['users']), t(case['items']), t(case['negs'])
    ratings = torch.ones(len(case['users']), device='cuda:0')
    lib = _lib.load()
    keep = []

    def args(loss='bpr', **kw):
        x = ops._bloom_args(*P, users, items, None if loss == 'regression' else negs,
                            ratings if loss == 'regression' else None, loss, 1, [], list(SEEDS[:3]), -1, 0)
        a = x.base
        out = torch.zeros(1, device='cuda:0')
        keep.append(out)
        a.loss_out = out.data_ptr()
        a.grad_mode, a.opt, a.lr, a.eps = _lib.GRAD_COMPACT, _lib.OPT_ADAM, LR, 1e-8
        ops._bloom_adam_args(x, P, S, dict(beta1=0.9, beta2=0.999, sched=sched, step=1))
        for k, v in kw.items():
            if hasattr(x, k):
                setattr(x, k, v)
            else:
                setattr(a, k, v)
        keep.append(ops._bloom_workspace('mfbfa', x, P[0].device))
        return x

    before = [p.cpu().numpy().copy() for p in P]
    cases = [(args(loss='regression'), 'pairwise losses only'), (args(state2_Wi=None), 'exp_avg_sq'),
             (args(state_bu=None), 'state'), (args(last_bi=None), 'last'), (args(last_u=None), 'last'),
             (args(adam_sched=None), 'schedule'), (args(adam_step=0), 'adam_step'),
             (args(grad_mode=_lib.GRAD_DENSE), 'compact')]
    for x, msg in cases:
        rc = lib.slb_mf_bloom_train_step(ctypes.byref(x), ops._stream())
        err = lib.slb_last_error().decode()
        assert rc != 0 and msg in err, (msg, err)
    torch.cuda.synchronize()
    for p, b in zip(P, before):
        assert (p.cpu().numpy() == b).all()
    for m, v, last in S:
        assert not m.any() and not v.any() and not last.any()


# ------------------------------------------------------------------ model level
def _bloom_model(opt_func, Hu, Hi, loss='bpr', n_iter=2, U=400, I=3000, D=16, seed=3):
    from spotlight_b200.factorization.implicit import ImplicitFactorizationModel
    from spotlight_b200.factorization.representations import BilinearNet
    from spotlight_b200.layers import BloomEmbedding, ScaledEmbedding
    torch.manual_seed(seed)
    ue = BloomEmbedding(U, D, compression_ratio=0.4, num_hash_functions=Hu) if Hu else ScaledEmbedding(U, D)
    ie = BloomEmbedding(I, D, compression_ratio=0.3, num_hash_functions=Hi) if Hi else ScaledEmbedding(I, D)
    rep = BilinearNet(U, I, D, user_embedding_layer=ue, item_embedding_layer=ie)
    return ImplicitFactorizationModel(loss=loss, embedding_dim=D, batch_size=128, n_iter=n_iter, representation=rep,
                                      optimizer_func=opt_func, use_cuda=True, random_state=np.random.RandomState(9))


def _interactions(U=400, I=3000, n=3000, seed=4):
    from spotlight_b200.interactions import Interactions
    rs = np.random.RandomState(seed)
    return Interactions(rs.randint(0, U, n).astype(np.int32), rs.randint(0, I // 3, n).astype(np.int32),
                        num_users=U, num_items=I)


def _fit(model, inter, state=None, capsys=None):
    model._initialize(inter)
    if state is not None:
        model._net.load_state_dict(state)
    init = {k: v.clone() for k, v in model._net.state_dict().items()}
    capsys.readouterr()
    model.fit(inter, verbose=True)
    lines = [l for l in capsys.readouterr().out.strip().split('\n') if l.startswith('Epoch')]
    return init, np.array([float(l.split('loss')[1]) for l in lines])


FITS = [(0, 3, 'bpr', 0.0), (2, 3, 'adaptive_hinge', 1e-3), (3, 0, 'hinge', 1e-3)]


@pytest.mark.parametrize('Hu,Hi,loss,l2', FITS, ids=['%d,%d-%s-l2%g' % f for f in FITS])
def test_fit_equals_torch_adam_on_bloom_route(Hu, Hi, loss, l2, capsys):
    """fit() with optim.fused_adam takes the in-place hashed step; against torch.optim.Adam on the
    dense bloom route (dense gradients of every table, dense Adam sweep) from the same weights and
    RandomState: same stream position, epoch losses at 1e-5, tables and moments as
    test_seq_adam_gpu.test_fit_equals_torch_adam_on_fused_route.  Most item ids are never drawn as
    positives, so rows miss steps."""
    from spotlight_b200 import optim
    inter = _interactions()
    lazy = _bloom_model(optim.fused_adam(lr=1e-2, weight_decay=l2), Hu, Hi, loss)
    init, ll = _fit(lazy, inter, capsys=capsys)
    dense = _bloom_model(lambda p: torch.optim.Adam(p, lr=1e-2, weight_decay=l2), Hu, Hi, loss)
    _, ld = _fit(dense, inter, state=init, capsys=capsys)
    assert lazy._route() == 'bloom' and dense._route() == 'bloom'
    s0, s1 = lazy._random_state.get_state(), dense._random_state.get_state()
    assert (s0[1] == s1[1]).all() and s0[2] == s1[2]
    assert_close(ll, ld, 1e-5, what='epoch losses')
    for (k, a), (_, b) in zip(lazy._net.state_dict().items(), dense._net.state_dict().items()):
        assert_close(a.cpu().numpy(), b.cpu().numpy(), 5e-4, atol=1e-7, what=k)
    opt = lazy._optimizer
    n_steps = 2 * ((len(inter.user_ids) + 127) // 128)
    assert opt.steps_taken == n_steps
    for p, q in zip(lazy._net.parameters(), dense._net.parameters()):
        st0, st1 = opt.state[p], dense._optimizer.state[q]
        assert p.grad is None
        assert int(st0['last'].min()) == n_steps
        assert_close(st0['exp_avg'].cpu().numpy(), st1['exp_avg'].cpu().numpy(), 2e-3, atol=1e-9, what='exp_avg')
        assert_close(st0['exp_avg_sq'].cpu().numpy(), st1['exp_avg_sq'].cpu().numpy(), 2e-3, atol=1e-12,
                     what='exp_avg_sq')


def test_resume_and_pickle(tmp_path, capsys):
    """A second fit() resumes the step count, and so does a torch.save / torch.load round trip; both
    continue identically."""
    from spotlight_b200 import optim
    inter = _interactions()
    model = _bloom_model(optim.fused_adam(lr=1e-2, weight_decay=1e-4), 2, 3, n_iter=1)
    _fit(model, inter, capsys=capsys)
    steps = (len(inter.user_ids) + 127) // 128
    assert model._optimizer.steps_taken == steps
    path = str(tmp_path / 'model.pt')
    torch.save(model, path)
    loaded = torch.load(path, weights_only=False)
    for m in (model, loaded):
        m.fit(inter)
        assert m._optimizer.steps_taken == 2 * steps
        for p in m._net.parameters():
            assert int(m._optimizer.state[p]['last'].min()) == 2 * steps
    for (k, x), (_, y) in zip(model._net.state_dict().items(), loaded._net.state_dict().items()):
        assert_close(x.cpu().numpy(), y.cpu().numpy(), 1e-6, atol=1e-9, what=k)
    assert np.isfinite(model.predict(3)).all()


FIXTURES = ['fit_bloom_adam_bpr', 'fit_bloom_adam_both']


@pytest.mark.parametrize('name', FIXTURES)
def test_fit_reproduces_reference_fixture(name, capsys):
    """tests/golden/make_golden_bloom_adam.py: two epochs of the reference's fit() with its default
    dense Adam, through optim.fused_adam(lr, weight_decay=l2) on the in-place hashed step.  Epoch
    losses at 1e-5, final state_dict and predict at 2e-3 of their scale (Adam: see the module
    docstring), the RandomState position exact, every row current after fit()."""
    from bloom_adam_common import fixture_case
    from conftest import load_golden
    from spotlight_b200 import optim
    from spotlight_b200.factorization.implicit import ImplicitFactorizationModel
    from spotlight_b200.factorization.representations import BilinearNet
    from spotlight_b200.interactions import Interactions
    from spotlight_b200.layers import BloomEmbedding, ScaledEmbedding
    g = load_golden(name)
    case = fixture_case(g)
    U, I, D = int(g['num_users']), int(g['num_items']), int(g['dim'])
    ue = (BloomEmbedding(U, D, compression_ratio=float(g['user_ratio']), num_hash_functions=case['Hu'])
          if case['Hu'] else ScaledEmbedding(U, D))
    ie = BloomEmbedding(I, D, compression_ratio=float(g['item_ratio']), num_hash_functions=case['Hi'])
    rep = BilinearNet(U, I, D, user_embedding_layer=ue, item_embedding_layer=ie)
    rep.load_state_dict({k[5:]: torch.from_numpy(v) for k, v in g.items() if k.startswith('init.')})
    model = ImplicitFactorizationModel(loss=case['loss'], embedding_dim=D, batch_size=int(g['batch']),
                                       n_iter=int(g['n_iter']), representation=rep,
                                       num_negative_samples=int(g['n_neg']),
                                       optimizer_func=optim.fused_adam(lr=float(g['lr']), weight_decay=float(g['l2'])),
                                       use_cuda=True, random_state=np.random.RandomState(0))
    inter = Interactions(g['users'], g['items'], num_users=U, num_items=I)
    model._initialize(inter)
    model._random_state.set_state(('MT19937', g['rs0_key'], int(g['rs0_pos'])))
    assert model._route() == 'bloom'
    capsys.readouterr()
    model.fit(inter, verbose=True)
    lines = [l for l in capsys.readouterr().out.strip().split('\n') if l.startswith('Epoch')]
    assert_close(np.array([float(l.split('loss')[1]) for l in lines]), g['epoch_losses'], 1e-5, what='epoch losses')
    for k, v in model._net.state_dict().items():
        assert_close(v.cpu().numpy(), g['final.' + k], 2e-3, atol=1e-7, what=k)
    st = model._random_state.get_state()
    assert (st[1] == g['rs_key']).all() and st[2] == int(g['rs_pos'])
    opt = model._optimizer
    for p in model._net.parameters():
        assert int(opt.state[p]['last'].min()) == opt.steps_taken
    assert_close(model.predict(int(g['predict_user'])), g['predict'], 2e-3, what='predict')


def test_config_size_steps_equal_dense_route():
    """BASELINE configs[3] size: 1 M users (plain table), 50 M items hashed to 1 M rows (H = 4), D = 64,
    hinge, B = 262 144, weight decay 1e-4.  Three steps on distinct minibatches through the in-place
    Adam step, then a flush, against the dense bloom route (dense gradients of every table) with
    torch.optim.Adam from the same state: the loss of every step, and all four tables and their
    moments after the flush.  Steps 2 and 3 run the prepass over rows and biases that step 1
    moved; the bias update sees P = 524 288 (id, g) pairs over the 50 M-entry item-bias table."""
    from spotlight_b200 import _lib, ops
    from spotlight_b200.factorization.representations import BilinearNet
    from spotlight_b200.layers import BloomEmbedding, ScaledEmbedding
    from spotlight_b200.optim import FusedAdam
    U, I, D, B, K, lr, wd = 1_000_000, 50_000_000, 64, 262_144, 3, 1e-3, 1e-4
    dev = torch.device('cuda:0')
    torch.manual_seed(0)
    lazy = BilinearNet(U, I, D, user_embedding_layer=ScaledEmbedding(U, D),
                       item_embedding_layer=BloomEmbedding(I, D, compression_ratio=0.02, num_hash_functions=4)).to(dev)
    dense = BilinearNet(U, I, D, user_embedding_layer=ScaledEmbedding(U, D),
                        item_embedding_layer=BloomEmbedding(I, D, compression_ratio=0.02, num_hash_functions=4)).to(dev)
    with torch.no_grad():
        for p, q in zip(lazy.parameters(), dense.parameters()):
            q.copy_(p)
    g = torch.Generator(device=dev).manual_seed(1)
    users = torch.randint(0, U, (K, B), device=dev, generator=g)
    items = torch.randint(0, I, (K, B), device=dev, generator=g)
    negs = torch.randint(0, I, (K, B), device=dev, generator=g)
    spec = lazy.fused_spec()
    params = (spec['Wu'], spec['Wi'], lazy.user_biases.weight, lazy.item_biases.weight)
    fopt = FusedAdam(lazy.parameters(), lr=lr, weight_decay=wd)
    states = [fopt.fused_states(p, own_last=True) for p in params]
    sched = fopt.schedule(K, dev)
    dspec = dense.fused_spec()
    dparams = (dspec['Wu'], dspec['Wi'], dense.user_biases.weight, dense.item_biases.weight)
    dopt = torch.optim.Adam(dparams, lr=lr, weight_decay=wd)
    for k in range(K):
        ll = ops.mf_bloom_train_step_inplace(*params, users[k], items[k], negs[k], 'hinge', 1, spec['user_seeds'],
                                             spec['item_seeds'], spec['user_pad'], spec['item_pad'], _lib.OPT_ADAM,
                                             lr, states, wd, 1e-8,
                                             adam=dict(beta1=0.9, beta2=0.999, sched=sched, step=k + 1)).item()
        dopt.zero_grad()
        ld = ops.fused_bloom_loss(*dparams, users[k], items[k], negs[k], 'hinge', 1, dspec)
        ld.backward()
        dopt.step()
        assert abs(ll - ld.item()) <= 1e-5 * abs(ld.item()), (k, ll, ld.item())
    fopt.advance(K)
    fopt.flush()
    names = ('Wu', 'Wi', 'bu', 'bi')
    with torch.no_grad():
        for p, q, (m, v, last), nm in zip(params, dparams, states, names):
            assert int(last.min()) == K, nm
            err = (p - q).abs().max().item()
            assert err <= 0.05 * lr + 2e-6 * q.abs().max().item(), '%s: %.3e' % (nm, err)
            st = dopt.state[q]
            for a, b, what in ((m, st['exp_avg'], 'exp_avg'), (v, st['exp_avg_sq'], 'exp_avg_sq')):
                e = (a - b).abs().max().item()
                assert e <= 2e-3 * b.abs().max().item() + 1e-12, '%s %s: %.3e' % (nm, what, e)


def _profiled_fit_kernel_names():
    """Kernel names of a two-epoch fit() of a Bloom model (both sides hashed) under fused_adam, as
    torch.profiler records them."""
    from torch.profiler import ProfilerActivity, profile
    from spotlight_b200 import optim
    inter = _interactions()
    model = _bloom_model(optim.fused_adam(lr=1e-2, weight_decay=1e-4), 2, 3)
    model._initialize(inter)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        model.fit(inter)
        torch.cuda.synchronize()
    return sorted({ev.name.replace(' ', '') for ev in prof.events()
                   if ev.device_type == torch.autograd.DeviceType.CUDA})


def test_fit_launches_the_lazy_adam_kernels():
    """fit() under fused_adam launches the prepass, the mode-0 backward, the row and bias Adam kernels
    and the flush, and none of the dense route's optimizer kernels.  The profiling runs in a child
    process, so its profiler session does not share this process's CUPTI state with the other suites'
    profiler tests."""
    import json
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    code = ('import json, sys; sys.path.insert(0, %r); sys.path.insert(0, %r); '
            'import test_mf_bloom_adam_gpu as m; print(json.dumps(m._profiled_fit_kernel_names()))'
            % (os.path.dirname(here), here))
    out = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, cwd=os.path.dirname(here),
                         timeout=600)
    assert out.returncode == 0, out.stderr[-4000:]
    names = json.loads(out.stdout.strip().split('\n')[-1])
    want = ['mf_bloom_adam_prepass_kernel<', 'mf_fwd_bloom_kernel<', 'mf_bwd_tile_kernel<4,0,', 'mf_bloom_adam_apply_kernel<',
            'bias_adam_apply_kernel<', 'adam_flush_table_kernel<']
    for w in want:
        assert any(w in n for n in names), (w, [n for n in names if 'mf_' in n or 'bias' in n or 'adam' in n])
    unwanted = ['mf_apply_kernel', 'bias_apply_kernel', 'multi_tensor_apply', 'embedding_backward']
    for w in unwanted:
        assert not any(w in n and 'adam_apply' not in n for n in names), (w, names)
