"""The planned MF step (csrc/mf_v2.cuh: plan, mf_user_kernel, mf_item_kernel and the hot-row
kernels, with the fused row-wise SGD / Adagrad) against the float64 oracle (oracle/mf.py).

Cases come from oracle/mf_cases.py: every member-list length class, hot rows, ties and
inactive rows are built in.  Each step is scaled so that the update measures the gradient
(mf_cases.hparams); the update (new - old) and the Adagrad state change are compared at 1e-5 of
the oracle's max, the loss at 1e-5, and rows without a non-zero term must stay bit-identical.
The small / large thresholds follow the library: B < sms * 768 selects the small user kernel,
2B < sms * 768 the small item kernel.
"""

import ctypes

import numpy as np
import pytest
import torch

from conftest import assert_close
from oracle import mf as omf
from oracle import mf_cases as mc

pytestmark = pytest.mark.gpu

DIMS = (8, 16, 32, 64, 128)
LOSSES = mc.LOSSES
OPT_WD = (('sgd', False), ('sgd', True), ('adagrad', False), ('adagrad', True))
TABLES = ('Wu', 'Wi', 'bu', 'bi')


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def small_B(D):
    return 3001 + D


def large_B():
    return mc.small_limit(sms()) + 1001          # both the user and the item kernel take the large variant


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def gpu_step(P, S, case, opt, lr, wd, users=None, items=None, negs=None):
    """One planned step in place on device tables P (and Adagrad states S); returns the loss."""
    from spotlight_b200 import _lib, ops
    kind = _lib.OPT_SGD if opt == 'sgd' else _lib.OPT_ADAGRAD
    u, i, j = (case[k] if x is None else x for k, x in (('users', users), ('items', items), ('negs', negs)))
    out = ops.mf_train_step_inplace(*P, t(u), t(i), t(j), case['loss'], kind, lr, states=S, weight_decay=wd)
    return out.item()


def oracle_step(P64, S64, case, opt, lr, wd, users=None, items=None, negs=None, **kw):
    u, i, j = (case[k] if x is None else x for k, x in (('users', users), ('items', items), ('negs', negs)))
    return omf.fused_step(P64, u, i, j, case['loss'], opt, lr, wd, 1e-10, S64, cap=case['cap'], **kw)


def compare(got, want, old, touched, what, rtol=1e-5):
    """The update got - old against want - old at rtol of the oracle's max; untouched rows exact."""
    got = got.detach().cpu().numpy().astype(np.float64).reshape(old.shape)
    old = old.astype(np.float64)
    assert_close(got - old, want.reshape(old.shape) - old, rtol, what=what)
    rows = ~touched
    assert (got[rows] == old[rows]).all(), '%s: a row without a non-zero term changed' % what


def run_and_check(case, opt, wd_on, steps=1, seed=0):
    lr, wd, S0 = mc.hparams(case, opt, wd_on, seed)
    P0 = [case[k] for k in TABLES]
    P, S = [t(p.copy()) for p in P0], ([t(s.copy()) for s in S0] if S0 else None)
    P64 = mc.tables64(case)
    S64 = [s.astype(np.float64) for s in S0] if S0 else None
    for _ in range(steps):
        loss = gpu_step(P, S, case, opt, lr, wd)
        ref = oracle_step(P64, S64, case, opt, lr, wd)
        assert_close(loss, ref['loss'], 1e-5, what='loss')
    # every step touches the same rows (the batch repeats)
    tu, ti = ref['touched_u'], ref['touched_i']
    for k, (p, nm) in enumerate(zip(P, TABLES)):
        compare(p, P64[k], P0[k], (tu, ti)[k % 2], nm)
        if S:
            compare(S[k], S64[k], S0[k], (tu, ti)[k % 2], 's' + nm)
    return ref


# ------------------------------------------------------------------ matrix

@pytest.mark.parametrize('opt,wd_on', OPT_WD, ids=['sgd', 'sgd_wd', 'adagrad', 'adagrad_wd'])
@pytest.mark.parametrize('loss', LOSSES)
@pytest.mark.parametrize('D', DIMS)
def test_small_batch_vs_oracle(D, loss, opt, wd_on):
    """Small batch: mf_user_kernel<LPR, 1, LOSS, 8>, mf_item_kernel<LPR, 8> and both hot-row kernels."""
    case = mc.small_case(D, loss, sms())
    assert case['B'] * 2 < mc.small_limit(sms())
    run_and_check(case, opt, wd_on)


@pytest.mark.parametrize('loss', LOSSES)
@pytest.mark.parametrize('D', DIMS)
def test_large_batch_vs_oracle(D, loss):
    """Large batch: mf_user_kernel<LPR/2, 2, LOSS, 32> at D = 64 / 128, <LPR, 1, LOSS, 32> below,
    mf_item_kernel<LPR, 32>; (opt, wd) cycles so that each pair appears at every D."""
    k = (DIMS.index(D) + LOSSES.index(loss)) % 4
    opt, wd_on = OPT_WD[k]
    case = mc.large_case(D, loss, sms())
    assert case['B'] >= mc.small_limit(sms())
    run_and_check(case, opt, wd_on)


def _kernel_names(prof):
    return {e.name.replace(' ', '') for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}


@pytest.mark.parametrize('D', DIMS)
def test_profiler_sees_every_variant(D):
    """A small and a large case of every loss run the kernel instantiations the matrix relies
    on: a change of the thresholds cannot silently drop a variant from the suite."""
    from spotlight_b200 import _lib
    from torch.profiler import ProfilerActivity, profile
    lpr = D // 4
    want = {'mf_item_kernel<%d,8>' % lpr, 'mf_item_kernel<%d,32>' % lpr, 'mf_item_long_kernel<%d>' % lpr}
    cases = []
    for loss in LOSSES:
        L = _lib.LOSS_KIND[loss]
        want |= {'mf_user_kernel<%d,1,%d,8>' % (lpr, L), 'mf_user_long_kernel<%d,%d>' % (lpr, L),
                 ('mf_user_kernel<%d,2,%d,32>' % (lpr // 2, L)) if D >= 64 else 'mf_user_kernel<%d,1,%d,32>' % (lpr, L)}
        for B in (small_B(D), large_B()):
            cases.append(mc.make_case(D, B, loss, seed=B + D, sms=sms()))
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        # two passes: the profiler can lose the records of a session's first launches (a variant
        # that only the first case launches has gone unrecorded), and a variant the cases do not
        # launch is still missing from both
        for case in cases + cases:
            P = [t(case[k]) for k in TABLES]
            gpu_step(P, None, case, 'sgd', 1e-3, 0.0)
        torch.cuda.synchronize()
    names = _kernel_names(prof)
    for w in sorted(want):
        assert any(w in n for n in names), (w, sorted(n for n in names if 'mf_' in n))


# ------------------------------------------------------------------ trajectory and first touch

@pytest.mark.parametrize('size', ['small', 'large'])
def test_adagrad_weight_decay_three_steps(size):
    """Three consecutive Adagrad steps with weight decay, the state carried, against the
    iterated oracle."""
    D = 64 if size == 'small' else 32
    case = mc.make_case(D, small_B(D) if size == 'small' else large_B(), 'bpr', seed=11, sms=sms())
    run_and_check(case, 'adagrad', True, steps=3)


def test_adagrad_from_zero_state():
    """First Adagrad step from a zero accumulator: w -= lr g / (|g| + eps) is lr sign(g), so the
    check is sign-conditioned (|g| > 1e-7); the state is g^2 at 1e-5, on all four tables."""
    case = mc.make_case(32, small_B(32), 'pointwise', seed=12, sms=sms())
    lr, wd = 0.05, 0.0
    P0 = [case[k] for k in TABLES]
    P = [t(p.copy()) for p in P0]
    S = [torch.zeros_like(p) for p in P]
    P64 = mc.tables64(case)
    S64 = [np.zeros(p.shape) for p in P64]
    loss = gpu_step(P, S, case, 'adagrad', lr, wd)
    ref = oracle_step(P64, S64, case, 'adagrad', lr, wd)
    assert_close(loss, ref['loss'], 1e-5, what='loss')
    for k, nm in enumerate(TABLES):
        g = (ref['dWu'], ref['dWi'], ref['dbu'], ref['dbi'])[k].reshape(P0[k].shape)
        assert_close(S[k].cpu().numpy(), S64[k].reshape(P0[k].shape), 1e-5, atol=1e-30, what='s' + nm)
        big = np.abs(g) > 1e-7
        err = np.abs(P[k].cpu().numpy().astype(np.float64) - P64[k].reshape(P0[k].shape))[big]
        assert big.any() and err.max() < 1e-6, (nm, err.max())


# ------------------------------------------------------------------ edges

def _tiny_case(D, users, items, negs, U, I, loss='bpr', seed=0):
    rs = np.random.RandomState(seed)
    se = 1.0 / D ** 0.25
    return dict(D=D, B=len(users), loss=loss, U=U, I=I, cap=mc.seg_sort_cap(D), hot=False,
                Wu=(rs.randn(U, D) * se).astype(np.float32), Wi=(rs.randn(I, D) * se).astype(np.float32),
                bu=(rs.randn(U, 1) * 0.1).astype(np.float32), bi=(rs.randn(I, 1) * 0.1).astype(np.float32),
                users=np.asarray(users, dtype=np.int64), items=np.asarray(items, dtype=np.int64),
                negs=np.asarray(negs, dtype=np.int64))


@pytest.mark.parametrize('D', [8, 128])
def test_batch_of_one_and_two(D):
    run_and_check(_tiny_case(D, [3], [5], [2], 7, 9), 'adagrad', True)
    run_and_check(_tiny_case(D, [4, 4], [1, 6], [6, 0], 7, 9, loss='pointwise'), 'sgd', True)


@pytest.mark.parametrize('D', [16, 64])
def test_one_user_owns_the_batch(D):
    """B = 5000 interactions of one user: one hot user row, walked in 256 / LPR chunks."""
    rs = np.random.RandomState(D)
    B, I = 5000, 3000
    case = _tiny_case(D, np.full(B, 6), rs.randint(0, I, B), rs.randint(0, I, B), 10, I, seed=D)
    run_and_check(case, 'sgd', True)
    run_and_check(case, 'adagrad', False)


def test_short_and_hot_free_batches_reuse_the_workspace():
    """Workspace reuse at one (U, I, D): a large hot-row batch, then a short batch, then a batch
    without hot rows, then the large one again.  Each is checked against the oracle, so a count,
    total or completion counter that is not re-armed to zero between steps shows up."""
    D = 32
    big = mc.make_case(D, large_B(), 'hinge', seed=21, sms=sms())
    U, I = big['U'], big['I']
    rs = np.random.RandomState(3)
    short = dict(big, B=37, users=rs.randint(0, U, 37), items=rs.randint(0, I, 37), negs=rs.randint(0, I, 37))
    cool = dict(big, B=4000, users=rs.permutation(U)[:4000], items=rs.randint(0, I, 4000), negs=rs.randint(0, I, 4000))
    for case, opt in ((big, 'sgd'), (short, 'adagrad'), (cool, 'sgd'), (big, 'adagrad'), (short, 'sgd')):
        if case is not big:
            case['loss'] = 'bpr'                  # the hinge boundary is only kept clear in the built case
        run_and_check(case, opt, True)
    assert max(np.bincount(cool['users']).max(), np.bincount(np.r_[cool['items'], cool['negs']]).max()) <= cool['cap']


# ------------------------------------------------------------------ gradient-out mode

@pytest.mark.parametrize('opt', ['sgd', 'adagrad'])
def test_gradient_out_mode(opt):
    """opt_users_only with GRAD_DENSE and norm_batch = 3B (a shard of a larger global batch):
    the user side updates in place, the item kernels (tile and hot-row) hand out dWi / dbi."""
    from spotlight_b200 import _lib, ops
    lib = _lib.load()
    case = mc.make_case(64, small_B(64), 'bpr', seed=31, sms=sms())
    B = case['B']
    norm = 3 * B
    lr, wd, S0 = mc.hparams(case, opt, True)
    if S0:
        S0 = [s * (B / norm) ** 2 for s in S0]   # gradients are a third as large
    P0 = [case[k] for k in TABLES]
    P = [t(p.copy()) for p in P0]
    S = [t(s.copy()) for s in S0] if S0 else None
    users, items, negs = t(case['users']), t(case['items']), t(case['negs'])
    dWi = torch.zeros(case['I'], 64, device='cuda')
    dbi = torch.zeros(case['I'], device='cuda')
    loss_out = torch.empty(1, device='cuda')
    a = ops.mf_step_args(*P, users, items, negs, 'bpr', 1)
    a.loss_out = loss_out.data_ptr()
    a.grad_mode = _lib.GRAD_DENSE
    a.dWi, a.dbi = dWi.data_ptr(), dbi.data_ptr()
    a.opt = _lib.OPT_SGD if opt == 'sgd' else _lib.OPT_ADAGRAD
    a.lr, a.weight_decay, a.eps = lr, wd, 1e-10
    if S:
        a.state_Wu, a.state_bu = S[0].data_ptr(), S[2].data_ptr()
    a.norm_batch, a.opt_users_only = norm, 1
    ws = ops.workspace('mf%d_%d' % (case['U'], case['I']),
                       lib.slb_mf_step_workspace_bytes(B, 1, a.loss, case['U'], case['I']), 'cuda')
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    fws = ops.workspace('mfv2_%d_%d_%d' % (case['U'], case['I'], 64),
                        lib.slb_mf_fused_workspace_bytes(B, case['U'], case['I'], 64), 'cuda')
    a.fused_workspace, a.fused_workspace_bytes = fws.data_ptr(), fws.numel()
    _lib.check(lib.slb_mf_train_step(ctypes.byref(a), ops._stream()), 'mf_train_step')
    P64 = mc.tables64(case)
    S64 = [s.astype(np.float64) for s in S0] if S0 else None
    ref = oracle_step(P64, S64, case, opt, lr, wd, norm=norm)
    assert_close(loss_out.item(), ref['loss'], 1e-5, what='loss')
    assert_close(dWi.cpu().numpy(), ref['dWi'], 1e-5, what='dWi')
    assert_close(dbi.cpu().numpy(), ref['dbi'].reshape(-1), 1e-5, what='dbi')
    for k in (0, 2):
        compare(P[k], P64[k], P0[k], ref['touched_u'], TABLES[k])
        if S:
            compare(S[k], S64[k], S0[k], ref['touched_u'], 's' + TABLES[k])
    for k in (1, 3):                             # the item tables belong to their owners
        assert torch.equal(P[k].cpu(), torch.from_numpy(P0[k]))


# ------------------------------------------------------------------ determinism

def test_hot_row_loss_is_bit_reproducible():
    """40 hot users spread over many 4096-row scan tiles, plus hot items: the scan lists hot rows
    in atomic order, the plan puts them in segment order, so parameters, states and the loss
    are bit-identical across runs."""
    case = mc.make_case(64, 30000, 'bpr', seed=41, sms=sms(), extra_hot_users=40, min_users=300_000)
    lens = mc.member_lengths(case)['user']
    assert (lens > case['cap']).sum() >= 41
    lr, wd, S0 = mc.hparams(case, 'adagrad', True)
    outs = []
    for _ in range(5):
        P = [t(case[k]) for k in TABLES]
        S = [t(s) for s in S0]
        losses = [gpu_step(P, S, case, 'adagrad', lr, wd) for _ in range(2)]
        outs.append((losses, P + S))
    for losses, tabs in outs[1:]:
        assert losses == outs[0][0], (losses, outs[0][0])
        for x, y in zip(tabs, outs[0][1]):
            assert torch.equal(x, y)


# ------------------------------------------------------------------ fit()

@pytest.mark.parametrize('opt', ['sgd', 'adagrad'])
@pytest.mark.parametrize('loss', LOSSES)
def test_fit_epoch_route_with_weight_decay(loss, opt, capsys):
    """ImplicitFactorizationModel.fit on the epoch route (plan stream, weight decay from the
    optimizer's hyper-parameters) against oracle.mf.fit from the same RandomState: 2 epochs,
    a short last batch.  Adagrad's final tables at 1e-3: its first-touch normalisation
    amplifies fp32 gradient differences (as in test_model_gpu) into differences on the scale
    of lr, so they also get 2e-3 lr absolute (the biases start at zero and stay within a few lr)."""
    from spotlight_b200 import optim
    from spotlight_b200.factorization.implicit import ImplicitFactorizationModel
    from spotlight_b200.interactions import Interactions
    rs = np.random.RandomState(51)
    U, I, D, n, B = 400, 300, 32, 5000, 1024
    users = rs.randint(0, U, n).astype(np.int32)
    items = rs.randint(0, I, n).astype(np.int32)
    inter = Interactions(users, items, num_users=U, num_items=I)
    lr, wd = (0.5, 1e-2) if opt == 'sgd' else (0.05, 1e-2)
    func = optim.fused_sgd(lr=lr, weight_decay=wd) if opt == 'sgd' else optim.fused_adagrad(lr=lr, weight_decay=wd)
    model = ImplicitFactorizationModel(loss=loss, embedding_dim=D, batch_size=B, n_iter=2, optimizer_func=func,
                                       use_cuda=True, random_state=np.random.RandomState(9))
    model._initialize(inter)
    assert model._route() == 'epoch'
    names = ['user_embeddings.weight', 'item_embeddings.weight', 'user_biases.weight', 'item_biases.weight']
    sd = model._net.state_dict()
    P64 = [sd[k].cpu().numpy().astype(np.float64) for k in names]
    S64 = [np.zeros(p.shape) for p in P64] if opt == 'adagrad' else None
    ref_rs = np.random.RandomState()
    ref_rs.set_state(model._random_state.get_state())
    model.fit(inter, verbose=True)
    lines = [l for l in capsys.readouterr().out.strip().split('\n') if l.startswith('Epoch')]
    losses = np.array([float(l.split('loss')[1]) for l in lines])
    ref_losses = omf.fit(P64, users, items, I, loss, B, 2, ref_rs, opt, lr, wd, 1e-10, S64)
    assert_close(losses, np.array(ref_losses), 1e-5, what='epoch losses')
    sd = model._net.state_dict()
    for k, p in zip(names, P64):
        assert_close(sd[k].cpu().numpy(), p, 1e-5 if opt == 'sgd' else 1e-3,
                     atol=1e-7 if opt == 'sgd' else 2e-3 * lr, what=k)
    st, rst = model._random_state.get_state(), ref_rs.get_state()
    assert (st[1] == rst[1]).all() and st[2] == rst[2]
