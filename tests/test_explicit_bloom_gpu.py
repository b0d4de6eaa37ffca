"""Explicit-feedback models with Bloom embedding layers on the fused hashed-table step
(csrc/mf.cu slb_mf_bloom_train_step with a rating loss: mf_fwd_bloom_rating_kernel, the
first-generation backward in modes 0 / 1 / 2, mf_apply_kernel<., 1> and the hash-bucket bias
update) against the float64 oracle (oracle/explicit_bloom.py).

Cases come from oracle/explicit_bloom_cases.py: every LPR with exact and non-exact widths, a
Bloom user or item layer or both, up to 24 hashes, padding ids 0 / 3 / none, hot rows around
seg_sort_cap and bias bucket collisions.  Dense mode is held at 1e-5 of the oracle's max (frozen
rows exactly 0); in-place mode compares the update (new - old) and the Adagrad state change at
1e-5 of the oracle's max, and every entry the oracle leaves untouched must stay bit-identical.
"""

import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import assert_close, load_golden
from oracle import bloom as ob
from oracle import explicit_bloom as oeb
from oracle import explicit_bloom_cases as ebc
from oracle.murmur import SEEDS

pytestmark = pytest.mark.gpu

TABLES = ('Wu', 'Wi', 'bu', 'bi')
OPT_WD = (('sgd', False), ('sgd', True), ('adagrad', False), ('adagrad', True))
MATRIX = ebc.matrix()
IDS = ['%d-%s-%d,%d-pad%d' % e[:5] for e in MATRIX]
_CASES = {}


def case_of(entry):
    if entry not in _CASES:
        _CASES[entry] = ebc.case_for(*entry)
    return _CASES[entry]


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def seeds(H):
    return list(SEEDS[:H])


def dense_step(case, want_scores=True):
    from spotlight_b200 import _lib, ops
    return ops.mf_bloom_rating_step(*[t(case[k]) for k in TABLES], t(case['users']), t(case['items']),
                                    t(case['ratings']), _lib.LOSS_KIND[case['loss']], seeds(case['Hu']),
                                    seeds(case['Hi']), case['pad_u'], case['pad_i'], want_scores)


def gpu_fused(P, S, case, opt, lr, wd):
    from spotlight_b200 import _lib, ops
    kind = _lib.OPT_SGD if opt == 'sgd' else _lib.OPT_ADAGRAD
    out = ops.mf_bloom_train_step_inplace(*P, t(case['users']), t(case['items']), None, case['loss'], 1,
                                          seeds(case['Hu']), seeds(case['Hi']), case['pad_u'], case['pad_i'], kind,
                                          lr, states=S, weight_decay=wd, ratings=t(case['ratings']))
    return out.item()


def compare(got, want, old, touched, what, rtol=1e-5):
    got = got.detach().cpu().numpy().astype(np.float64).reshape(old.shape)
    old = old.astype(np.float64)
    assert_close(got - old, want.reshape(old.shape) - old, rtol, what=what)
    rows = ~touched
    assert (got[rows] == old[rows]).all(), '%s: an untouched entry changed' % what


def run_and_check(case, opt, wd_on, steps=1):
    lr, wd, S0 = ebc.hparams(case, opt, wd_on)
    P0 = [case[k] for k in TABLES]
    P, S = [t(p.copy()) for p in P0], ([t(s.copy()) for s in S0] if S0 else None)
    P64 = ebc.bc.tables64(case)
    S64 = [s.astype(np.float64) for s in S0] if S0 else None
    touched = [np.zeros(p.shape[0], dtype=bool) for p in P0]
    for _ in range(steps):
        loss = gpu_fused(P, S, case, opt, lr, wd)
        ref = ebc.step(case, P64, opt, lr, wd, S64)
        assert_close(loss, ref['loss'], 1e-5, what='loss')
        touched = [a | b for a, b in zip(touched, ref['touched'])]
    for k, (p, nm) in enumerate(zip(P, TABLES)):
        compare(p, P64[k], P0[k], touched[k], nm)
        if S:
            compare(S[k], S64[k], S0[k], touched[k], 's' + nm)


# ------------------------------------------------------------------ matrix

@pytest.mark.parametrize('entry', MATRIX, ids=IDS)
def test_dense_vs_oracle(entry):
    case = case_of(entry)
    l, pos, dWu, dWi, dbu, dbi = [o.cpu().numpy() for o in dense_step(case)]
    ref = ebc.step(case)
    assert_close(l, ref['loss'], 1e-5, what='loss')
    assert_close(pos, ref['pos'], 1e-5, what='pos')
    for got, nm in zip((dWu, dWi, dbu, dbi), ('dWu', 'dWi', 'dbu', 'dbi')):
        assert_close(got, ref[nm], 1e-5, what=nm)
    for got, H, pad in ((dWu, case['Hu'], case['pad_u']), (dWi, case['Hi'], case['pad_i'])):
        fr = ob.frozen_row(H, pad)
        if fr >= 0:
            assert (got[fr] == 0).all(), 'the frozen row has a gradient'


@pytest.mark.parametrize('entry', MATRIX, ids=IDS)
def test_fused_vs_oracle(entry):
    """Each entry with one (optimizer, weight decay) pair cycling, and once more with weight decay."""
    k = MATRIX.index(entry)
    case = case_of(entry)
    opt, wd_on = OPT_WD[k % 4]
    run_and_check(case, opt, wd_on)
    if not wd_on:
        run_and_check(case, 'adagrad' if k % 2 else 'sgd', True)


def test_adagrad_weight_decay_three_steps():
    """Three Adagrad + weight-decay steps with the state carried over (Bloom on both sides)."""
    run_and_check(ebc.make_case(32, 'regression', 2, 3, 0, seed=92), 'adagrad', True, steps=3)


def test_rating_and_pairwise_steps_share_no_workspace():
    """Dense pairwise and rating steps of the same shapes and batch, interleaved: each loss family
    keeps its own workspace, so neither runs on the other's layout."""
    from spotlight_b200 import _lib, ops
    case = ebc.make_case(32, 'poisson', 0, 3, 0, seed=93)
    negs = case['items'][::-1].copy()
    pair_ref = ob.step(ebc.bc.tables64(case), case['users'], case['items'], negs, 'bpr', case['Hu'], case['Hi'],
                       case['pad_u'], case['pad_i'])
    rating_ref = ebc.step(case)
    for _ in range(2):
        out = ops.mf_bloom_train_step(*[t(case[k]) for k in TABLES], t(case['users']), t(case['items']), t(negs),
                                      _lib.LOSS_KIND['bpr'], 1, seeds(case['Hu']), seeds(case['Hi']), case['pad_u'],
                                      case['pad_i'], False)
        assert_close(out[0].item(), pair_ref['loss'], 1e-5, what='bpr loss')
        assert_close(out[4].cpu().numpy(), pair_ref['dWi'], 1e-5, what='bpr dWi')
        out = dense_step(case, want_scores=False)
        assert_close(out[0].item(), rating_ref['loss'], 1e-5, what='rating loss')
        assert_close(out[3].cpu().numpy(), rating_ref['dWi'], 1e-5, what='rating dWi')
        assert_close(out[5].cpu().numpy(), rating_ref['dbi'], 1e-5, what='rating dbi')


def test_bit_reproducible():
    case = ebc.make_case(64, 'logistic', 2, 3, 3, seed=94)
    lr, wd, S0 = ebc.hparams(case, 'adagrad', True)
    outs = []
    for _ in range(2):
        P, S = [t(case[k]) for k in TABLES], [t(s) for s in S0]
        loss = gpu_fused(P, S, case, 'adagrad', lr, wd)
        outs.append((loss, P + S))
    assert outs[0][0] == outs[1][0]
    for x, y in zip(outs[0][1], outs[1][1]):
        assert torch.equal(x, y)


# ------------------------------------------------------------------ the model

def _bloom_net(U, I, D, Hu, Hi, seed=3):
    from spotlight_b200.factorization.representations import BilinearNet
    from spotlight_b200.layers import BloomEmbedding, ScaledEmbedding
    torch.manual_seed(seed)
    rep = BilinearNet(U, I, D,
                      user_embedding_layer=(BloomEmbedding(U, D, compression_ratio=0.5, num_hash_functions=Hu)
                                            if Hu else ScaledEmbedding(U, D)),
                      item_embedding_layer=BloomEmbedding(I, D, compression_ratio=0.3, num_hash_functions=Hi))
    with torch.no_grad():
        rep.user_biases.weight.normal_(0, 0.1)
        rep.item_biases.weight.normal_(0, 0.1)
    return rep


def _model(rep, loss, func, n_iter=2, batch=512, sparse=False):
    from spotlight_b200.factorization.explicit import ExplicitFactorizationModel
    return ExplicitFactorizationModel(loss=loss, batch_size=batch, n_iter=n_iter, representation=rep,
                                      optimizer_func=func, use_cuda=True, sparse=sparse,
                                      random_state=np.random.RandomState(9))


def _params(model):
    net = model._net
    spec = net.fused_spec()
    return (spec['Wu'], spec['Wi'], net.user_biases.weight, net.item_biases.weight), spec


def _fit_against_oracle(model, inter, users, items, ratings, loss, opt, lr, wd, Hu, Hi, capsys, fits=1):
    """fit() (``fits`` calls of n_iter epochs each) against oracle.explicit_bloom.fit from the
    same RandomState and weights; tolerances as the implicit hashed-table fit() test."""
    params, spec = _params(model)
    P64 = [p.detach().cpu().numpy().astype(np.float64) for p in params]
    S64 = [np.zeros(p.shape) for p in P64] if opt == 'adagrad' else None
    ref_rs = np.random.RandomState()
    ref_rs.set_state(model._random_state.get_state())
    for _ in range(fits):
        model.fit(inter, verbose=True)
    lines = [l for l in capsys.readouterr().out.strip().split('\n') if l.startswith('Epoch')]
    losses = np.array([float(l.split('loss')[1]) for l in lines])
    ref = oeb.fit(P64, users, items, ratings, loss, model._batch_size, model._n_iter * fits, ref_rs, opt, lr, Hu, Hi,
                  spec['user_pad'], spec['item_pad'], wd, 1e-10, S64)
    assert_close(losses, np.array(ref), 1e-5, what='epoch losses')
    for p, want, nm in zip(params, P64, TABLES):
        assert_close(p.detach().cpu().numpy(), want, 1e-5 if opt == 'sgd' else 1e-3,
                     atol=1e-7 if opt == 'sgd' else 2e-3 * lr, what=nm)
    st, rst = model._random_state.get_state(), ref_rs.get_state()
    assert (st[1] == rst[1]).all() and st[2] == rst[2]


def _data(loss, U, I, n=3000, seed=51):
    from spotlight_b200.interactions import Interactions
    rs = np.random.RandomState(seed)
    users, items = rs.randint(0, U, n).astype(np.int32), rs.randint(0, I, n).astype(np.int32)
    ratings = ebc.ratings(loss, rs, n)
    return Interactions(users, items, ratings=ratings, num_users=U, num_items=I), users, items, ratings


@pytest.mark.parametrize('wd', [0.0, 1e-2])
@pytest.mark.parametrize('opt', ['sgd', 'adagrad'])
@pytest.mark.parametrize('Hu,Hi,loss', [(0, 3, 'regression'), (2, 3, 'poisson'), (0, 2, 'logistic')])
def test_fit_bloom_fused_route(Hu, Hi, loss, opt, wd, capsys):
    """fit() through _fit_epoch_bloom_fused against oracle.explicit_bloom.fit from the same
    RandomState: two epochs, a short last batch (3000 = 5 * 512 + 440)."""
    from spotlight_b200 import optim
    U, I, D = 300, 2000, 32
    lr = 0.1 if opt == 'sgd' else 0.05
    func = optim.fused_sgd(lr=lr, weight_decay=wd) if opt == 'sgd' else optim.fused_adagrad(lr=lr, weight_decay=wd)
    inter, users, items, ratings = _data(loss, U, I)
    model = _model(_bloom_net(U, I, D, Hu, Hi), loss, func)
    model._initialize(inter)
    assert model._route() == 'bloom'
    _fit_against_oracle(model, inter, users, items, ratings, loss, opt, lr, wd, Hu, Hi, capsys)


def test_second_fit_resumes(capsys):
    """Two fit() calls of one epoch each equal one two-epoch oracle run: the second call resumes
    from the current weights and the Adagrad state."""
    from spotlight_b200 import optim
    U, I, D = 300, 2000, 32
    inter, users, items, ratings = _data('regression', U, I, seed=52)
    model = _model(_bloom_net(U, I, D, 2, 3), 'regression', optim.fused_adagrad(lr=0.05, weight_decay=1e-3), n_iter=1)
    model._initialize(inter)
    assert model._route() == 'bloom'
    _fit_against_oracle(model, inter, users, items, ratings, 'regression', 'adagrad', 0.05, 1e-3, 2, 3, capsys,
                        fits=2)


@pytest.mark.parametrize('name,opt', [('fit_explicit_bloom_sgd', 'sgd'), ('fit_explicit_bloom_adagrad', 'adagrad')])
def test_fit_reproduces_reference_fixture(name, opt):
    """fit_explicit_bloom_*.npz: two epochs of the reference's fit() with a Bloom item layer under
    torch.optim.SGD / Adagrad (wd = 0), through fused_sgd / fused_adagrad on the hashed step."""
    from spotlight_b200 import optim
    from spotlight_b200.evaluation import rmse_score
    from spotlight_b200.factorization.explicit import ExplicitFactorizationModel
    from spotlight_b200.factorization.representations import BilinearNet
    from spotlight_b200.interactions import Interactions
    from spotlight_b200.layers import BloomEmbedding, ScaledEmbedding
    g = load_golden(name)
    U, I, D, H = int(g['num_users']), int(g['num_items']), int(g['dim']), int(g['bloom_H'])
    loss, lr = str(g['loss_kind']), float(g['lr'])
    rep = BilinearNet(U, I, D, user_embedding_layer=ScaledEmbedding(U, D),
                      item_embedding_layer=BloomEmbedding(I, D, compression_ratio=float(g['bloom_ratio']),
                                                          num_hash_functions=H))
    rep.load_state_dict({k[5:]: torch.from_numpy(v) for k, v in g.items() if k.startswith('init.')})
    func = optim.fused_sgd(lr=lr) if opt == 'sgd' else optim.fused_adagrad(lr=lr)
    model = ExplicitFactorizationModel(loss=loss, embedding_dim=D, batch_size=int(g['batch']),
                                       n_iter=int(g['n_iter']), representation=rep, optimizer_func=func,
                                       use_cuda=True, random_state=np.random.RandomState(0))
    inter = Interactions(g['users'], g['items'], ratings=g['ratings'], num_users=U, num_items=I)
    model._initialize(inter)
    model._random_state.set_state(('MT19937', g['rs0_key'], int(g['rs0_pos'])))
    assert model._route() == 'bloom'
    model.fit(inter)
    rtol, atol = (1e-5, 1e-7) if opt == 'sgd' else (1e-3, 2e-3 * lr)
    sd = model._net.state_dict()
    for k in sd:
        assert_close(sd[k].cpu().numpy(), g['final.' + k], rtol, atol=atol, what=k)
    st = model._random_state.get_state()
    assert (st[1] == g['rs_key']).all() and st[2] == int(g['rs_pos'])
    assert_close(model.predict(int(g['predict_user'])), g['predict'], rtol, atol=1e-4, what='predict')
    test = Interactions(g['test_users'], g['test_items'], ratings=g['test_ratings'], num_users=U, num_items=I)
    assert_close(rmse_score(model, test), g['rmse'], rtol, what='rmse')


def test_route_selection():
    """'bloom' for a Bloom BilinearNet under fused SGD / Adagrad; 'generic' under torch.optim,
    FusedAdam, the default Adam, a sparse model and a non-Bloom custom layer."""
    from spotlight_b200 import optim
    from spotlight_b200.factorization.representations import BilinearNet
    from spotlight_b200.layers import ScaledEmbedding
    U, I, D = 50, 80, 16
    inter, _, _, _ = _data('regression', U, I, n=200)

    class Custom(ScaledEmbedding):
        pass

    cases = [
        (_bloom_net(U, I, D, 0, 2), optim.fused_sgd(lr=0.1), False, 'bloom'),
        (_bloom_net(U, I, D, 2, 2), optim.fused_adagrad(lr=0.1), False, 'bloom'),
        (_bloom_net(U, I, D, 0, 2), lambda p: torch.optim.SGD(p, lr=0.1), False, 'generic'),
        (_bloom_net(U, I, D, 0, 2), lambda p: torch.optim.Adagrad(p, lr=0.1), False, 'generic'),
        (_bloom_net(U, I, D, 0, 2), lambda p: optim.FusedAdam(p, lr=0.1), False, 'generic'),
        (_bloom_net(U, I, D, 0, 2), None, False, 'generic'),
        (_bloom_net(U, I, D, 0, 2), optim.fused_sgd(lr=0.1), True, 'generic'),
        (BilinearNet(U, I, D, item_embedding_layer=Custom(I, D)), optim.fused_sgd(lr=0.1), False, 'generic'),
    ]
    for k, (rep, func, sparse, want) in enumerate(cases):
        model = _model(rep, 'regression', func, n_iter=1, batch=64, sparse=sparse)
        model._initialize(inter)
        assert model._route() == want, (k, model._route(), want)
        if not isinstance(model._optimizer, optim.FusedAdam):     # its flush() takes plain tables only
            model.fit(inter)


# ------------------------------------------------------------------ the C ABI

def _abi_args(case, bufs):
    """A valid dense-mode rating-loss slb_mf_bloom_args for ``case``."""
    from spotlight_b200 import _lib, ops
    P = [t(case[k]) for k in TABLES]
    users, items, ratings = t(case['users']), t(case['items']), t(case['ratings'])
    x = ops._bloom_args(*P, users, items, None, ratings, case['loss'], 1, seeds(case['Hu']), seeds(case['Hi']),
                        case['pad_u'], case['pad_i'])
    loss_out = torch.full((1,), float('nan'), device='cuda')
    grads = [torch.zeros_like(p) for p in P]
    a = x.base
    a.loss_out = loss_out.data_ptr()
    a.grad_mode = _lib.GRAD_DENSE
    a.dWu, a.dWi, a.dbu, a.dbi = [g.data_ptr() for g in grads]
    need = _lib.load().slb_mf_bloom_workspace_bytes(ctypes.byref(x))
    ws = torch.zeros(need, dtype=torch.uint8, device='cuda')
    a.workspace, a.workspace_bytes = ws.data_ptr(), need
    bufs.extend(P + [users, items, ratings, loss_out, ws] + grads)
    return x, loss_out, grads


def test_c_abi_rejects_bad_rating_arguments():
    """A rating loss with no ratings, with negatives, n_neg > 1, a neg_out or bias-pair buffers is
    refused with SLB_EINVAL before any launch: the loss and the gradients stay unwritten."""
    from spotlight_b200 import _lib, ops
    lib = _lib.load()
    case = ebc.make_case(16, 'regression', 0, 3, 0, seed=95, hot=False, B=64)
    keep = []
    spare = torch.zeros(64, dtype=torch.int64, device='cuda')
    spare_f = torch.zeros(64, device='cuda')

    def no_ratings(x):
        x.base.ratings = None

    def with_negs(x):
        x.base.negs = spare.data_ptr()

    def two_negs(x):
        x.base.n_neg = 2

    def with_neg_out(x):
        x.base.neg_out = spare_f.data_ptr()

    def with_pairs(x):
        x.pair_ids_u, x.pair_g_u = spare.data_ptr(), spare_f.data_ptr()

    def with_item_pairs(x):
        x.pair_ids_i, x.pair_g_i = spare.data_ptr(), spare_f.data_ptr()

    for bad in (no_ratings, with_negs, two_negs, with_neg_out, with_pairs, with_item_pairs):
        x, loss_out, grads = _abi_args(case, keep)
        bad(x)
        rc = lib.slb_mf_bloom_train_step(ctypes.byref(x), ops._stream())
        assert rc == -1, (bad.__name__, rc)
        torch.cuda.synchronize()
        assert torch.isnan(loss_out).all(), bad.__name__
        assert all(not g.any() for g in grads), bad.__name__
    # the same arguments, unmodified, run
    x, loss_out, grads = _abi_args(case, keep)
    assert lib.slb_mf_bloom_train_step(ctypes.byref(x), ops._stream()) == 0
    assert_close(loss_out.item(), ebc.step(case)['loss'], 1e-5, what='loss')


# ------------------------------------------------------------------ kernel names

def _profiled_kernel_names():
    """Kernel names of one dense and one in-place step per D of the matrix and one pairwise step,
    as torch.profiler records them."""
    from torch.profiler import ProfilerActivity, profile
    from spotlight_b200 import _lib, ops
    picks = {}
    for e in MATRIX:
        picks.setdefault(e[0], e)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for e in picks.values():
            case = case_of(e)
            dense_step(case, want_scores=False)
            gpu_fused([t(case[k]) for k in TABLES], None, case, 'sgd', 1e-3, 0.0)
        case = case_of(picks[32])
        ops.mf_bloom_train_step(*[t(case[k]) for k in TABLES], t(case['users']), t(case['items']),
                                t(case['users'] % case['NI']), _lib.LOSS_KIND['bpr'], 1, seeds(case['Hu']),
                                seeds(case['Hi']), case['pad_u'], case['pad_i'], False)
        torch.cuda.synchronize()
    return sorted({ev.name.replace(' ', '') for ev in prof.events()
                   if ev.device_type == torch.autograd.DeviceType.CUDA})


def test_profiler_sees_every_variant():
    """The matrix launches mf_fwd_bloom_rating_kernel at all six LPRs; the pairwise losses still
    launch mf_fwd_bloom_kernel under its own name.  The profiling runs in a child process, so its
    profiler session does not share this process's CUPTI state with the other suites' profiler
    tests."""
    here = os.path.dirname(os.path.abspath(__file__))
    code = ('import json, sys; sys.path.insert(0, %r); sys.path.insert(0, %r); '
            'import test_explicit_bloom_gpu as m; print(json.dumps(m._profiled_kernel_names()))'
            % (os.path.dirname(here), here))
    out = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, cwd=os.path.dirname(here),
                         timeout=600)
    assert out.returncode == 0, out.stderr[-4000:]
    names = json.loads(out.stdout.strip().split('\n')[-1])
    want = ['mf_fwd_bloom_rating_kernel<%d>' % l for l in (1, 2, 4, 8, 16, 32)] + ['mf_fwd_bloom_kernel<8>']
    want += ['mf_bwd_tile_kernel<%d,%d,32,' % (l, m) for m in (0, 1, 2) for l in (8, 32)]
    want += ['mf_apply_kernel<%d,1>' % l for l in (1, 32)] + ['bias_apply_kernel']
    for w in want:
        assert any(w in n for n in names), (w, [n for n in names if 'mf_' in n or 'bias' in n])
