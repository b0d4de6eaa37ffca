"""The hashed-table (Bloom) MF step (csrc/mf.cu slb_mf_bloom_train_step: mf_fwd_bloom_kernel, the
first-generation backward in modes 0 / 1 / 2, mf_apply_kernel<., 1> and the hash-bucket bias update)
against the float64 oracle (oracle/bloom.py).

Cases come from oracle/bloom_cases.py: every LPR with exact and non-exact widths, hash counts from
plain tables to 24 hashes on one side and Bloom on both, padding ids 0 / 3 / none, ids on row 0 and
on the frozen row, repeated rows of one id, hot rows around seg_sort_cap, bias bucket collisions.
Dense mode is held at 1e-5 of the oracle's max (frozen rows exactly 0); fused mode compares the
update (new - old) and the Adagrad state change at 1e-5 of the oracle's max, and every entry the
oracle leaves untouched must stay bit-identical.
"""

import numpy as np
import pytest
import torch

from conftest import assert_close, load_golden
from oracle import bloom as ob
from oracle import bloom_cases as bc
from oracle.murmur import SEEDS

pytestmark = pytest.mark.gpu

TABLES = ('Wu', 'Wi', 'bu', 'bi')
OPT_WD = (('sgd', False), ('sgd', True), ('adagrad', False), ('adagrad', True))
MATRIX = bc.matrix()
IDS = ['%d-%s%d-%d,%d-pad%d' % e[:6] for e in MATRIX]
_CASES = {}


def case_of(entry):
    if entry not in _CASES:
        _CASES[entry] = bc.case_for(*entry)
    return _CASES[entry]


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def seeds(H):
    return list(SEEDS[:H])


def gpu_fused(P, S, case, opt, lr, wd, users=None, items=None, negs=None):
    from spotlight_b200 import _lib, ops
    kind = _lib.OPT_SGD if opt == 'sgd' else _lib.OPT_ADAGRAD
    u, i, j = (case[k] if x is None else x for k, x in (('users', users), ('items', items), ('negs', negs)))
    out = ops.mf_bloom_train_step_inplace(*P, t(u), t(i), t(j), case['loss'], case['n_neg'], seeds(case['Hu']),
                                          seeds(case['Hi']), case['pad_u'], case['pad_i'], kind, lr, states=S,
                                          weight_decay=wd)
    return out.item()


def oracle_fused(P64, S64, case, opt, lr, wd, users=None, items=None, negs=None):
    u, i, j = (case[k] if x is None else x for k, x in (('users', users), ('items', items), ('negs', negs)))
    return ob.step(P64, u, i, j, case['loss'], case['Hu'], case['Hi'], case['pad_u'], case['pad_i'],
                   case['n_neg'], opt, lr, wd, 1e-10, S64)


def compare(got, want, old, touched, what, rtol=1e-5):
    got = got.detach().cpu().numpy().astype(np.float64).reshape(old.shape)
    old = old.astype(np.float64)
    assert_close(got - old, want.reshape(old.shape) - old, rtol, what=what)
    rows = ~touched
    assert (got[rows] == old[rows]).all(), '%s: an untouched entry changed' % what


def run_and_check(case, opt, wd_on, steps=1):
    lr, wd, S0 = bc.hparams(case, opt, wd_on)
    P0 = [case[k] for k in TABLES]
    P, S = [t(p.copy()) for p in P0], ([t(s.copy()) for s in S0] if S0 else None)
    P64 = bc.tables64(case)
    S64 = [s.astype(np.float64) for s in S0] if S0 else None
    touched = [np.zeros(p.shape[0], dtype=bool) for p in P0]
    for _ in range(steps):
        loss = gpu_fused(P, S, case, opt, lr, wd)
        ref = oracle_fused(P64, S64, case, opt, lr, wd)
        assert_close(loss, ref['loss'], 1e-5, what='loss')
        touched = [a | b for a, b in zip(touched, ref['touched'])]
    for k, (p, nm) in enumerate(zip(P, TABLES)):
        compare(p, P64[k], P0[k], touched[k], nm)
        if S:
            compare(S[k], S64[k], S0[k], touched[k], 's' + nm)
    return ref


# ------------------------------------------------------------------ matrix

@pytest.mark.parametrize('entry', MATRIX, ids=IDS)
def test_dense_vs_oracle(entry):
    from spotlight_b200 import _lib, ops
    case = case_of(entry)
    out = ops.mf_bloom_train_step(*[t(case[k]) for k in TABLES], t(case['users']), t(case['items']),
                                  t(case['negs']), _lib.LOSS_KIND[case['loss']], case['n_neg'], seeds(case['Hu']),
                                  seeds(case['Hi']), case['pad_u'], case['pad_i'], True)
    l, pos, neg, dWu, dWi, dbu, dbi = [o.cpu().numpy() for o in out]
    ref = bc.scores(case)
    assert_close(l, ref['loss'], 1e-5, what='loss')
    assert_close(pos, ref['pos'], 1e-5, what='pos')
    assert_close(neg, ref['neg'], 1e-5, what='neg')
    for got, nm in zip((dWu, dWi, dbu, dbi), ('dWu', 'dWi', 'dbu', 'dbi')):
        assert_close(got, ref[nm], 1e-5, what=nm)
    for got, H, pad in ((dWu, case['Hu'], case['pad_u']), (dWi, case['Hi'], case['pad_i'])):
        fr = ob.frozen_row(H, pad)
        if fr >= 0:
            assert (got[fr] == 0).all(), 'the frozen row has a gradient'


@pytest.mark.parametrize('entry', MATRIX, ids=IDS)
def test_fused_vs_oracle(entry):
    """Each entry with one (optimizer, weight decay) pair cycling, and once with weight decay."""
    k = MATRIX.index(entry)
    case = case_of(entry)
    opt, wd_on = OPT_WD[k % 4]
    run_and_check(case, opt, wd_on)
    if not wd_on:
        run_and_check(case, 'adagrad' if k % 2 else 'sgd', True)


@pytest.mark.parametrize('Hu,Hi', [(0, 0), (0, 4)])
def test_large_batch_grid_stride(Hu, Hi):
    """B > 8448: mf_fwd_bloom_kernel's grid-stride loop runs twice at LPR = 32."""
    case = bc.make_case(128, 'bpr', Hu, Hi, 0, seed=77 + Hu + Hi, B=9000)
    run_and_check(case, 'adagrad', True)


def _tiny_case(D, loss, n, Hu, Hi, pad, B, seed):
    rs = np.random.RandomState(seed)
    NU, NI = 50, 70
    Mu, Mi = (13 if Hu else NU), (17 if Hi else NI)
    su, si = D ** 0.25 * np.sqrt(max(Hu, 1)), D ** 0.25 * np.sqrt(max(Hi, 1))     # dots ~ N(0, 1)
    return dict(D=D, B=B, loss=loss, n_neg=n, Hu=Hu, Hi=Hi, pad_u=pad if Hu else -1, pad_i=pad if Hi else -1,
                NU=NU, NI=NI, Wu=(rs.randn(Mu, D) / su).astype(np.float32), Wi=(rs.randn(Mi, D) / si).astype(np.float32), bu=(rs.randn(NU, 1) * 0.1).astype(np.float32),
                bi=(rs.randn(NI, 1) * 0.1).astype(np.float32), users=rs.randint(0, NU, B).astype(np.int64),
                items=rs.randint(0, NI, B).astype(np.int64), negs=rs.randint(0, NI, B * n).astype(np.int64))


@pytest.mark.parametrize('D', [4, 100])
def test_batch_of_one_and_a_few(D):
    for loss, n in (('bpr', 1), ('pointwise', 1), ('adaptive_hinge', 3)):
        run_and_check(_tiny_case(D, loss, n, 2, 3, 3, 1, D), 'adagrad', True)
        run_and_check(_tiny_case(D, loss, n, 0, 24, 0, 37, D + 1), 'sgd', True)


# ------------------------------------------------------------------ trajectory, reuse, determinism

def test_adagrad_weight_decay_three_steps():
    """Three Adagrad + weight-decay steps with the state carried over (Bloom on both sides)."""
    run_and_check(bc.make_case(32, 'bpr', 2, 3, 0, seed=92), 'adagrad', True, steps=3)


def test_workspace_reuse_after_a_hot_batch():
    """A hot batch, then a hot-free batch with the same shapes and B, on one workspace."""
    hot = bc.make_case(32, 'pointwise', 0, 4, 0, seed=91)
    rs = np.random.RandomState(5)
    B = hot['B']
    cool = dict(hot, users=rs.randint(0, hot['NU'], B), items=rs.randint(0, hot['NI'], B),
                negs=rs.randint(0, hot['NI'], B))
    for case in (hot, cool, hot):
        run_and_check(case, 'adagrad', True)


def test_bit_reproducible():
    case = bc.make_case(64, 'hinge', 2, 3, 3, seed=93)
    lr, wd, S0 = bc.hparams(case, 'adagrad', True)
    outs = []
    for _ in range(2):
        P, S = [t(case[k]) for k in TABLES], [t(s) for s in S0]
        loss = gpu_fused(P, S, case, 'adagrad', lr, wd)
        outs.append((loss, P + S))
    assert outs[0][0] == outs[1][0]
    for x, y in zip(outs[0][1], outs[1][1]):
        assert torch.equal(x, y)


# ------------------------------------------------------------------ the sparse bias update

@pytest.mark.parametrize('n', [1, 2047, 2048, 2049, 2 ** 20 + 3])
@pytest.mark.parametrize('opt,wd_on', OPT_WD, ids=['sgd', 'sgd_wd', 'adagrad', 'adagrad_wd'])
def test_bias_sparse_apply(n, opt, wd_on):
    """(id, g) pairs with ids equal modulo the bucket count, one id repeated, and g == 0 padding
    pairs (which touch nothing)."""
    from spotlight_b200 import _lib, ops
    rs = np.random.RandomState(n)
    nb = 4096
    while nb < 2 * n:
        nb <<= 1
    N = max(3_000_000, 2 * nb + 1000)          # ids up to 17 + 2 nb are in the table
    ids = rs.randint(0, N, n).astype(np.int64)
    if n > 8:
        ids[:3] = [17, 17 + nb, 17 + 2 * nb]
        ids[3:3 + min(150, n // 4)] = N - 1
    g = rs.randn(n).astype(np.float32)
    g[rs.rand(n) < 0.2] = 0.0
    b0 = (rs.randn(N) * 0.1).astype(np.float32)
    s0 = rs.uniform(0.5, 1.5, N).astype(np.float32)
    lr, wd = 0.1, (0.3 if wd_on else 0.0)
    b, s = t(b0.copy()), t(s0.copy())
    kind = _lib.OPT_SGD if opt == 'sgd' else _lib.OPT_ADAGRAD
    ops.bias_sparse_apply(t(ids), t(g), b, s if opt == 'adagrad' else None, kind, lr, wd)
    live = g != 0
    gs = np.zeros(N)
    np.add.at(gs, ids[live], g[live].astype(np.float64))
    touched = np.zeros(N, dtype=bool)
    touched[ids[live]] = True
    B64, S64 = b0.astype(np.float64), s0.astype(np.float64)
    from oracle.explicit import apply_rowwise
    apply_rowwise((B64,), (gs,), (touched,), opt, lr, (wd,), 1e-10, (S64,))
    compare(b, B64, b0, touched, 'bias')
    if opt == 'adagrad':
        compare(s, S64, s0, touched, 'state')


# ------------------------------------------------------------------ pairs mode

@pytest.mark.parametrize('loss', ['bpr', 'hinge', 'pointwise'])
def test_pairs_mode_sums_are_the_bias_gradients(loss):
    from spotlight_b200 import ops
    case = bc.make_case(64, loss, 0, 4, 0, seed=95)
    norm = 3 * case['B']
    lval, dWu, dWi, (iu, gu), (ii, gi) = ops.mf_bloom_step_pairs(
        *[t(case[k]) for k in TABLES], t(case['users']), t(case['items']), t(case['negs']), loss, seeds(4), 0,
        norm_batch=norm)
    ref = ob.step(bc.tables64(case), case['users'], case['items'], case['negs'], loss, 0, 4, -1, 0, norm=norm)
    assert_close(lval.item(), ref['loss'], 1e-5, what='loss')
    assert_close(dWu.cpu().numpy(), ref['dWu'], 1e-5, what='dWu')
    assert_close(dWi.cpu().numpy(), ref['dWi'], 1e-5, what='dWi')
    for (ids, g), want, N in (((iu, gu), ref['dbu'], case['NU']), ((ii, gi), ref['dbi'], case['NI'])):
        got = np.zeros(N)
        np.add.at(got, ids.cpu().numpy(), g.cpu().numpy().astype(np.float64))
        assert_close(got, want.reshape(-1), 1e-5, atol=1e-12, what='pair sums')


# ------------------------------------------------------------------ fit()

def _model(Hu, Hi, loss, opt, lr, wd, n_neg=2):
    from spotlight_b200 import optim
    from spotlight_b200.factorization.implicit import ImplicitFactorizationModel
    from spotlight_b200.factorization.representations import BilinearNet
    from spotlight_b200.layers import BloomEmbedding, ScaledEmbedding
    U, I, D = 300, 2000, 32
    torch.manual_seed(3)
    rep = BilinearNet(U, I, D,
                      user_embedding_layer=(BloomEmbedding(U, D, compression_ratio=0.5, num_hash_functions=Hu)
                                            if Hu else ScaledEmbedding(U, D)),
                      item_embedding_layer=BloomEmbedding(I, D, compression_ratio=0.3, num_hash_functions=Hi))
    with torch.no_grad():
        rep.user_biases.weight.normal_(0, 0.1)
        rep.item_biases.weight.normal_(0, 0.1)
    func = optim.fused_sgd(lr=lr, weight_decay=wd) if opt == 'sgd' else optim.fused_adagrad(lr=lr, weight_decay=wd)
    return ImplicitFactorizationModel(loss=loss, embedding_dim=D, batch_size=512, n_iter=2, representation=rep,
                                      optimizer_func=func, num_negative_samples=n_neg, use_cuda=True,
                                      random_state=np.random.RandomState(9)), U, I


@pytest.mark.parametrize('wd', [0.0, 1e-2])
@pytest.mark.parametrize('opt', ['sgd', 'adagrad'])
@pytest.mark.parametrize('Hu,Hi,loss', [(0, 3, 'bpr'), (2, 3, 'hinge'), (0, 2, 'adaptive_hinge')])
def test_fit_bloom_fused_route(Hu, Hi, loss, opt, wd, capsys):
    """fit() through _fit_epoch_bloom_fused against oracle.bloom.fit from the same RandomState:
    two epochs, a short last batch; tolerances as the planned step's fit() test."""
    from spotlight_b200.interactions import Interactions
    lr = 0.5 if opt == 'sgd' else 0.05
    model, U, I = _model(Hu, Hi, loss, opt, lr, wd)
    rs = np.random.RandomState(51)
    n = 3000
    users, items = rs.randint(0, U, n).astype(np.int32), rs.randint(0, I, n).astype(np.int32)
    inter = Interactions(users, items, num_users=U, num_items=I)
    model._initialize(inter)
    assert model._route() == 'bloom'
    spec = model._net.fused_spec()
    net = model._net
    params = (spec['Wu'], spec['Wi'], net.user_biases.weight, net.item_biases.weight)
    P64 = [p.detach().cpu().numpy().astype(np.float64) for p in params]
    S64 = [np.zeros(p.shape) for p in P64] if opt == 'adagrad' else None
    ref_rs = np.random.RandomState()
    ref_rs.set_state(model._random_state.get_state())
    model.fit(inter, verbose=True)
    lines = [l for l in capsys.readouterr().out.strip().split('\n') if l.startswith('Epoch')]
    losses = np.array([float(l.split('loss')[1]) for l in lines])
    ref = ob.fit(P64, users, items, I, loss, 512, 2, ref_rs, opt, lr, Hu, Hi, spec['user_pad'], spec['item_pad'],
                 model._n_neg(), wd, 1e-10, S64)
    assert_close(losses, np.array(ref), 1e-5, what='epoch losses')
    for p, want, nm in zip(params, P64, TABLES):
        assert_close(p.detach().cpu().numpy(), want, 1e-5 if opt == 'sgd' else 1e-3,
                     atol=1e-7 if opt == 'sgd' else 2e-3 * lr, what=nm)
    st, rst = model._random_state.get_state(), ref_rs.get_state()
    assert (st[1] == rst[1]).all() and st[2] == rst[2]


def test_fit_reproduces_reference_fixture():
    """fit_bloom_adagrad.npz: two epochs of the reference's fit() with a Bloom item layer and
    Adagrad (wd = 0), through fused_adagrad on the hashed step."""
    from spotlight_b200 import optim
    from spotlight_b200.factorization.implicit import ImplicitFactorizationModel
    from spotlight_b200.factorization.representations import BilinearNet
    from spotlight_b200.interactions import Interactions
    from spotlight_b200.layers import BloomEmbedding, ScaledEmbedding
    g = load_golden('fit_bloom_adagrad')
    U, I, D, H = int(g['num_users']), int(g['num_items']), int(g['dim']), int(g['bloom_H'])
    rep = BilinearNet(U, I, D, user_embedding_layer=ScaledEmbedding(U, D),
                      item_embedding_layer=BloomEmbedding(I, D, compression_ratio=float(g['bloom_ratio']),
                                                          num_hash_functions=H))
    rep.load_state_dict({k[5:]: torch.from_numpy(v) for k, v in g.items() if k.startswith('init.')})
    rs = np.random.RandomState()
    rs.set_state(('MT19937', g['rs0_key'], int(g['rs0_pos'])))
    model = ImplicitFactorizationModel(loss='bpr', embedding_dim=D, batch_size=int(g['batch']), n_iter=2,
                                       representation=rep, optimizer_func=optim.fused_adagrad(lr=float(g['lr'])),
                                       use_cuda=True, random_state=rs)
    inter = Interactions(g['users'], g['items'], num_users=U, num_items=I)
    model._initialize(inter)
    model._random_state.set_state(('MT19937', g['rs0_key'], int(g['rs0_pos'])))
    assert model._route() == 'bloom'
    model.fit(inter)
    sd = model._net.state_dict()
    for k in sd:
        assert_close(sd[k].cpu().numpy(), g['final.' + k], 1e-3, atol=2e-3 * float(g['lr']), what=k)
    st = model._random_state.get_state()
    assert (st[1] == g['rs_key']).all() and st[2] == int(g['rs_pos'])
    assert_close(model.predict(int(g['predict_user'])), g['predict'], 1e-3, atol=1e-4, what='predict')


# ------------------------------------------------------------------ kernel names

def test_profiler_sees_every_variant():
    """The matrix launches mf_fwd_bloom_kernel at all six LPRs, mf_bwd_tile_kernel in modes 0 / 1 / 2
    with exact and non-exact widths, mf_bwd_long_kernel in modes 0 / 1 / 2, mf_apply_kernel<., 1>
    and bias_apply_kernel."""
    from spotlight_b200 import _lib, ops
    from torch.profiler import ProfilerActivity, profile
    picks = {}
    for e in MATRIX:
        picks.setdefault(e[0], e)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for e in picks.values():
            case = case_of(e)
            P = [t(case[k]) for k in TABLES]
            ops.mf_bloom_train_step(*P, t(case['users']), t(case['items']), t(case['negs']),
                                    _lib.LOSS_KIND[case['loss']], case['n_neg'], seeds(case['Hu']),
                                    seeds(case['Hi']), case['pad_u'], case['pad_i'], False)
            gpu_fused(P, None, case, 'sgd', 1e-3, 0.0)
        torch.cuda.synchronize()
    names = {ev.name.replace(' ', '') for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA}
    want = ['mf_fwd_bloom_kernel<%d>' % l for l in (1, 2, 4, 8, 16, 32)]
    want += ['mf_bwd_tile_kernel<%d,%d,32,%s>' % (l, m, w) for m in (0, 1, 2) for l, w in
             ((8, 'true'), (8, 'false'), (16, 'false'), (32, 'false'), (32, 'true'))]
    want += ['mf_bwd_long_kernel<%d,%d>' % (l, m) for m in (0, 1, 2) for l in (1, 2)]
    want += ['mf_apply_kernel<%d,1>' % l for l in (1, 32)] + ['bias_apply_kernel']
    for w in want:
        assert any(w in n for n in names), (w, sorted(n for n in names if 'mf_' in n or 'bias' in n))
