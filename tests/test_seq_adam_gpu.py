"""Row-wise lazy-exact Adam in the fused sequence step (csrc/seq.cu seq_adam_prepass_kernel and
seq_reduce_adam_kernel, optim.FusedAdam) against the float64 oracles and torch.optim.Adam.

Step parity: several consecutive steps on one table, each against the oracle's gradients at the
oracle's own state, with oracle.adam.LazyAdamTable applying the same lazy scheme in float64.  The
moments are checked at 2e-5 of their scale.  An Adam step moves an element by at most ~lr, in the
direction of m / sqrt(v); where a gradient component is ~0 that direction is last-bit noise in both
fp32 and float64 (g / |g| on the first step), so the parameters are checked at 5 % of one step where
the first moment is above 1e-3 of its maximum, at half a step where it is between 1e-5 and 1e-3
(clearly non-zero, but its direction more sensitive), and within one step's bound on the rest."""

import numpy as np
import pytest
import torch

from conftest import assert_close
from oracle import lstm_cases as lc
from oracle import mixture_cases as mc
from oracle import seq_bloom as sb
from oracle import seq_cases as sc
from oracle.adam import LazyAdamTable
from oracle.murmur import bloom_rows

pytestmark = pytest.mark.gpu

LR = 1e-3


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to('cuda:0')


def _make(net, hashed, seed, **kw):
    if hashed:
        return sb.make_case(net, seed=seed, **kw)
    kw.pop('rows', None)
    kw.pop('H', None)
    if net in ('pool', 'cnn'):
        return sc.make_case(net, seed=seed, **kw)
    return (lc if net == 'lstm' else mc).make_case(seed=seed, **kw)


def _oracle(case, hashed):
    """(table gradient, bias gradient, updated table rows, updated bias ids)."""
    if hashed:
        ref = sb.step(case)
        rows, ids = sb.updated(case, ref)
        return ref['dW'], ref['dbias'], rows, ids
    net = case['net']
    ref = (sc.oracle_step(case) if net in ('pool', 'cnn') else
           lc.oracle_step(case) if net == 'lstm' else mc.oracle_step(case))
    rows = sc.updated_rows(case, ref)
    return ref['dE'], ref['dbias'], rows, rows


def _kwargs(case, hashed):
    kw = {}
    if hashed:
        kw['item_hash'] = dict(seeds=case['seeds'], padding_idx=0)
    if case['cnn'] is not None:
        kw['cnn'] = dict(case['cnn'], weights=[t(w) for w, _ in case['convs']], biases=[t(b) for _, b in case['convs']])
    if case['net'] in ('lstm', 'mixture'):
        kw['lstm'] = {k: t(v) for k, v in case['lstm'].items()}
    if case['net'] == 'mixture':
        kw['mixture'] = dict(num_mixtures=case['M'], w=t(case['proj']['w']), b=t(case['proj']['b']))
    return kw


def _check_param(dev, tab, what):
    w, m = dev.cpu().numpy().astype(np.float64), tab.m
    scale = np.abs(m).max()
    quiet = np.abs(m) < 1e-3 * scale
    noise = np.abs(m) < 1e-5 * scale          # at the fp32 gradient's own rounding level
    err = np.abs(w - tab.w)
    tol = 2e-6 * np.abs(tab.w).max()
    assert err[~quiet].max(initial=0.0) <= 0.05 * LR + tol, '%s: %.3e' % (what, err[~quiet].max())
    assert err[quiet & ~noise].max(initial=0.0) <= 0.5 * LR + tol, '%s (small moments): %.3e' % (
        what, err[quiet & ~noise].max(initial=0.0))
    assert err.max() <= 2.1 * LR, '%s moved by more than an Adam step' % what


STEPS = 4
NETS = [(net, hashed, wd) for net in ('pool', 'cnn', 'lstm', 'mixture') for hashed in (False, True) for wd in (0.0, 0.1)]


@pytest.mark.parametrize('net,hashed,wd', NETS, ids=['%s-%s-wd%g' % (n, 'hashed' if h else 'plain', w) for n, h, w in NETS])
def test_step_parity(net, hashed, wd):
    """Four steps; table, bias, exp_avg, exp_avg_sq and last after each.  The items (I = 2000, 24 or
    48 sequences of 10 a step) leave most rows untouched for several steps; the cases carry padding
    positions and the padding id as a negative; the pool case draws its targets Zipf-distributed
    and the hashed tables are small, so some rows have more terms than the reduction sorts in
    shared memory."""
    from spotlight_b200 import _lib, ops
    from spotlight_b200.optim import FusedAdam
    kw = dict(D=32, S=10, B=24, I=2000, loss='bpr', rows=8, H=3)
    if net == 'cnn':
        kw.update(kernel_width=(3,), dilation=(1,))
    if net == 'mixture':
        kw['M'] = 3
    if net == 'pool' and not hashed:
        kw.update(zipf=2.0, B=48)
    if hashed:
        kw.update(rows=4, B=48)
    base = _make(net, hashed, 11, **kw)
    key = 'W' if hashed else 'E'
    tabE = LazyAdamTable(base[key], lr=LR, weight_decay=wd)
    tabB = LazyAdamTable(base['bias'], lr=LR, weight_decay=wd)
    E, bias = t(base[key]), t(base['bias'])
    mE, vE, mb, vb = (torch.zeros_like(x) for x in (E, E, bias, bias))
    lastE = torch.zeros(E.shape[0], dtype=torch.int32, device='cuda:0')
    lastb = torch.zeros(bias.shape[0], dtype=torch.int32, device='cuda:0')
    sched = FusedAdam([torch.nn.Parameter(torch.zeros(1))], lr=LR).schedule(STEPS, torch.device('cuda:0'))
    hot = False
    for step in range(1, STEPS + 1):
        case = _make(net, hashed, 11 + 100 * step, **kw)
        for k in ('convs', 'lstm', 'proj'):
            if k in base:
                case[k] = base[k]
        ref_rows = np.concatenate([case['seqs'].ravel(), case['negs'].ravel()])
        if hashed:
            tabE.catch_up(bloom_rows(ref_rows, case['H'], tabE.w.shape[0]).ravel(), step - 1)
        else:
            tabE.catch_up(ref_rows, step - 1)
        tabB.catch_up(ref_rows, step - 1)
        case[key] = tabE.w.astype(np.float32)
        case['bias'] = tabB.w.astype(np.float32)
        if hashed:
            case['E'] = sb.virtual_table(case['W'], case['bias'].shape[0], case['H']).astype(np.float32)
        dE, db, rows, ids = _oracle(case, hashed)
        ids_in = case['seqs'][case['seqs'] != 0]
        if hashed:
            ids_in = bloom_rows(ids_in, case['H'], kw['rows']).ravel()
        hot |= bool(np.bincount(ids_in).max() > sc.seg_sort_cap(kw['D']))
        tabE.apply(np.flatnonzero(rows), dE[rows], step)
        tabB.apply(np.flatnonzero(ids), db[ids], step)
        fused = dict(kind=_lib.OPT_ADAM, lr=LR, weight_decay=wd, eps=1e-8, beta1=0.9, beta2=0.999,
                     state_E=mE, state_bias=mb, state2_E=vE, state2_bias=vb, last_E=lastE,
                     last_bias=lastb if hashed else None, sched=sched, step=step)
        out = ops.seq_train_step(E, bias, t(case['seqs']), t(case['negs']), case['loss'], case['n_neg'],
                                 fused=fused, **_kwargs(case, hashed))
        assert out['dE'] is None
        what = '%s step %d' % (net, step)
        assert_close(mE.cpu().numpy(), tabE.m, 2e-5, what=what + ' exp_avg')
        assert_close(vE.cpu().numpy(), tabE.v, 2e-5, what=what + ' exp_avg_sq')
        assert_close(mb.cpu().numpy(), tabB.m, 2e-5, what=what + ' bias exp_avg')
        assert_close(vb.cpu().numpy(), tabB.v, 2e-5, what=what + ' bias exp_avg_sq')
        _check_param(E, tabE, what + ' table')
        _check_param(bias, tabB, what + ' bias')
        assert (lastE.cpu().numpy() == tabE.last).all(), what + ' last'
        if hashed:
            assert (lastb.cpu().numpy() == tabB.last).all(), what + ' bias last'
    assert hot or not (hashed or net == 'pool')
    assert (tabB.last[1:] < STEPS - 1).any(), 'no item was left untouched for several steps'


# ------------------------------------------------------------------ model level
def _seqs(I, n=256, S=12, seed=17, hi=None):
    from spotlight_b200.interactions import SequenceInteractions
    rs = np.random.RandomState(seed)
    seqs = rs.randint(1, hi or I, (n, S)).astype(np.int32)
    for b in range(0, n, 3):
        seqs[b, :rs.randint(0, S)] = 0
    return SequenceInteractions(seqs, num_items=I)


def _fit(rep, opt_func, inter, D, state=None, n_iter=2, capsys=None):
    from spotlight_b200.sequence.implicit import ImplicitSequenceModel
    torch.manual_seed(0)
    model = ImplicitSequenceModel(loss='bpr', representation=rep, embedding_dim=D, batch_size=32, n_iter=n_iter,
                                  optimizer_func=opt_func, use_cuda=True,
                                  random_state=np.random.RandomState(5))
    model._initialize(inter)
    if state is not None:
        model._net.load_state_dict(state)
    init = {k: v.clone() for k, v in model._net.state_dict().items()}
    if capsys is not None:
        capsys.readouterr()
    model.fit(inter, verbose=True)
    losses = None
    if capsys is not None:
        lines = [l for l in capsys.readouterr().out.strip().split('\n') if l.startswith('Epoch')]
        losses = np.array([float(l.split('loss')[1]) for l in lines])
    return model, init, losses


FITS = [('pool', 0.0), ('cnn', 1e-3), ('lstm', 0.0), ('mixture', 1e-3)]


@pytest.mark.parametrize('rep,l2', FITS, ids=['%s-l2%g' % f for f in FITS])
def test_fit_equals_torch_adam_on_fused_route(rep, l2, capsys):
    """fit() with optim.fused_adam against torch.optim.Adam on the fused route (the dense gradient
    and table sweep) from the same init: 20000 items, sequences over the first 3000, so most rows
    are untouched by any step.  Tolerances as test_model_gpu.test_lazy_adam_equals_dense_adam."""
    from spotlight_b200 import optim
    I, D = 20000, 16
    inter = _seqs(I, hi=3000)
    rep = 'pooling' if rep == 'pool' else rep
    lazy, init, ll = _fit(rep, optim.fused_adam(lr=1e-2, weight_decay=l2), inter, D, capsys=capsys)
    dense, _, ld = _fit(rep, lambda p: torch.optim.Adam(p, lr=1e-2, weight_decay=l2), inter, D, state=init,
                        capsys=capsys)
    assert lazy._route() == 'fused' and dense._route() == 'fused'
    assert_close(ll, ld, 1e-5, what='epoch losses')
    for (k, a), (_, b) in zip(lazy._net.state_dict().items(), dense._net.state_dict().items()):
        assert_close(a.cpu().numpy(), b.cpu().numpy(), 5e-4, atol=1e-7, what=k)
    opt, W = lazy._optimizer, lazy._net.item_embeddings.weight
    st0, st1 = opt.state[W], dense._optimizer.state[dense._net.item_embeddings.weight]
    assert_close(st0['exp_avg'].cpu().numpy(), st1['exp_avg'].cpu().numpy(), 2e-3, atol=1e-9, what='exp_avg')
    assert_close(st0['exp_avg_sq'].cpu().numpy(), st1['exp_avg_sq'].cpu().numpy(), 2e-3, atol=1e-12, what='exp_avg_sq')
    assert int(st0['last'].min()) == opt.steps_taken == 2 * 8
    assert W.grad is None and lazy._net.item_biases.weight.grad is None


def _bloom(net, I, D, H=4, ratio=0.2):
    from spotlight_b200.layers import BloomEmbedding
    from spotlight_b200.sequence.representations import LSTMNet, MixtureLSTMNet, PoolNet, CNNNet
    emb = BloomEmbedding(I, D, compression_ratio=ratio, num_hash_functions=H, padding_idx=0)
    if net == 'mixture':
        return MixtureLSTMNet(I, D, num_mixtures=2, item_embedding_layer=emb)
    return {'pool': PoolNet, 'cnn': CNNNet, 'lstm': LSTMNet}[net](I, D, item_embedding_layer=emb)


@pytest.mark.parametrize('net', ['pool', 'lstm'])
def test_bloom_fit_fused_hashed_against_generic(net, capsys):
    """A Bloom item layer under fused_adam trains on the fused_hashed route, with no .grad on the
    tables; against the generic route (autograd through the Bloom gather) under torch.optim.Adam.
    The two routes' gradients differ in the last bits, and Adam's first steps take g / |g|, which
    turns that into whole-step differences on near-zero components, so only the epoch losses are
    compared, at 1e-3 (one step moves a parameter by 1e-2 at most)."""
    from spotlight_b200 import optim
    I, D = 600, 16
    inter = _seqs(I)
    fused, init, lf = _fit(_bloom(net, I, D), optim.fused_adam(lr=1e-2), inter, D, capsys=capsys)
    assert fused._route() == 'fused_hashed'
    assert fused._net.item_embeddings.embeddings.weight.grad is None and fused._net.item_biases.weight.grad is None
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
            plain, _, lp = _fit(_bloom(net, I, D), lambda p: torch.optim.Adam(p, lr=1e-2), inter, D, state=init,
                                capsys=capsys)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    assert plain._route() == 'generic'
    assert_close(lf, lp, 1e-3, what='epoch losses')
    st = fused._optimizer.state[fused._net.item_embeddings.embeddings.weight]
    assert int(st['last'].min()) == fused._optimizer.steps_taken


def test_generic_route_fused_adam_equals_torch_adam():
    """LSTMNet at D = 260 (beyond the fused LSTM) takes the generic route; FusedAdam there is the
    dense fallback and follows torch.optim.Adam, in fp32 (no TF32).  Dense tables: with sparse=True
    torch.optim.Adam rejects the sparse gradients, and so does FusedAdam (tests/test_seq_adam_oracle_cpu.py).  Checked at 5 % of one Adam step
    (lr = 1e-2): the two optimizers evaluate the same formulas in different fp32 orders, and Adam's
    m / sqrt(v) turns last-bit differences on near-zero gradient components into fractions of a step."""
    from spotlight_b200 import optim
    from spotlight_b200.sequence.representations import LSTMNet
    I, D = 300, 260
    inter = _seqs(I, n=64)
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
            a, init, _ = _fit(LSTMNet(I, D), optim.fused_adam(lr=1e-2), inter, D, n_iter=1)
            b, _, _ = _fit(LSTMNet(I, D), lambda p: torch.optim.Adam(p, lr=1e-2), inter, D, state=init, n_iter=1)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    assert a._route() == 'generic'
    for (k, x), (_, y) in zip(a._net.state_dict().items(), b._net.state_dict().items()):
        assert_close(x.cpu().numpy(), y.cpu().numpy(), 0.0, atol=5e-4, what=k)


def test_mrr_resume_and_pickle(tmp_path):
    """sequence_mrr_score after a fused_adam fit (it flushes), a second fit() that resumes the step
    count, and a torch.save / torch.load round trip that resumes it too."""
    from spotlight_b200 import optim
    from spotlight_b200.evaluation import sequence_mrr_score
    I, D = 5000, 16
    inter = _seqs(I, hi=1000)
    model, _, _ = _fit('lstm', optim.fused_adam(lr=1e-2, weight_decay=1e-4), inter, D, n_iter=1)
    mrr = sequence_mrr_score(model, inter)
    assert mrr.shape == (len(inter.sequences),) and np.isfinite(mrr).all()
    opt = model._optimizer
    assert opt.steps_taken == 8
    path = str(tmp_path / 'model.pt')
    torch.save(model, path)
    loaded = torch.load(path, weights_only=False)
    for m in (model, loaded):
        m.fit(inter)
        assert m._optimizer.steps_taken == 16
        W = m._net.item_embeddings.weight
        assert int(m._optimizer.state[W]['last'].min()) == 16
    for (k, x), (_, y) in zip(model._net.state_dict().items(), loaded._net.state_dict().items()):
        assert_close(x.cpu().numpy(), y.cpu().numpy(), 1e-6, atol=1e-9, what=k)


GOLDEN_FITS = [('fit_pool_adam', 'pooling'), ('fit_cnn_adam', 'cnn'), ('fit_lstm_adam', 'lstm')]


@pytest.mark.parametrize('name,rep', GOLDEN_FITS, ids=[g[0] for g in GOLDEN_FITS])
def test_fit_golden(name, rep, capsys):
    """fit() with optim.fused_adam(lr, weight_decay=l2) on the fused route against the live
    reference's fit() with its default Adam (tests/golden/make_golden_seq_adam.py): epoch losses at
    1e-5, final state_dict and predict at 2e-3 of their scale (Adam: see the module docstring), the
    RandomState position exact; every row current after fit().  The item biases at 5e-3: under bpr
    a bias's target and negative terms nearly cancel, and Adam's m / sqrt(v) magnifies the fp32
    rounding of such sums.  The float64 lazy scheme of tests/test_seq_adam_oracle_cpu.py lands 1.0e-3
    from fit_pool_adam's biases with float64 gradients and 2.3e-3 with float32 ones, no kernel
    involved."""
    from conftest import load_golden
    from spotlight_b200 import optim
    from spotlight_b200.interactions import SequenceInteractions
    from spotlight_b200.sequence.implicit import ImplicitSequenceModel
    g = load_golden(name)
    inter = SequenceInteractions(g['seqs'], num_items=int(g['num_items']))
    model = ImplicitSequenceModel(loss=str(g['loss']), representation=rep, embedding_dim=int(g['dim']),
                                  batch_size=int(g['batch']), n_iter=int(g['n_iter']),
                                  optimizer_func=optim.fused_adam(lr=float(g['lr']), weight_decay=float(g['l2'])),
                                  use_cuda=True, random_state=np.random.RandomState(int(g['seed'])))
    model._initialize(inter)
    model._net.load_state_dict({k[5:]: torch.from_numpy(v) for k, v in g.items() if k.startswith('init.')})
    assert model._route() == 'fused'
    capsys.readouterr()
    model.fit(inter, verbose=True)
    lines = [l for l in capsys.readouterr().out.strip().split('\n') if l.startswith('Epoch')]
    assert_close(np.array([float(l.split('loss')[1]) for l in lines]), g['epoch_losses'], 1e-5, what='epoch losses')
    for k, v in model._net.state_dict().items():
        assert_close(v.cpu().numpy(), g['final.' + k], 5e-3 if k == 'item_biases.weight' else 2e-3, atol=1e-7, what=k)
    st = model._random_state.get_state()
    assert (st[1] == g['rs_key']).all() and st[2] == int(g['rs_pos'])
    opt = model._optimizer
    assert int(opt.state[model._net.item_embeddings.weight]['last'].min()) == opt.steps_taken
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):     # predict runs nn.LSTM
        assert_close(model.predict(g['seqs'][1]), g['predict'], 2e-3, what='predict')
