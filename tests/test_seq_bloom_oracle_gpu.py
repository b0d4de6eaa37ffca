"""The sequence training step on a hashed (Bloom) item table -- csrc/seq.cu with item_hashes > 0:
seq_gather_hashed_kernel, the position-indexed pool kernels, seq_score_kernel / mix_score_kernel
with hashed negatives, the two-key-space segment index and seq_reduce_kernel -- against the float64
oracle (oracle/seq_bloom.py), and ImplicitSequenceModel's fused_hashed route.

Tolerances are those of tests/test_seq_oracle_gpu.py: loss and scores 1e-5, gradients 2e-5, each
relative to the tensor's maximum magnitude.  tests/test_seq_bloom_oracle_cpu.py shows that these
tolerances catch plausible kernel mistakes on the cases of oracle.seq_bloom.CASES."""

import numpy as np
import pytest
import torch

from conftest import assert_close
from oracle import seq_bloom as sb

pytestmark = pytest.mark.gpu


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to('cuda:0')


def step_kwargs(case):
    kw = dict(item_hash=dict(seeds=case['seeds'], padding_idx=0))
    if case['cnn'] is not None:
        kw['cnn'] = dict(case['cnn'], weights=[t(w) for w, _ in case['convs']], biases=[t(b) for _, b in case['convs']])
    if case['net'] in ('lstm', 'mixture'):
        kw['lstm'] = {k: t(v) for k, v in case['lstm'].items()}
    if case['net'] == 'mixture':
        kw['mixture'] = dict(num_mixtures=case['M'], w=t(case['proj']['w']), b=t(case['proj']['b']))
    return kw


def run_step(case, W=None, bias=None, **kw):
    from spotlight_b200 import ops
    W = t(case['W']) if W is None else W
    bias = t(case['bias']) if bias is None else bias
    return ops.seq_train_step(W, bias, t(case['seqs']), t(case['negs']), case['loss'], case['n_neg'],
                              want_scores=True, **step_kwargs(case), **kw)


def check_net_grads(out, ref):
    for i, (dW, db) in enumerate(ref.get('dconvs', [])):
        assert_close(out['dconv_w'][i].cpu().numpy(), dW, 2e-5, what='dconv_w%d' % i)
        assert_close(out['dconv_b'][i].cpu().numpy(), db, 2e-5, what='dconv_b%d' % i)
    for k, v in (ref.get('dlstm') or {}).items():
        assert_close(out['dlstm'][k].cpu().numpy(), v, 2e-5, what='dlstm ' + k)
    for k, v in (ref.get('dmix') or {}).items():
        assert_close(out['dmix'][k].cpu().numpy(), v, 2e-5, what='dmix ' + k)


def check_step(out, ref):
    assert_close(out['pos'].cpu().numpy(), ref['pos'], 1e-5, what='pos')
    assert_close(out['neg'].cpu().numpy().reshape(ref['neg'].shape), ref['neg'], 1e-5, what='neg')
    assert_close(out['loss'].item(), ref['loss'], 1e-5, what='loss')
    assert_close(out['dE'].cpu().numpy(), ref['dW'], 2e-5, what='dW')
    assert_close(out['dbias'].cpu().numpy(), ref['dbias'], 2e-5, what='dbias')
    assert float(out['dE'][0].abs().sum()) == 0.0 and float(out['dbias'][0].abs().sum()) == 0.0, \
        'the frozen row or the padding bias received a gradient'
    check_net_grads(out, ref)


def run_case(case):
    ref = sb.step(case)
    assert sb.check_properties(case, ref) == []
    check_step(run_step(case), ref)
    return ref


# ------------------------------------------------------------------ the shared cases
@pytest.mark.parametrize('kw', sb.CASES, ids=[sb.case_id(k) for k in sb.CASES])
def test_cases(kw):
    run_case(sb.make_case(**kw))


# ------------------------------------------------------------------ live-reference fixtures
@pytest.mark.parametrize('name', sb.GOLDEN)
def test_step_golden(name):
    """The reference's Bloom CNNNet / LSTMNet / MixtureLSTMNet steps (tests/golden/make_golden_seq_bloom.py)."""
    from conftest import load_golden
    g = load_golden(name)
    case = sb.golden_case(g)
    out = run_step(case)
    want = sb.golden_grads(g)
    assert_close(out['pos'].cpu().numpy(), g['pos'], 1e-5, what='pos')
    assert_close(out['neg'].cpu().numpy().reshape(g['neg'].shape), g['neg'], 1e-5, what='neg')
    assert_close(out['loss'].item(), g['loss'], 1e-5, what='loss')
    assert_close(out['dE'].cpu().numpy(), want['dW'], 2e-5, what='dW')
    assert_close(out['dbias'].cpu().numpy(), want['dbias'], 2e-5, what='dbias')
    check_net_grads(out, want)


def test_fit_golden(capsys):
    """fit_bloom_lstm_adagrad.npz: two epochs of the reference's fit() with a Bloom LSTMNet and
    torch.optim.Adagrad; here on the fused_hashed route with optim.fused_adagrad (row-wise Adagrad
    without weight decay follows the same trajectory).  Epoch losses, final parameters, the
    RandomState afterwards and predict."""
    from conftest import load_golden
    from spotlight_b200 import optim
    from spotlight_b200.interactions import SequenceInteractions
    from spotlight_b200.layers import BloomEmbedding
    from spotlight_b200.sequence.implicit import ImplicitSequenceModel
    from spotlight_b200.sequence.representations import LSTMNet
    g = load_golden('fit_bloom_lstm_adagrad')
    I, D, H = int(g['num_items']), int(g['dim']), int(g['bloom_H'])
    net = LSTMNet(I, D, item_embedding_layer=BloomEmbedding(I, D, compression_ratio=float(g['bloom_ratio']),
                                                            num_hash_functions=H, padding_idx=0))
    net.load_state_dict({k[5:]: torch.from_numpy(v) for k, v in g.items() if k.startswith('init.')})
    model = ImplicitSequenceModel(loss='bpr', representation=net, embedding_dim=D, batch_size=int(g['batch']),
                                  n_iter=int(g['n_iter']), optimizer_func=optim.fused_adagrad(lr=float(g['lr'])),
                                  use_cuda=True, random_state=np.random.RandomState(int(g['seed'])))
    inter = SequenceInteractions(g['seqs'], num_items=I)
    model._initialize(inter)
    st = model._random_state.get_state()
    assert (st[1] == g['rs0_key']).all() and st[2] == int(g['rs0_pos'])
    assert model._route() == 'fused_hashed'
    capsys.readouterr()
    model.fit(inter, verbose=True)
    lines = [l for l in capsys.readouterr().out.strip().split('\n') if l.startswith('Epoch')]
    assert_close(np.array([float(l.split('loss')[1]) for l in lines]), g['epoch_losses'], 1e-5, what='epoch losses')
    for k, v in model._net.state_dict().items():
        assert_close(v.cpu().numpy(), g['final.' + k], 1e-4, atol=1e-7, what=k)
    st = model._random_state.get_state()
    assert (st[1] == g['rs_key']).all() and st[2] == int(g['rs_pos'])
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):     # predict runs nn.LSTM
        assert_close(model.predict(g['seqs'][1]), g['predict'], 1e-4, what='predict')


# ------------------------------------------------------------------ dimensions x hash counts
# Pool / CNN: every pool chunk count and lane-group width, the wgmma conv at D = 128; LSTM /
# mixture: all three cluster sizes (D <= 64, <= 128, <= 256).  Hash counts and losses cycle.
HS = (1, 2, 4, 24)
LOSSES = (('pointwise', 1), ('bpr', 1), ('hinge', 1), ('adaptive_hinge', 5))
DIMS = [('pool', D) for D in (4, 12, 36, 128, 512)] + [('cnn', D) for D in (4, 12, 36, 128, 512)] + \
       [('lstm', D) for D in (16, 128, 256)] + [('mixture', D) for D in (16, 128, 256)]


@pytest.mark.parametrize('net,D', DIMS, ids=['%s-%d' % d for d in DIMS])
def test_dims(net, D):
    i = DIMS.index((net, D))
    loss, n_neg = LOSSES[i % 4]
    H = HS[i % 4]
    kw = dict(kernel_width=(3, 2), dilation=(1, 2)) if net == 'cnn' else {}
    if net == 'mixture':
        kw['M'] = 4
    S, B = (12, 6) if D >= 256 else (20, 10)
    case = sb.make_case(net, D=D, S=S, B=B, I=400, rows=30 * H, H=H, loss=loss, n_neg=n_neg, seed=100 + i, **kw)
    run_case(case)


@pytest.mark.parametrize('H', HS)
@pytest.mark.parametrize('loss,n_neg', LOSSES, ids=[l for l, _ in LOSSES])
def test_losses_and_hashes(loss, n_neg, H):
    net = ('pool', 'cnn', 'lstm', 'mixture')[(HS.index(H) + [l for l, _ in LOSSES].index(loss)) % 4]
    kw = dict(M=4) if net == 'mixture' else {}
    case = sb.make_case(net, D=32, S=20, B=12, I=400, rows=20 * H, H=H, loss=loss, n_neg=n_neg,
                        seed=7 * H + n_neg, **kw)
    run_case(case)


# ------------------------------------------------------------------ hot hashed rows
@pytest.mark.parametrize('net,D,rows', [('pool', 32, 40), ('lstm', 16, 4), ('cnn', 128, 5)])
def test_hot_rows(net, D, rows):
    """Tiny tables: rows with more terms than the reduce sorts in shared memory, and (rows = 4 / 5)
    rows with >= 10^4 terms, all through seg_sort_long_kernel; two runs bit-identical."""
    kw = dict(kernel_width=(3,), dilation=(1,)) if net == 'cnn' else {}
    S, B = (200, 128) if rows <= 5 else (100, 64)
    case = sb.make_case(net, D=D, S=S, B=B, I=400, rows=rows, H=4, loss='pointwise', seed=rows, **kw)
    ref = sb.step(case)
    seqs = case['seqs']
    from oracle.murmur import bloom_rows
    terms = np.bincount(bloom_rows(seqs[seqs != 0], 4, rows).ravel(), minlength=rows)[1:]
    assert terms.max() > 128
    if rows <= 5:
        assert terms.max() >= 10 ** 4
    a, b = run_step(case), run_step(case)
    check_step(a, ref)
    for k in ('dE', 'dbias', 'loss'):
        assert torch.equal(a[k], b[k]), '%s is not bit-reproducible' % k


# ------------------------------------------------------------------ fused optimizers
FUSED = [
    dict(net='pool', D=32, loss='bpr', opt='sgd', wd=0.0, H=4),
    dict(net='pool', D=16, loss='hinge', opt='adagrad', wd=0.1, H=2),
    dict(net='cnn', D=32, loss='hinge', opt='sgd', wd=0.1, H=4),
    dict(net='cnn', D=128, loss='adaptive_hinge', n_neg=5, opt='adagrad', wd=0.05, H=3),
    dict(net='lstm', D=32, loss='pointwise', opt='adagrad', wd=0.1, H=4),
    dict(net='mixture', D=16, loss='hinge', opt='sgd', wd=0.05, H=2, M=3),
]


@pytest.mark.parametrize('f', FUSED, ids=['%s-%s-%s' % (f['net'], f['opt'], f['loss']) for f in FUSED])
def test_fused_optimizer(f):
    """SGD / Adagrad with weight decay fused into the reduction, against torch's update rules
    restated on the oracle gradients for the rows and biases oracle.seq_bloom.updated names; every
    other row (row 0 included) and bias stays bit-identical."""
    from oracle import seq_cases as sc
    from spotlight_b200 import _lib
    f = dict(f)
    kw = {k: f[k] for k in ('n_neg', 'M') if k in f}
    if f['net'] == 'cnn':
        kw.update(kernel_width=(3,), dilation=(1,))
    # a table large enough to leave rows untouched
    case = sb.make_case(f['net'], D=f['D'], S=20, B=12, I=400, rows=500, H=f['H'], loss=f['loss'], seed=3, **kw)
    ref = sb.step(case)
    rows, ids = sb.updated(case, ref)
    assert rows.sum() > 0 and (~rows[1:]).sum() > 0 and ids.sum() > 0
    W, b = t(case['W']), t(case['bias'])
    wd = f['wd']
    if f['opt'] == 'sgd':
        lr = 0.3 / max(np.abs(ref['dW']).max(), np.abs(ref['dbias']).max())
        fused = dict(kind=_lib.OPT_SGD, lr=lr, weight_decay=wd, eps=0.0)
        W_exp = sc.sgd(case['W'], ref['dW'], rows[:, None], lr, wd)
        b_exp = sc.sgd(case['bias'], ref['dbias'], ids[:, None], lr, wd)
    else:
        rs = np.random.RandomState(1)
        lr, eps = 0.05, 1e-10
        sW0 = (rs.rand(*case['W'].shape) * 0.02 + 1e-4).astype(np.float32)
        sb0 = (rs.rand(*case['bias'].shape) * 0.02 + 1e-4).astype(np.float32)
        sW, sbias = t(sW0), t(sb0)
        fused = dict(kind=_lib.OPT_ADAGRAD, lr=lr, weight_decay=wd, eps=eps, state_E=sW, state_bias=sbias)
        W_exp, sW_exp = sc.adagrad(case['W'], sW0, ref['dW'], rows[:, None], lr, wd, eps)
        b_exp, sb_exp = sc.adagrad(case['bias'], sb0, ref['dbias'], ids[:, None], lr, wd, eps)
    out = run_step(case, W, b, fused=fused)
    assert out['dE'] is None and out['dbias'] is None
    assert_close(out['loss'].item(), ref['loss'], 1e-5, what='loss')
    Wn, bn = W.cpu().numpy(), b.cpu().numpy()
    assert_close(Wn, W_exp, 5e-6, what='W')
    assert_close(bn, b_exp, 5e-6, what='bias')
    assert (Wn[~rows] == case['W'][~rows]).all(), 'a row without terms (or row 0) changed'
    assert (bn[~ids] == case['bias'][~ids]).all(), 'a bias without a non-zero score gradient changed'
    if f['opt'] == 'adagrad':
        assert_close(sW.cpu().numpy(), sW_exp, 1e-5, what='Adagrad sum (W)')
        assert_close(sbias.cpu().numpy(), sb_exp, 1e-5, what='Adagrad sum (bias)')
        assert (sW.cpu().numpy()[~rows] == sW0[~rows]).all() and (sbias.cpu().numpy()[~ids] == sb0[~ids]).all()
    check_net_grads(out, ref)


# ------------------------------------------------------------------ workspace, determinism, limits
def test_workspace_reuse_and_plain_calls_in_between():
    """One (num_items, rows) pair, so one cached hashed workspace, through calls that change the net,
    B, S, D and H; plain-table calls on the same num_items run in between on their own workspace."""
    from oracle import seq_cases as sc
    calls = [
        dict(net='cnn', D=128, S=60, B=16, H=4, loss='bpr', kernel_width=(2, 5), dilation=(1, 2)),
        dict(net='pool', D=16, S=40, B=30, H=24, loss='hinge'),
        dict(net='lstm', D=64, S=9, B=7, H=1, loss='adaptive_hinge', n_neg=3),
        dict(net='mixture', D=32, S=30, B=5, H=2, loss='pointwise', M=2),
        dict(net='pool', D=512, S=9, B=4, H=4, loss='bpr'),
    ]
    for n, kw in enumerate(calls):
        case = sb.make_case(I=997, rows=150, seed=40 + n, **kw)
        check_step(run_step(case), sb.step(case))
        plain = sc.make_case('pool', D=32, S=11, B=6, I=997, loss='bpr', seed=n)
        from spotlight_b200 import ops
        out = ops.seq_train_step(t(plain['E']), t(plain['bias']), t(plain['seqs']), t(plain['negs']), 'bpr', 1)
        pref = sc.oracle_step(plain)
        assert_close(out['dE'].cpu().numpy(), pref['dE'], 2e-5, what='plain dE')


def test_bit_reproducible():
    case = sb.make_case(**sb.CASES[4])
    a, b = run_step(case), run_step(case)
    for k in ('pos', 'neg', 'loss', 'dE', 'dbias'):
        assert torch.equal(a[k], b[k]), k
    for k in a['dlstm']:
        assert torch.equal(a['dlstm'][k], b['dlstm'][k]), k


def test_term_count_guard():
    """2 * B * S * (H + 1) >= 2^31 gradient terms is rejected before any launch."""
    from spotlight_b200 import ops
    from oracle.murmur import SEEDS
    B, S = 1024, 42000                           # 2 * B * S * 25 = 2.15e9
    seqs = torch.ones((B, S), dtype=torch.int64, device='cuda:0')
    W = torch.zeros((8, 4), dtype=torch.float32, device='cuda:0')
    bias = torch.zeros((10, 1), dtype=torch.float32, device='cuda:0')
    with pytest.raises(ValueError, match='2\\^31'):
        ops.seq_train_step(W, bias, seqs, seqs, 'bpr', 1, item_hash=dict(seeds=SEEDS[:24], padding_idx=0))
    del seqs
    torch.cuda.empty_cache()


# ------------------------------------------------------------------ model level
def _bloom_net(net, I, D, H=2, ratio=0.5, padding_idx=0, M=2):
    from spotlight_b200.layers import BloomEmbedding
    from spotlight_b200.sequence.representations import CNNNet, LSTMNet, MixtureLSTMNet, PoolNet
    emb = BloomEmbedding(I, D, compression_ratio=ratio, num_hash_functions=H, padding_idx=padding_idx)
    if net == 'mixture':
        return MixtureLSTMNet(I, D, num_mixtures=M, item_embedding_layer=emb)
    return {'pool': PoolNet, 'cnn': CNNNet, 'lstm': LSTMNet}[net](I, D, item_embedding_layer=emb)


def _seqs(I, n=300, S=12, seed=17):
    from spotlight_b200.interactions import SequenceInteractions
    rs = np.random.RandomState(seed)
    seqs = rs.randint(1, I, (n, S)).astype(np.int32)
    for b in range(0, n, 3):
        seqs[b, :rs.randint(0, S)] = 0
    return SequenceInteractions(seqs, num_items=I)


@pytest.mark.parametrize('net', ['pool', 'cnn', 'lstm', 'mixture'])
def test_fit_fused_sgd_matches_generic_route(net, capsys):
    """fit() on the fused_hashed route with optim.fused_sgd (no weight decay) against a copy on the
    generic route (nn.LSTM / nn.Conv / autograd through the Bloom gather) with torch.optim.SGD:
    row-wise SGD without decay leaves a row whose gradient is zero unchanged, so both follow one
    trajectory.  (SGD rather than Adagrad: the two routes' gradients differ in the last bits, and
    Adagrad's first steps, g / |g|, amplify that on near-zero entries; the Adagrad trajectory is
    checked against the reference in test_fit_golden.)  Then predict and sequence_mrr_score run on
    the trained model."""
    from spotlight_b200 import optim
    from spotlight_b200.evaluation import sequence_mrr_score
    from spotlight_b200.sequence.implicit import ImplicitSequenceModel
    I, D = 300, 16
    inter = _seqs(I)

    def fit(opt_func, state=None):
        torch.manual_seed(0)
        model = ImplicitSequenceModel(loss='bpr', representation=_bloom_net(net, I, D), embedding_dim=D,
                                      batch_size=64, n_iter=2, optimizer_func=opt_func, use_cuda=True,
                                      random_state=np.random.RandomState(5))
        model._initialize(inter)
        if state is not None:
            model._net.load_state_dict(state)
        init = {k: v.clone() for k, v in model._net.state_dict().items()}
        capsys.readouterr()
        model.fit(inter, verbose=True)
        lines = [l for l in capsys.readouterr().out.strip().split('\n') if l.startswith('Epoch')]
        return model, init, np.array([float(l.split('loss')[1]) for l in lines])

    fused, init, lf = fit(optim.fused_sgd(lr=0.5))
    assert fused._route() == 'fused_hashed'
    assert fused._net.item_embeddings.embeddings.weight.grad is None and fused._net.item_biases.weight.grad is None
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False          # the generic route's convs / LSTM in fp32
    try:
        with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
            plain, _, lp = fit(lambda p: torch.optim.SGD(p, lr=0.5), init)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    assert plain._route() == 'generic'
    assert len(lf) == 2
    assert_close(lf, lp, 1e-5, what='epoch losses')
    for k, v in plain._net.state_dict().items():
        assert_close(fused._net.state_dict()[k].cpu().numpy(), v.cpu().numpy(), 1e-4, atol=1e-7, what=k)
    scores = fused.predict(inter.sequences[1])
    assert scores.shape == (I,) and np.isfinite(scores).all()
    mrr = sequence_mrr_score(fused, inter)
    assert mrr.shape == (len(inter.sequences),) and np.isfinite(mrr).all()


def test_fit_fused_sgd_with_decay_runs():
    from spotlight_b200 import optim
    from spotlight_b200.sequence.implicit import ImplicitSequenceModel
    inter = _seqs(300)
    model = ImplicitSequenceModel(loss='adaptive_hinge', representation=_bloom_net('lstm', 300, 16, H=4),
                                  embedding_dim=16, batch_size=64, n_iter=2,
                                  optimizer_func=optim.fused_sgd(lr=0.1, weight_decay=1e-3), use_cuda=True,
                                  random_state=np.random.RandomState(2))
    model._initialize(inter)
    W0 = model._net.item_embeddings.embeddings.weight.detach().clone()
    model.fit(inter)
    assert model._route() == 'fused_hashed'
    W = model._net.item_embeddings.embeddings.weight.detach()
    assert torch.equal(W[0], W0[0]), 'row 0 of the hashed table changed'
    assert not torch.equal(W, W0)


@pytest.mark.parametrize('kind', ['padding_none', 'sparse', 'lstm_d260', 'mixture_m9', 'torch_adagrad'])
def test_other_bloom_nets_stay_generic(kind):
    from spotlight_b200 import optim
    from spotlight_b200.sequence.implicit import ImplicitSequenceModel
    I, D, sparse, opt = 300, 16, False, optim.fused_adagrad(lr=0.05)
    if kind == 'padding_none':
        net = _bloom_net('pool', I, D, padding_idx=None)
    elif kind == 'sparse':
        net, sparse = _bloom_net('pool', I, D), True
    elif kind == 'lstm_d260':
        D = 260
        net = _bloom_net('lstm', I, D)
    elif kind == 'mixture_m9':
        net = _bloom_net('mixture', I, D, M=9)
    else:
        net, opt = _bloom_net('cnn', I, D), (lambda p: torch.optim.Adagrad(p, lr=0.05))
    assert not net.fusable()
    model = ImplicitSequenceModel(loss='bpr', representation=net, embedding_dim=D, batch_size=64, n_iter=1,
                                  optimizer_func=opt, use_cuda=True, sparse=sparse,
                                  random_state=np.random.RandomState(1))
    model._initialize(_seqs(I, n=64))
    assert model._route() == 'generic'
    if kind in ('padding_none', 'lstm_d260', 'mixture_m9'):
        assert net.hashed_spec() is None
