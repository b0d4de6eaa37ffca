"""The sequence training step (PoolNet, CNNNet) and its representation against the float64
oracle, across the kernel variants: lane-group widths, wide pool rows, partial conv tiles on
both conv paths (mma.sync, and wgmma at D = 128), conv geometry, all four losses, padding,
long gradient segments, the fused optimizers, workspace reuse and the configs[4] size.

Tolerances are those of tests/test_seq_gpu.py: loss and scores 1e-5, gradients 2e-5, each
relative to the tensor's maximum magnitude.  tests/test_seq_oracle_cpu.py shows that these
tolerances catch plausible kernel mistakes on the same cases."""

import numpy as np
import pytest
import torch

from conftest import assert_close
from oracle import seq_cases as sc

pytestmark = pytest.mark.gpu


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to('cuda:0')


def gpu_spec(case):
    if case['cnn'] is None:
        return None
    return dict(case['cnn'], weights=[t(w) for w, _ in case['convs']], biases=[t(b) for _, b in case['convs']])


def run_step(case, E=None, bias=None, **kw):
    from spotlight_b200 import ops
    E = t(case['E']) if E is None else E
    bias = t(case['bias']) if bias is None else bias
    return ops.seq_train_step(E, bias, t(case['seqs']), t(case['negs']), case['loss'], case['n_neg'],
                              gpu_spec(case), want_scores=True, **kw)


def check_step(case, out, ref, rows=None):
    """Scores, loss, every gradient; ``rows``: compare dE on these rows only."""
    assert_close(out['pos'].cpu().numpy(), ref['pos'], 1e-5, what='pos')
    assert_close(out['neg'].cpu().numpy().reshape(ref['neg'].shape), ref['neg'], 1e-5, what='neg')
    assert_close(out['loss'].item(), ref['loss'], 1e-5, what='loss')
    dE = out['dE'].cpu().numpy()
    if rows is None:
        assert_close(dE, ref['dE'], 2e-5, what='dE')
    else:
        assert_close(dE[rows], ref['dE'][rows], 2e-5, what='dE (touched rows)')
    assert_close(out['dbias'].cpu().numpy(), ref['dbias'], 2e-5, what='dbias')
    assert float(out['dE'][0].abs().sum()) == 0.0 and float(out['dbias'][0].abs().sum()) == 0.0, \
        'the padding row received a gradient'
    for i, (dW, db) in enumerate(ref.get('dconvs', [])):
        assert_close(out['dconv_w'][i].cpu().numpy(), dW, 2e-5, what='dW%d' % i)
        assert_close(out['dconv_b'][i].cpu().numpy(), db, 2e-5, what='db%d' % i)


def check_representation(case):
    from spotlight_b200 import ops
    rep = ops.seq_representation(t(case['E']), t(case['seqs']), gpu_spec(case))
    # Above D = 256 a conv output sums k * D >= 1152 products on the tensor cores (3xTF32 with
    # fp32 accumulation); the measured error there is 1.3e-5 / 1.5e-5 of the largest entry at
    # D = 384 / 512 with two layers (k = 3, 2), so those representations are held to 2e-5.
    # Every score, loss and gradient of the same cases meets the 1e-5 / 2e-5 tolerances.
    rtol = 2e-5 if case['cnn'] is not None and case['E'].shape[1] > 256 else 1e-5
    assert_close(rep.cpu().numpy(), sc.oracle_representation(case), rtol, what='representation')


def run_case(case):
    ref = sc.oracle_step(case)
    assert sc.check_properties(case, ref) == []
    check_step(case, run_step(case), ref)
    check_representation(case)
    return ref


# ------------------------------------------------------------------ dimensions
# D = 4 runs one lane per row; 12, 20, 36, 100 leave lanes of each group idle (D / 4 is not a
# power of two) and tiles of the mma.sync conv partial (D % 16, D % 64); 384 and 512 run the
# 4-chunk pool kernels; 128 is the wgmma conv.
DIMS = [4, 12, 20, 36, 100, 128, 384, 512]


@pytest.mark.parametrize('D', DIMS)
@pytest.mark.parametrize('net', ['pool', 'cnn'])
def test_dims(net, D):
    i = DIMS.index(D) + (net == 'cnn')
    loss = sc.LOSS_CYCLE[i % 4]
    case = sc.make_case(net, D=D, S=23, B=11, loss=loss, n_neg=2, kernel_width=(3, 2), dilation=(1, 2),
                        nonlinearity='relu' if i % 3 == 0 else 'tanh', seed=D)
    run_case(case)


# ------------------------------------------------------------------ conv geometry
@pytest.mark.parametrize('g', range(len(sc.GEOMETRIES)))
@pytest.mark.parametrize('D', [32, 128], ids=['mma', 'wgmma'])
def test_conv_geometry(D, g):
    geo = dict(sc.GEOMETRIES[g])
    S, B = geo.pop('S'), geo.pop('B')
    loss = sc.LOSS_CYCLE[(g + (D == 128)) % 4]
    case = sc.make_case('cnn', D=D, S=S, B=B, loss=loss, n_neg=3, seed=100 + g, **geo)
    run_case(case)


# ------------------------------------------------------------------ losses
PATHS = {'pool': dict(net='pool', D=32), 'mma': dict(net='cnn', D=32), 'wgmma': dict(net='cnn', D=128)}
LOSSES = [('pointwise', 1), ('bpr', 1), ('hinge', 1), ('adaptive_hinge', 2), ('adaptive_hinge', 5)]


@pytest.mark.parametrize('loss,n_neg', LOSSES, ids=['pointwise', 'bpr', 'hinge', 'adaptive2', 'adaptive5'])
@pytest.mark.parametrize('path', sorted(PATHS))
def test_losses(path, loss, n_neg):
    case = sc.make_case(S=20, B=16, loss=loss, n_neg=n_neg, kernel_width=(3, 2), dilation=(1, 2),
                        seed=7 + n_neg, **PATHS[path])
    run_case(case)


@pytest.mark.parametrize('path', sorted(PATHS))
def test_adaptive_hinge_tied_negatives(path):
    """Two negative ids with bit-identical rows score the same; the gradient goes to the one
    drawn first (torch.max over dim 0 credits the first maximal index)."""
    case = sc.make_case(S=20, B=16, loss='adaptive_hinge', n_neg=2, neg_tie=True, seed=11, **PATHS[path])
    ref = run_case(case)
    half = case['E'].shape[0] // 2
    j1, j2 = half + 1, half + 2
    # both tied rows are credited somewhere, so swapping the tie-break would move their gradients
    assert (ref['dE'][j1] != 0).any() and (ref['dE'][j2] != 0).any()


@pytest.mark.parametrize('path', sorted(PATHS))
def test_padding_and_zeros(path):
    """A fully padded sequence, padding mid-sequence, padding negatives, a non-zero E[0] (read
    by the forward; dE[0] / dbias[0] stay 0) and exact zeros inside rows (PoolNet's count)."""
    case = sc.make_case(S=30, B=9, loss='bpr', e0_nonzero=True, zero_frac=0.3, seed=5, **PATHS[path])
    assert (case['seqs'][0] == 0).all() and (case['negs'] == 0).any() and (case['E'][0] != 0).all()
    run_case(case)


# ------------------------------------------------------------------ long segments
@pytest.mark.parametrize('D', [4, 8, 16, 64, 256])
def test_long_segments(D):
    """Zipf-drawn targets: several rows have more terms than the reduce sorts in shared memory
    (the min-selection walk of seg_visit_sorted), one item holds over half of the targets."""
    net = 'cnn' if D in (8, 64) else 'pool'
    case = sc.make_case(net, D=D, S=100, B=40, loss=sc.LOSS_CYCLE[D % 3], zipf=2.0, seed=D)
    ref = sc.oracle_step(case)
    lens = sc.segment_lengths(case, ref)
    assert (lens > sc.seg_sort_cap(D)).sum() >= 3
    targets = case['seqs'][case['seqs'] != 0]
    assert np.bincount(targets).max() > targets.size / 2
    assert sc.check_properties(case, ref) == []
    out = run_step(case)
    check_step(case, out, ref)
    out2 = run_step(case)
    assert torch.equal(out['dE'], out2['dE']) and torch.equal(out['dbias'], out2['dbias']), \
        'sequence step is not bit-reproducible'


# ------------------------------------------------------------------ fused optimizers
FUSED = [
    dict(id='pool-sgd', net='pool', D=32, S=20, B=16, loss='bpr', opt='sgd', wd=0.0),
    dict(id='pool-adagrad-wd', net='pool', D=32, S=20, B=16, loss='hinge', opt='adagrad', wd=0.1),
    # S = 1: every item is a target at t = 0 only, where r_0 = 0: the embedding gradient is
    # exactly zero while the bias gradient is not -- the row is still decayed as a whole
    dict(id='pool-t0-sgd-wd', net='pool', D=16, S=1, B=64, loss='pointwise', opt='sgd', wd=0.1),
    dict(id='pool-t0-adagrad-wd', net='pool', D=16, S=1, B=64, loss='bpr', opt='adagrad', wd=0.1),
    # relu without residual at S = 1: r_0 = relu(conv bias), whose first 4-chunk is forced to 0
    dict(id='cnn-relu-zero-chunk-adagrad-wd', net='cnn', D=32, S=1, B=64, loss='pointwise', opt='adagrad',
         wd=0.1, nonlinearity='relu', residual=False, kernel_width=(3,), dilation=(1,)),
    dict(id='wgmma-adagrad-wd', net='cnn', D=128, S=30, B=8, loss='adaptive_hinge', n_neg=2, opt='adagrad',
         wd=0.05),
    dict(id='mma-sgd', net='cnn', D=32, S=30, B=8, loss='hinge', opt='sgd', wd=0.0, nonlinearity='relu'),
]


@pytest.mark.parametrize('f', FUSED, ids=[f['id'] for f in FUSED])
def test_fused_optimizer(f):
    """SGD / Adagrad fused into the reduction against torch's update rules restated in NumPy on
    the oracle gradients, applied to the rows the step updates (sc.updated_rows); every other
    row, the padding row included, stays bit-identical."""
    from spotlight_b200 import _lib
    f = dict(f)
    kw = {k: f.pop(k) for k in ('nonlinearity', 'residual', 'kernel_width', 'dilation', 'n_neg') if k in f}
    case = sc.make_case(f['net'], D=f['D'], S=f['S'], B=f['B'], loss=f['loss'], seed=3, **kw)
    if f['id'].startswith('cnn-relu-zero-chunk'):
        case['convs'][0][1][:4] = -np.abs(case['convs'][0][1][:4]) - 0.05
    ref = sc.oracle_step(case)
    rows = sc.updated_rows(case, ref)
    assert rows.sum() > 0 and (~rows[1:]).sum() > 0
    rs = np.random.RandomState(1)
    E, b = t(case['E']), t(case['bias'])
    wd = f['wd']
    if f['opt'] == 'sgd':
        lr = 0.3 / max(np.abs(ref['dE']).max(), np.abs(ref['dbias']).max())
        fused = dict(kind=_lib.OPT_SGD, lr=lr, weight_decay=wd, eps=0.0)
        E_exp = sc.sgd(case['E'], ref['dE'], rows[:, None], lr, wd)
        b_exp = sc.sgd(case['bias'], ref['dbias'], rows[:, None], lr, wd)
    else:
        lr, eps = 0.05, 1e-10
        sE0 = (rs.rand(*case['E'].shape) * 0.02 + 1e-4).astype(np.float32)
        sb0 = (rs.rand(*case['bias'].shape) * 0.02 + 1e-4).astype(np.float32)
        sE, sb = t(sE0), t(sb0)
        fused = dict(kind=_lib.OPT_ADAGRAD, lr=lr, weight_decay=wd, eps=eps, state_E=sE, state_bias=sb)
        E_exp, sE_exp = sc.adagrad(case['E'], sE0, ref['dE'], rows[:, None], lr, wd, eps)
        b_exp, sb_exp = sc.adagrad(case['bias'], sb0, ref['dbias'], rows[:, None], lr, wd, eps)
    out = run_step(case, E, b, fused=fused)
    assert out['dE'] is None and out['dbias'] is None
    assert_close(out['loss'].item(), ref['loss'], 1e-5, what='loss')
    En, bn = E.cpu().numpy(), b.cpu().numpy()
    assert_close(En, E_exp, 5e-6, what='E')
    assert_close(bn, b_exp, 5e-6, what='bias')
    assert (En[~rows] == case['E'][~rows]).all() and (bn[~rows] == case['bias'][~rows]).all(), \
        'a row without gradient terms changed'
    if f['opt'] == 'adagrad':
        assert_close(sE.cpu().numpy(), sE_exp, 1e-5, what='Adagrad sum (E)')
        assert_close(sb.cpu().numpy(), sb_exp, 1e-5, what='Adagrad sum (bias)')
        assert (sE.cpu().numpy()[~rows] == sE0[~rows]).all()
    for i, (dW, db) in enumerate(ref.get('dconvs', [])):
        assert_close(out['dconv_w'][i].cpu().numpy(), dW, 2e-5, what='dW%d' % i)
        assert_close(out['dconv_b'][i].cpu().numpy(), db, 2e-5, what='db%d' % i)


# ------------------------------------------------------------------ workspace reuse
def test_workspace_reuse_across_shapes():
    """One num_items, so one cached workspace (zero-at-rest counters), through training and
    representation calls that change B, S, D, the layer stack and the kernel width."""
    I = 997
    calls = [
        ('train', dict(net='cnn', D=128, S=60, B=16, loss='bpr', kernel_width=(2, 5, 3), dilation=(1, 2, 1))),
        ('rep', dict(net='pool', D=64, S=200, B=5)),
        ('train', dict(net='pool', D=16, S=40, B=30, loss='hinge')),
        ('rep', dict(net='cnn', D=32, S=20, B=4, kernel_width=(1, 2, 5, 16, 2, 1, 5, 2), dilation=(1,) * 8)),
        ('train', dict(net='cnn', D=32, S=7, B=9, loss='adaptive_hinge', n_neg=3, kernel_width=(16,))),
        ('train', dict(net='cnn', D=128, S=200, B=3, loss='pointwise', kernel_width=(1,), nonlinearity='relu')),
        ('rep', dict(net='cnn', D=128, S=9, B=7, kernel_width=(3, 2), dilation=(2, 1), residual=False)),
        ('train', dict(net='pool', D=512, S=9, B=4, loss='bpr')),
        ('train', dict(net='cnn', D=20, S=33, B=6, loss='hinge', kernel_width=(5, 3), dilation=(3, 1))),
    ]
    for n, (kind, kw) in enumerate(calls):
        kw = dict(kw)
        if 'kernel_width' in kw and 'dilation' not in kw:
            kw['dilation'] = (1,) * len(kw['kernel_width'])
        case = sc.make_case(I=I, seed=40 + n, **kw)
        if kind == 'train':
            check_step(case, run_step(case), sc.oracle_step(case))
        else:
            check_representation(case)


# ------------------------------------------------------------------ configs[4] size
@pytest.mark.parametrize('net', ['pool', 'cnn'])
def test_config5_size(net):
    """1M items, D = 128, S = 200, B = 1024, pointwise; CNNNet with one k = 3 layer."""
    case = sc.make_case(net, D=128, S=200, B=1024, I=1000000, loss='pointwise', kernel_width=(3,),
                        dilation=(1,), seed=2024)
    ref = sc.oracle_step(case)
    out = run_step(case)
    touched = np.unique(np.concatenate([case['seqs'].ravel(), case['negs'].ravel()]))
    check_step(case, out, ref, rows=touched)
    dE = out['dE']
    mask = torch.ones(dE.shape[0], dtype=torch.bool, device=dE.device)
    mask[t(touched)] = False
    assert float(dE[mask].abs().max()) == 0.0


# ------------------------------------------------------------------ model level
@pytest.mark.parametrize('rep', ['pooling', 'cnn'])
def test_fit_fused_adagrad_matches_torch_adagrad(rep, capsys):
    """ImplicitSequenceModel.fit with optim.fused_adagrad (item table updated inside the step)
    against a copy trained with torch.optim.Adagrad on the step's dense gradients."""
    from spotlight_b200 import optim
    from spotlight_b200.interactions import SequenceInteractions
    from spotlight_b200.sequence.implicit import ImplicitSequenceModel
    rs = np.random.RandomState(17)
    seqs = rs.randint(1, 300, (400, 12)).astype(np.int32)
    for b in range(0, 400, 3):
        seqs[b, :rs.randint(0, 12)] = 0
    inter = SequenceInteractions(seqs, num_items=300)

    def fit(opt_func, state=None):
        model = ImplicitSequenceModel(loss='bpr', representation=rep, embedding_dim=32, batch_size=64,
                                      n_iter=2, optimizer_func=opt_func, use_cuda=True,
                                      random_state=np.random.RandomState(5))
        model._initialize(inter)
        if state is not None:
            model._net.load_state_dict(state)
        init = {k: v.clone() for k, v in model._net.state_dict().items()}
        capsys.readouterr()
        model.fit(inter, verbose=True)
        lines = [l for l in capsys.readouterr().out.strip().split('\n') if l.startswith('Epoch')]
        return model, init, np.array([float(l.split('loss')[1]) for l in lines])

    fused, init, lf = fit(optim.fused_adagrad(lr=0.05))
    assert fused._route() == 'fused' and fused._net.item_embeddings.weight.grad is None
    plain, _, lp = fit(lambda p: torch.optim.Adagrad(p, lr=0.05), init)
    assert len(lf) == 2
    assert_close(lf, lp, 1e-5, what='epoch losses')
    for k, v in plain._net.state_dict().items():
        assert_close(fused._net.state_dict()[k].cpu().numpy(), v.cpu().numpy(), 1e-4, atol=1e-7, what=k)
