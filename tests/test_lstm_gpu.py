"""The fused LSTMNet sequence step (csrc/seq_lstm.cuh plus the k = 1 conv GEMMs) and its
representation against the float64 oracle and the live reference's fixtures: every cluster size
(c = 1 up to D = 64, 4 up to 128, 8 up to 256), the wgmma projections at D = 128, idle units
(D = 100), partial sequence tiles, all four losses, padding, the fused optimizers,
reproducibility, workspace reuse, the configs[4] size, fit() and the generic route.

Tolerances are those of tests/test_seq_oracle_gpu.py: loss and scores 1e-5, gradients 2e-5, each
relative to the tensor's maximum magnitude.  tests/test_lstm_oracle_cpu.py shows that they catch
plausible recurrence mistakes on the same cases."""

import numpy as np
import pytest
import torch

from conftest import assert_close, load_golden
from oracle import lstm_cases as lc
from oracle import seq_cases as sc

pytestmark = pytest.mark.gpu

LSTM_KEYS = ('w_ih', 'w_hh', 'b_ih', 'b_hh')
SD_KEYS = dict(w_ih='weight_ih_l0', w_hh='weight_hh_l0', b_ih='bias_ih_l0', b_hh='bias_hh_l0')


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to('cuda:0')


def run_step(case, E=None, bias=None, **kw):
    from spotlight_b200 import ops
    E = t(case['E']) if E is None else E
    bias = t(case['bias']) if bias is None else bias
    lstm = {k: t(v) for k, v in case['lstm'].items()}
    return ops.seq_train_step(E, bias, t(case['seqs']), t(case['negs']), case['loss'], case['n_neg'], None,
                              want_scores=True, lstm=lstm, **kw)


def check_lstm_grads(out, ref):
    for k in LSTM_KEYS:
        assert_close(out['dlstm'][k].cpu().numpy(), ref['dlstm'][k], 2e-5, what='d' + k)


def check_step(case, out, ref, rows=None):
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
    check_lstm_grads(out, ref)


def check_representation(case):
    from spotlight_b200 import ops
    lstm = {k: t(v) for k, v in case['lstm'].items()}
    rep = ops.seq_representation(t(case['E']), t(case['seqs']), None, lstm=lstm)
    assert_close(rep.cpu().numpy(), lc.oracle_representation(case), 1e-5, what='representation')


def run_case(case):
    ref = lc.oracle_step(case)
    assert lc.check_properties(case, ref) == []
    check_step(case, run_step(case), ref)
    check_representation(case)
    return ref


# ------------------------------------------------------------------ dimensions and shapes
DIMS = [4, 12, 32, 64, 100, 128, 256]


@pytest.mark.parametrize('D', DIMS)
def test_dims(D):
    case = lc.make_case(D=D, S=23, B=11, loss=sc.LOSS_CYCLE[DIMS.index(D) % 4], n_neg=2, seed=D)
    run_case(case)


@pytest.mark.parametrize('S', [1, 2, 23, 200])
@pytest.mark.parametrize('B', [1, 11, 64])
def test_shapes(S, B):
    D = 128 if (S + B) % 2 else 32
    case = lc.make_case(D=D, S=S, B=B, loss='bpr', seed=S * 100 + B)
    run_case(case)


# ------------------------------------------------------------------ losses and padding
LOSSES = [('pointwise', 1), ('bpr', 1), ('hinge', 1), ('adaptive_hinge', 2), ('adaptive_hinge', 5)]


@pytest.mark.parametrize('loss,n_neg', LOSSES, ids=['pointwise', 'bpr', 'hinge', 'adaptive2', 'adaptive5'])
@pytest.mark.parametrize('D', [32, 128])
def test_losses(D, loss, n_neg):
    case = lc.make_case(D=D, S=20, B=16, loss=loss, n_neg=n_neg, seed=7 + n_neg)
    run_case(case)


@pytest.mark.parametrize('D', [32, 128])
def test_adaptive_hinge_tied_negatives(D):
    case = lc.make_case(D=D, S=20, B=16, loss='adaptive_hinge', n_neg=2, neg_tie=True, seed=11)
    ref = run_case(case)
    half = case['E'].shape[0] // 2
    assert (ref['dE'][half + 1] != 0).any() and (ref['dE'][half + 2] != 0).any()


@pytest.mark.parametrize('D', [32, 128])
def test_padding_and_zeros(D):
    """A fully padded sequence, padding mid-sequence (the state still advances through it),
    padding negatives and a non-zero E[0] read as stored (dE[0] / dbias[0] stay 0)."""
    case = lc.make_case(D=D, S=30, B=9, loss='bpr', e0_nonzero=True, zero_frac=0.3, seed=5)
    assert (case['seqs'][0] == 0).all() and (case['negs'] == 0).any() and (case['E'][0] != 0).all()
    run_case(case)


# ------------------------------------------------------------------ fused optimizers
@pytest.mark.parametrize('opt,wd', [('sgd', 0.0), ('sgd', 0.1), ('adagrad', 0.0), ('adagrad', 0.05)])
def test_fused_optimizer(opt, wd):
    """SGD / Adagrad fused into the item-table reduction, against torch's update rules on the
    oracle gradients (rows as tests/test_seq_oracle_gpu.py); the LSTM gradients are returned."""
    from spotlight_b200 import _lib
    case = lc.make_case(D=64, S=20, B=16, loss='hinge' if opt == 'sgd' else 'bpr', seed=3)
    ref = lc.oracle_step(case)
    rows = sc.updated_rows(case, ref)
    E, b = t(case['E']), t(case['bias'])
    if opt == 'sgd':
        lr = 0.3 / max(np.abs(ref['dE']).max(), np.abs(ref['dbias']).max())
        fused = dict(kind=_lib.OPT_SGD, lr=lr, weight_decay=wd, eps=0.0)
        E_exp = sc.sgd(case['E'], ref['dE'], rows[:, None], lr, wd)
        b_exp = sc.sgd(case['bias'], ref['dbias'], rows[:, None], lr, wd)
    else:
        rs = np.random.RandomState(1)
        lr, eps = 0.05, 1e-10
        sE0 = (rs.rand(*case['E'].shape) * 0.02 + 1e-4).astype(np.float32)
        sb0 = (rs.rand(*case['bias'].shape) * 0.02 + 1e-4).astype(np.float32)
        sE, sb = t(sE0), t(sb0)
        fused = dict(kind=_lib.OPT_ADAGRAD, lr=lr, weight_decay=wd, eps=eps, state_E=sE, state_bias=sb)
        E_exp, sE_exp = sc.adagrad(case['E'], sE0, ref['dE'], rows[:, None], lr, wd, eps)
        b_exp, _ = sc.adagrad(case['bias'], sb0, ref['dbias'], rows[:, None], lr, wd, eps)
    out = run_step(case, E, b, fused=fused)
    assert out['dE'] is None and out['dbias'] is None
    assert_close(out['loss'].item(), ref['loss'], 1e-5, what='loss')
    En, bn = E.cpu().numpy(), b.cpu().numpy()
    assert_close(En, E_exp, 5e-6, what='E')
    assert_close(bn, b_exp, 5e-6, what='bias')
    assert (En[~rows] == case['E'][~rows]).all() and (bn[~rows] == case['bias'][~rows]).all()
    if opt == 'adagrad':
        assert_close(sE.cpu().numpy(), sE_exp, 1e-5, what='Adagrad sum (E)')
    check_lstm_grads(out, ref)


# ------------------------------------------------------------------ reproducibility, workspace
@pytest.mark.parametrize('D', [32, 128, 256])
def test_bit_reproducible(D):
    case = lc.make_case(D=D, S=40, B=70, loss='adaptive_hinge', n_neg=3, seed=D + 1)
    a, b = run_step(case), run_step(case)
    for k in ('pos', 'neg', 'loss', 'dE', 'dbias'):
        assert torch.equal(a[k], b[k]), k
    for k in LSTM_KEYS:
        assert torch.equal(a['dlstm'][k], b['dlstm'][k]), k


def test_workspace_reuse_across_nets():
    """LSTM, CNN and pool steps and representations alternate on one cached workspace."""
    from spotlight_b200 import ops
    I = 997
    calls = [
        ('train', dict(net='lstm', D=128, S=60, B=16, loss='bpr')),
        ('train', dict(net='cnn', D=128, S=30, B=8, loss='hinge', kernel_width=(3,), dilation=(1,))),
        ('rep', dict(net='lstm', D=64, S=200, B=5)),
        ('train', dict(net='pool', D=16, S=40, B=30, loss='hinge')),
        ('train', dict(net='lstm', D=256, S=9, B=4, loss='pointwise')),
        ('rep', dict(net='cnn', D=32, S=20, B=4, kernel_width=(2, 5), dilation=(1, 1))),
        ('train', dict(net='lstm', D=12, S=33, B=6, loss='adaptive_hinge', n_neg=3)),
    ]
    for n, (kind, kw) in enumerate(calls):
        kw = dict(kw)
        if kw.pop('net') == 'lstm':
            case = lc.make_case(I=I, seed=60 + n, **kw)
            if kind == 'train':
                check_step(case, run_step(case), lc.oracle_step(case))
            else:
                check_representation(case)
            continue
        case = sc.make_case(I=I, seed=60 + n, net='cnn' if 'kernel_width' in kw else 'pool', **kw)
        spec = None
        if case['cnn'] is not None:
            spec = dict(case['cnn'], weights=[t(w) for w, _ in case['convs']], biases=[t(b) for _, b in case['convs']])
        if kind == 'train':
            out = ops.seq_train_step(t(case['E']), t(case['bias']), t(case['seqs']), t(case['negs']),
                                     case['loss'], case['n_neg'], spec)
            ref = sc.oracle_step(case)
            assert_close(out['loss'].item(), ref['loss'], 1e-5, what='loss')
            assert_close(out['dE'].cpu().numpy(), ref['dE'], 2e-5, what='dE')
        else:
            rep = ops.seq_representation(t(case['E']), t(case['seqs']), spec)
            assert_close(rep.cpu().numpy(), sc.oracle_representation(case), 1e-5, what='representation')


def test_config5_size():
    """1M items, D = 128, S = 200, B = 256 (the reference's default batch), pointwise."""
    case = lc.make_case(D=128, S=200, B=256, I=1000000, loss='pointwise', seed=2024)
    ref = lc.oracle_step(case)
    out = run_step(case)
    touched = np.unique(np.concatenate([case['seqs'].ravel(), case['negs'].ravel()]))
    check_step(case, out, ref, rows=touched)
    mask = torch.ones(out['dE'].shape[0], dtype=torch.bool, device=out['dE'].device)
    mask[t(touched)] = False
    assert float(out['dE'][mask].abs().max()) == 0.0


# ------------------------------------------------------------------ live-reference fixtures
def golden_lstm(g):
    lstm, rows = lc.golden_lstm(g)
    return {k: t(v) for k, v in lstm.items()}, rows


@pytest.mark.parametrize('name,loss', [('lstm_pointwise', 'pointwise'), ('lstm_adaptive_hinge', 'adaptive_hinge'),
                                       ('lstm_bpr_d128', 'bpr')])
def test_step_golden(name, loss):
    from spotlight_b200 import ops
    g = load_golden(name)
    n_neg = int(g['n_neg']) if loss == 'adaptive_hinge' else 1
    E = t(g['sd.item_embeddings.weight'])
    lstm, rows = golden_lstm(g)                    # rows: the D = 128 fixture's sampled gradient rows
    out = ops.seq_train_step(E, t(g['sd.item_biases.weight']), t(g['seqs']), t(g['negs']), loss, n_neg, None,
                             want_scores=True, lstm=lstm)
    assert_close(out['pos'].cpu().numpy(), g['pos'], 1e-5, what='pos')
    assert_close(out['neg'].cpu().numpy().reshape(g['neg'].shape), g['neg'], 1e-5, what='neg')
    assert_close(out['loss'].item(), g['loss'], 1e-5, what='loss')
    assert_close(out['dE'].cpu().numpy(), g['grad.item_embeddings.weight'], 2e-5, what='dE')
    assert_close(out['dbias'].cpu().numpy(), g['grad.item_biases.weight'], 2e-5, what='dbias')
    for k, v in SD_KEYS.items():
        d = out['dlstm'][k].cpu().numpy()
        assert_close(d if rows is None or d.ndim == 1 else d[rows], g['grad.lstm.' + v], 2e-5, what=k)
    rep = ops.seq_representation(E, t(g['seqs']), None, lstm=lstm)
    assert_close(rep[:, -1].cpu().numpy(), g['final'], 1e-5, what='final')
    assert_close(rep[:, :-1].permute(0, 2, 1).cpu().numpy(), g['user_rep'], 1e-5, what='user_rep')


def _fit_model(g, optimizer_func):
    from spotlight_b200.interactions import SequenceInteractions
    from spotlight_b200.sequence.implicit import ImplicitSequenceModel
    inter = SequenceInteractions(g['seqs'], num_items=int(g['num_items']))
    model = ImplicitSequenceModel(loss='bpr', representation='lstm', embedding_dim=int(g['dim']),
                                  batch_size=int(g['batch']), n_iter=int(g['n_iter']),
                                  optimizer_func=optimizer_func, use_cuda=True,
                                  random_state=np.random.RandomState(int(g['seed'])))
    model._initialize(inter)
    model._net.load_state_dict({k[5:]: torch.from_numpy(v) for k, v in g.items() if k.startswith('init.')})
    return model, inter


def _epoch_losses(capsys):
    lines = [l for l in capsys.readouterr().out.strip().split('\n') if l.startswith('Epoch')]
    return np.array([float(l.split('loss')[1]) for l in lines])


@pytest.mark.parametrize('fused', [False, True], ids=['torch_sgd', 'fused_sgd'])
def test_fit_golden(fused, capsys):
    """fit() against the reference's trajectory: epoch losses, final state_dict, RandomState
    position and predict."""
    from spotlight_b200 import optim
    g = load_golden('fit_lstm_sgd')
    opt = optim.fused_sgd(lr=0.5) if fused else (lambda p: torch.optim.SGD(p, lr=0.5))
    model, inter = _fit_model(g, opt)
    assert model._route() == 'fused'
    capsys.readouterr()
    model.fit(inter, verbose=True)
    assert_close(_epoch_losses(capsys), g['epoch_losses'], 1e-5, what='epoch losses')
    for k, v in model._net.state_dict().items():
        assert_close(v.cpu().numpy(), g['final.' + k], 1e-4, atol=1e-7, what=k)
    st = model._random_state.get_state()
    assert (st[1] == g['rs_key']).all() and st[2] == int(g['rs_pos'])
    assert_close(model.predict(g['seqs'][1]), g['predict'], 1e-4, what='predict')


def test_fit_fused_adagrad_matches_torch_adagrad(capsys):
    from spotlight_b200 import optim
    g = load_golden('fit_lstm_sgd')
    fused, inter = _fit_model(g, optim.fused_adagrad(lr=0.05))
    fused.fit(inter, verbose=True)
    lf = _epoch_losses(capsys)
    assert fused._route() == 'fused' and fused._net.item_embeddings.weight.grad is None
    plain, _ = _fit_model(g, lambda p: torch.optim.Adagrad(p, lr=0.05))
    plain.fit(inter, verbose=True)
    lp = _epoch_losses(capsys)
    assert len(lf) == 2
    assert_close(lf, lp, 1e-5, what='epoch losses')
    for k, v in plain._net.state_dict().items():
        assert_close(fused._net.state_dict()[k].cpu().numpy(), v.cpu().numpy(), 1e-4, atol=1e-7, what=k)


# ------------------------------------------------------------------ generic route
def test_autograd_route_matches_kernel():
    """With autograd enabled LSTMNet runs nn.LSTM; its gradients equal the oracle's, and the
    no-grad representation (the kernel) equals the autograd one.  cuDNN's TF32 mode is switched
    off here: with it (torch's default for cuDNN) the dE of this case is off by 4e-4 of its
    maximum."""
    from spotlight_b200 import losses
    from spotlight_b200.sequence.representations import LSTMNet
    case = lc.make_case(D=32, S=15, B=9, loss='pointwise', seed=21)
    I, D = case['E'].shape
    net = LSTMNet(I, D)
    sd = {'item_embeddings.weight': torch.from_numpy(case['E']), 'item_biases.weight': torch.from_numpy(case['bias'])}
    sd.update({'lstm.' + v: torch.from_numpy(case['lstm'][k]) for k, v in SD_KEYS.items()})
    net.load_state_dict(sd)
    net = net.to('cuda:0')
    assert net.fusable()
    seqs, negs = t(case['seqs']), t(case['negs'])
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
        rep, final = net.user_representation(seqs)
        assert rep.requires_grad
        loss = losses.pointwise_loss(net(rep, seqs), net(rep, negs), mask=(seqs != 0))
        loss.backward()
    ref = lc.oracle_step(case)
    assert_close(loss.item(), ref['loss'], 1e-5, what='loss')
    assert_close(net.item_embeddings.weight.grad.cpu().numpy(), ref['dE'], 2e-5, what='dE')
    for k, v in SD_KEYS.items():
        assert_close(getattr(net.lstm, v).grad.cpu().numpy(), ref['dlstm'][k], 2e-5, what=k)
    with torch.no_grad():
        rep_k, final_k = net.user_representation(seqs)
    assert_close(rep_k.cpu().numpy(), rep.detach().cpu().numpy(), 1e-5, what='representation')
    assert_close(final_k.cpu().numpy(), final.detach().cpu().numpy(), 1e-5, what='final')


@pytest.mark.parametrize('kind', ['bloom', 'd260'])
def test_generic_route_fit_runs(kind):
    """A Bloom-embedded LSTMNet and D = 260 (beyond the fused range) train on the generic route."""
    from spotlight_b200.interactions import SequenceInteractions
    from spotlight_b200.layers import BloomEmbedding
    from spotlight_b200.sequence.implicit import ImplicitSequenceModel
    from spotlight_b200.sequence.representations import LSTMNet
    rs = np.random.RandomState(0)
    seqs = rs.randint(1, 200, (64, 8)).astype(np.int32)
    if kind == 'bloom':
        D = 16
        rep = LSTMNet(200, D, item_embedding_layer=BloomEmbedding(200, D, compression_ratio=0.5,
                                                                  num_hash_functions=2, padding_idx=0))
    else:
        D = 260
        rep = LSTMNet(200, D)
    model = ImplicitSequenceModel(loss='bpr', representation=rep, embedding_dim=D, batch_size=32,
                                  n_iter=2, use_cuda=True, random_state=np.random.RandomState(1))
    model.fit(SequenceInteractions(seqs, num_items=200))
    assert model._route() == 'generic' and not model._net.fusable()
    assert np.isfinite(model.predict(seqs[0])).all()
