"""The fused MixtureLSTMNet sequence step (the LSTM of csrc/seq_lstm.cuh, the 2M projection GEMMs
and mix_score_kernel of csrc/seq_mix.cuh) and its representation against the float64 oracle and the
live reference's fixtures: every cluster size, the wgmma projections at D = 128, idle units
(D = 100), M in {1, 2, 4, 8}, all four losses, padding, the fused optimizers, reproducibility,
workspace reuse, the configs[4] size, fit() and the generic route.

Tolerances are those of tests/test_lstm_gpu.py: loss and scores 1e-5, gradients 2e-5, each relative
to the tensor's maximum magnitude.  tests/test_mixture_oracle_cpu.py shows that they catch
plausible mistakes of the head and the projection on the same cases."""

import numpy as np
import pytest
import torch

from conftest import assert_close, load_golden
from oracle import lstm_cases as lc
from oracle import mixture_cases as mc
from oracle import seq_cases as sc

pytestmark = pytest.mark.gpu

LSTM_KEYS = ('w_ih', 'w_hh', 'b_ih', 'b_hh')
SD_KEYS = dict(w_ih='weight_ih_l0', w_hh='weight_hh_l0', b_ih='bias_ih_l0', b_hh='bias_hh_l0')


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to('cuda:0')


def specs(case):
    lstm = {k: t(v) for k, v in case['lstm'].items()}
    mixture = dict(num_mixtures=case['M'], w=t(case['proj']['w']), b=t(case['proj']['b']))
    return lstm, mixture


def run_step(case, E=None, bias=None, **kw):
    from spotlight_b200 import ops
    E = t(case['E']) if E is None else E
    bias = t(case['bias']) if bias is None else bias
    lstm, mixture = specs(case)
    return ops.seq_train_step(E, bias, t(case['seqs']), t(case['negs']), case['loss'], case['n_neg'], None,
                              want_scores=True, lstm=lstm, mixture=mixture, **kw)


def check_net_grads(out, ref):
    for k in LSTM_KEYS:
        assert_close(out['dlstm'][k].cpu().numpy(), ref['dlstm'][k], 2e-5, what='d' + k)
    assert out['dmix']['w'].shape == ref['dmix']['w'].shape
    assert_close(out['dmix']['w'].cpu().numpy(), ref['dmix']['w'], 2e-5, what='dmix w')
    assert_close(out['dmix']['b'].cpu().numpy(), ref['dmix']['b'], 2e-5, what='dmix b')


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
    check_net_grads(out, ref)


def check_representation(case):
    from spotlight_b200 import ops
    lstm, mixture = specs(case)
    rep = ops.seq_representation(t(case['E']), t(case['seqs']), None, lstm=lstm, mixture=mixture)
    assert_close(rep.cpu().numpy(), mc.oracle_representation(case), 1e-5, what='representation')


def run_case(case):
    ref = mc.oracle_step(case)
    assert mc.check_properties(case, ref) == []
    check_step(case, run_step(case), ref)
    check_representation(case)
    return ref


# ------------------------------------------------------------------ dimensions, mixtures, shapes
DIMS = [4, 12, 32, 64, 100, 128, 256]


@pytest.mark.parametrize('D', DIMS)
def test_dims(D):
    case = mc.make_case(D=D, S=23, B=11, loss=sc.LOSS_CYCLE[DIMS.index(D) % 4], n_neg=2, M=4, seed=D)
    run_case(case)


@pytest.mark.parametrize('M', [1, 2, 4, 8])
@pytest.mark.parametrize('D', [32, 128])
def test_num_mixtures(D, M):
    case = mc.make_case(D=D, S=20, B=16, loss='bpr', M=M, seed=D + M)
    run_case(case)


def test_single_mixture_is_lstm_plus_projection():
    """M = 1: the score is beta + c_0 . e with the mixture weight 1, so the step equals an LSTMNet
    step whose representation is the component block: an LSTMNet with identity projection (W = I,
    b = 0) gives the LSTMNet step's scores and LSTM gradients."""
    case = mc.make_case(D=32, S=20, B=16, loss='hinge', M=1, seed=4)
    D = 32
    case['proj'] = dict(w=np.concatenate([np.eye(D), np.eye(D)]).astype(np.float32)[:, :, None],
                        b=np.zeros(2 * D, np.float32))
    out = run_step(case)
    from spotlight_b200 import ops
    plain = ops.seq_train_step(t(case['E']), t(case['bias']), t(case['seqs']), t(case['negs']), case['loss'],
                               case['n_neg'], None, want_scores=True, lstm={k: t(v) for k, v in case['lstm'].items()})
    ref = lc.oracle_step(case)
    assert_close(out['pos'].cpu().numpy(), ref['pos'], 1e-5, what='pos')
    assert_close(out['loss'].item(), plain['loss'].item(), 1e-5, what='loss')
    assert_close(out['dE'].cpu().numpy(), plain['dE'].cpu().numpy(), 2e-5, what='dE')
    for k in LSTM_KEYS:
        assert_close(out['dlstm'][k].cpu().numpy(), plain['dlstm'][k].cpu().numpy(), 2e-5, what=k)


@pytest.mark.parametrize('S', [1, 2, 23, 200])
@pytest.mark.parametrize('B', [1, 11, 64])
def test_shapes(S, B):
    D = 128 if (S + B) % 2 else 32
    case = mc.make_case(D=D, S=S, B=B, loss='bpr', M=4, seed=S * 100 + B)
    ref = mc.oracle_step(case)
    check_step(case, run_step(case), ref)
    check_representation(case)


# ------------------------------------------------------------------ losses and padding
LOSSES = [('pointwise', 1), ('bpr', 1), ('hinge', 1), ('adaptive_hinge', 2), ('adaptive_hinge', 5)]


@pytest.mark.parametrize('loss,n_neg', LOSSES, ids=['pointwise', 'bpr', 'hinge', 'adaptive2', 'adaptive5'])
@pytest.mark.parametrize('D', [32, 128])
def test_losses(D, loss, n_neg):
    case = mc.make_case(D=D, S=20, B=16, loss=loss, n_neg=n_neg, seed=7 + n_neg)
    run_case(case)


@pytest.mark.parametrize('D', [32, 128])
def test_adaptive_hinge_tied_negatives(D):
    """Bit-identical negatives score identically; the first of them takes the gradient."""
    case = mc.make_case(D=D, S=20, B=16, loss='adaptive_hinge', n_neg=2, neg_tie=True, seed=11)
    ref = run_case(case)
    half = case['E'].shape[0] // 2
    assert (ref['dE'][half + 1] != 0).any() and (ref['dE'][half + 2] != 0).any()


@pytest.mark.parametrize('D', [32, 128])
def test_padding_and_zeros(D):
    """A fully padded sequence, padding mid-sequence (the state still advances through it),
    padding negatives and a non-zero E[0] read as stored (dE[0] / dbias[0] stay 0)."""
    case = mc.make_case(D=D, S=30, B=9, loss='bpr', e0_nonzero=True, zero_frac=0.3, seed=5)
    assert (case['seqs'][0] == 0).all() and (case['negs'] == 0).any() and (case['E'][0] != 0).all()
    run_case(case)


# ------------------------------------------------------------------ fused optimizers
@pytest.mark.parametrize('opt,wd', [('sgd', 0.0), ('sgd', 0.1), ('adagrad', 0.0), ('adagrad', 0.05)])
def test_fused_optimizer(opt, wd):
    from spotlight_b200 import _lib
    case = mc.make_case(D=64, S=20, B=16, loss='hinge' if opt == 'sgd' else 'bpr', seed=3)
    ref = mc.oracle_step(case)
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
    check_net_grads(out, ref)


# ------------------------------------------------------------------ reproducibility, workspace
@pytest.mark.parametrize('D', [32, 128, 256])
def test_bit_reproducible(D):
    case = mc.make_case(D=D, S=40, B=70, loss='adaptive_hinge', n_neg=3, M=8 if D == 32 else 4, seed=D + 1)
    a, b = run_step(case), run_step(case)
    for k in ('pos', 'neg', 'loss', 'dE', 'dbias'):
        assert torch.equal(a[k], b[k]), k
    for k in LSTM_KEYS:
        assert torch.equal(a['dlstm'][k], b['dlstm'][k]), k
    for k in ('w', 'b'):
        assert torch.equal(a['dmix'][k], b['dmix'][k]), k


def test_workspace_reuse_across_nets():
    """Mixture, LSTM, CNN and pool steps and representations alternate on one cached workspace."""
    from spotlight_b200 import ops
    I = 997
    calls = [
        ('train', dict(net='mixture', D=128, S=60, B=16, loss='bpr', M=4)),
        ('train', dict(net='lstm', D=64, S=30, B=8, loss='hinge')),
        ('rep', dict(net='mixture', D=64, S=200, B=5, M=8)),
        ('train', dict(net='cnn', D=128, S=30, B=8, loss='hinge', kernel_width=(3,), dilation=(1,))),
        ('train', dict(net='pool', D=16, S=40, B=30, loss='hinge')),
        ('train', dict(net='mixture', D=256, S=9, B=4, loss='pointwise', M=2)),
        ('rep', dict(net='lstm', D=32, S=20, B=4)),
        ('train', dict(net='mixture', D=12, S=33, B=6, loss='adaptive_hinge', n_neg=3, M=3)),
    ]
    for n, (kind, kw) in enumerate(calls):
        kw = dict(kw)
        net = kw.pop('net')
        if net == 'mixture':
            case = mc.make_case(I=I, seed=60 + n, **kw)
            if kind == 'train':
                check_step(case, run_step(case), mc.oracle_step(case))
            else:
                check_representation(case)
            continue
        if net == 'lstm':
            case = lc.make_case(I=I, seed=60 + n, **kw)
            lstm = {k: t(v) for k, v in case['lstm'].items()}
            if kind == 'train':
                out = ops.seq_train_step(t(case['E']), t(case['bias']), t(case['seqs']), t(case['negs']),
                                         case['loss'], case['n_neg'], None, lstm=lstm)
                ref = lc.oracle_step(case)
                assert_close(out['loss'].item(), ref['loss'], 1e-5, what='loss')
                assert_close(out['dE'].cpu().numpy(), ref['dE'], 2e-5, what='dE')
            else:
                rep = ops.seq_representation(t(case['E']), t(case['seqs']), None, lstm=lstm)
                assert_close(rep.cpu().numpy(), lc.oracle_representation(case), 1e-5, what='representation')
            continue
        case = sc.make_case(I=I, seed=60 + n, net=net, **kw)
        spec = None
        if case['cnn'] is not None:
            spec = dict(case['cnn'], weights=[t(w) for w, _ in case['convs']], biases=[t(b) for _, b in case['convs']])
        out = ops.seq_train_step(t(case['E']), t(case['bias']), t(case['seqs']), t(case['negs']),
                                 case['loss'], case['n_neg'], spec)
        ref = sc.oracle_step(case)
        assert_close(out['loss'].item(), ref['loss'], 1e-5, what='loss')
        assert_close(out['dE'].cpu().numpy(), ref['dE'], 2e-5, what='dE')


def test_config5_size():
    """1M items, D = 128, S = 200, B = 256, M = 4, pointwise: the loss is finite and the gradients
    of the touched rows and of the net equal an fp32 ATen restatement (autograd through nn.LSTM,
    nn.Conv1d and the reference's head, TF32 off) to 1e-5 of their maximum."""
    from spotlight_b200.sequence.representations import MixtureLSTMNet
    case = mc.make_case(D=128, S=200, B=256, I=1000000, loss='pointwise', M=4, seed=2024)
    out = run_step(case)
    assert np.isfinite(out['loss'].item())
    I, D = case['E'].shape
    net = MixtureLSTMNet(I, D, num_mixtures=4).to('cuda:0')
    with torch.no_grad():
        net.item_embeddings.weight.copy_(t(case['E']))
        net.item_biases.weight.copy_(t(case['bias']))
        for k, v in SD_KEYS.items():
            getattr(net.lstm, v).copy_(t(case['lstm'][k]))
        net.projection.weight.copy_(t(case['proj']['w']))
        net.projection.bias.copy_(t(case['proj']['b']))
    seqs, negs = t(case['seqs']), t(case['negs'])
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
            rep, _ = net._user_representation_autograd(seqs)
            pos, neg = net(rep, seqs), net(rep, negs)
            mask = (seqs != 0).float()
            per = (1.0 - torch.sigmoid(pos)) + torch.sigmoid(neg)
            loss = (per * mask).sum() / mask.sum()
            loss.backward()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    assert_close(out['loss'].item(), loss.item(), 1e-5, what='loss')
    touched = t(np.unique(np.concatenate([case['seqs'].ravel(), case['negs'].ravel()])))
    assert_close(out['dE'][touched].cpu().numpy(), net.item_embeddings.weight.grad[touched].cpu().numpy(), 1e-5,
                 what='dE (touched rows)')
    assert_close(out['dbias'][touched].cpu().numpy(), net.item_biases.weight.grad[touched].cpu().numpy(), 1e-5,
                 what='dbias (touched rows)')
    mask = torch.ones(I, dtype=torch.bool, device=out['dE'].device)
    mask[touched] = False
    assert float(out['dE'][mask].abs().max()) == 0.0
    for k, v in SD_KEYS.items():
        assert_close(out['dlstm'][k].cpu().numpy(), getattr(net.lstm, v).grad.cpu().numpy(), 1e-5, what=k)
    assert_close(out['dmix']['w'].cpu().numpy(), net.projection.weight.grad.cpu().numpy(), 1e-5, what='dmix w')
    assert_close(out['dmix']['b'].cpu().numpy(), net.projection.bias.grad.cpu().numpy(), 1e-5, what='dmix b')


# ------------------------------------------------------------------ live-reference fixtures
@pytest.mark.parametrize('name,loss', [('mixture_pointwise', 'pointwise'), ('mixture_adaptive_hinge', 'adaptive_hinge'),
                                       ('mixture_bpr_d128', 'bpr')])
def test_step_golden(name, loss):
    from spotlight_b200 import ops
    g = load_golden(name)
    n_neg = int(g['n_neg']) if loss == 'adaptive_hinge' else 1
    M, D = int(g['num_mixtures']), int(g['dim'])
    lstm_np, proj, rows, prows = mc.golden_params(g)
    lstm = {k: t(v) for k, v in lstm_np.items()}
    mixture = dict(num_mixtures=M, w=t(proj['w']), b=t(proj['b']))
    E = t(g['sd.item_embeddings.weight'])
    out = ops.seq_train_step(E, t(g['sd.item_biases.weight']), t(g['seqs']), t(g['negs']), loss, n_neg, None,
                             want_scores=True, lstm=lstm, mixture=mixture)
    assert_close(out['pos'].cpu().numpy(), g['pos'], 1e-5, what='pos')
    assert_close(out['neg'].cpu().numpy().reshape(g['neg'].shape), g['neg'], 1e-5, what='neg')
    assert_close(out['loss'].item(), g['loss'], 1e-5, what='loss')
    assert_close(out['dE'].cpu().numpy(), g['grad.item_embeddings.weight'], 2e-5, what='dE')
    assert_close(out['dbias'].cpu().numpy(), g['grad.item_biases.weight'], 2e-5, what='dbias')
    for k, v in SD_KEYS.items():
        d = out['dlstm'][k].cpu().numpy()
        assert_close(d if rows is None or d.ndim == 1 else d[rows], g['grad.lstm.' + v], 2e-5, what=k)
    dw = out['dmix']['w'].cpu().numpy()
    assert_close(dw if prows is None else dw[prows], g['grad.projection.weight'], 2e-5, what='dmix w')
    assert_close(out['dmix']['b'].cpu().numpy(), g['grad.projection.bias'], 2e-5, what='dmix b')
    rep = ops.seq_representation(E, t(g['seqs']), None, lstm=lstm, mixture=mixture)
    B, T = rep.shape[:2]
    rep = rep.view(B, T, 2 * M, D).permute(0, 2, 3, 1)
    assert_close(rep[..., -1:].cpu().numpy(), g['final'], 1e-5, what='final')
    if 'user_rep' in g:
        assert_close(rep[..., :-1].cpu().numpy(), g['user_rep'], 1e-5, what='user_rep')


def test_user_representation_shapes():
    """The module protocol of the reference: (B, 2M, D, S) and (B, 2M, D, 1), from the kernels
    under no_grad and from nn.LSTM / nn.Conv1d under autograd, equal to each other."""
    from spotlight_b200.sequence.representations import MixtureLSTMNet
    net = MixtureLSTMNet(50, 16, num_mixtures=3).to('cuda:0')
    assert net.fusable()
    seqs = t(np.random.RandomState(0).randint(0, 50, (4, 7)).astype(np.int64))
    with torch.no_grad():
        rep_k, final_k = net.user_representation(seqs)
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
        rep_a, final_a = net.user_representation(seqs)
    assert rep_a.requires_grad and rep_k.shape == (4, 6, 16, 7) and final_k.shape == (4, 6, 16, 1)
    assert_close(rep_k.cpu().numpy(), rep_a.detach().cpu().numpy(), 1e-5, what='representation')
    assert_close(final_k.cpu().numpy(), final_a.detach().cpu().numpy(), 1e-5, what='final')


def _fit_model(g, optimizer_func):
    from spotlight_b200.interactions import SequenceInteractions
    from spotlight_b200.sequence.implicit import ImplicitSequenceModel
    inter = SequenceInteractions(g['seqs'], num_items=int(g['num_items']))
    model = ImplicitSequenceModel(loss='bpr', representation='mixture', embedding_dim=int(g['dim']),
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
    g = load_golden('fit_mixture_sgd')
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
    g = load_golden('fit_mixture_sgd')
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


def test_default_model_routes_fused():
    from spotlight_b200.interactions import SequenceInteractions
    from spotlight_b200.sequence.implicit import ImplicitSequenceModel
    seqs = np.random.RandomState(0).randint(1, 100, (32, 6)).astype(np.int32)
    model = ImplicitSequenceModel(representation='mixture', use_cuda=True, n_iter=1,
                                  random_state=np.random.RandomState(2))
    model.fit(SequenceInteractions(seqs, num_items=100))
    assert model._route() == 'fused'
    assert np.isfinite(model.predict(seqs[0])).all()


# ------------------------------------------------------------------ generic route
@pytest.mark.parametrize('kind', ['bloom', 'm9', 'd260'])
def test_generic_route_fit_runs(kind):
    """A Bloom-embedded mixture net, M = 9 and D = 260 (beyond the fused range) train on the generic route."""
    from spotlight_b200.interactions import SequenceInteractions
    from spotlight_b200.layers import BloomEmbedding
    from spotlight_b200.sequence.implicit import ImplicitSequenceModel
    from spotlight_b200.sequence.representations import MixtureLSTMNet
    rs = np.random.RandomState(0)
    seqs = rs.randint(1, 200, (64, 8)).astype(np.int32)
    if kind == 'bloom':
        D = 16
        rep = MixtureLSTMNet(200, D, item_embedding_layer=BloomEmbedding(200, D, compression_ratio=0.5,
                                                                         num_hash_functions=2, padding_idx=0))
    elif kind == 'm9':
        D = 16
        rep = MixtureLSTMNet(200, D, num_mixtures=9)
    else:
        D = 260
        rep = MixtureLSTMNet(200, D, num_mixtures=2)
    model = ImplicitSequenceModel(loss='bpr', representation=rep, embedding_dim=D, batch_size=32,
                                  n_iter=2, use_cuda=True, random_state=np.random.RandomState(1))
    model.fit(SequenceInteractions(seqs, num_items=200))
    assert model._route() == 'generic' and not model._net.fusable()
    assert np.isfinite(model.predict(seqs[0])).all()
