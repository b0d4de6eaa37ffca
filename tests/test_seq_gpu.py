"""GPU parity tests for the sequence hot path (PoolNet, CNNNet) against the
live reference's golden vectors and the oracle."""

import numpy as np
import pytest
import torch

from conftest import assert_close, load_golden
from oracle import seq as oseq

pytestmark = pytest.mark.gpu


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to('cuda:0')


def _cnn_spec(g):
    L = int(g['cnn.num_layers'])
    kw = np.atleast_1d(g['cnn.kernel_width'])
    dl = np.atleast_1d(g['cnn.dilation'])
    return dict(kernel_width=[int(kw[i % len(kw)]) for i in range(L)],
                dilation=[int(dl[i % len(dl)]) for i in range(L)],
                nonlinearity=str(g['cnn.nonlinearity']) if 'cnn.nonlinearity' in g else 'tanh',
                residual=bool(g['cnn.residual_connections']) if 'cnn.residual_connections' in g else True,
                weights=[t(g['sd.cnn_%d.weight' % i]) for i in range(L)],
                biases=[t(g['sd.cnn_%d.bias' % i]) for i in range(L)])


@pytest.mark.parametrize('name', ['pool_pointwise', 'pool_bpr', 'pool_hinge', 'pool_adaptive_hinge'])
def test_pool_step_golden(name):
    from spotlight_b200 import ops
    g = load_golden(name)
    loss = name.split('_', 1)[1]
    n_neg = int(g['n_neg']) if loss == 'adaptive_hinge' else 1
    out = ops.seq_train_step(t(g['sd.item_embeddings.weight']), t(g['sd.item_biases.weight']),
                             t(g['seqs']), t(g['negs']), loss, n_neg, None, want_scores=True)
    assert_close(out['pos'].cpu().numpy(), g['pos'], 1e-5, what='pos')
    assert_close(out['neg'].cpu().numpy().reshape(g['neg'].shape), g['neg'], 1e-5, what='neg')
    assert_close(out['loss'].item(), g['loss'], 1e-5, what='loss')
    assert_close(out['dE'].cpu().numpy(), g['grad.item_embeddings.weight'], 1e-5, what='dE')
    assert_close(out['dbias'].cpu().numpy(), g['grad.item_biases.weight'], 1e-5, what='dbias')
    assert float(out['dE'][0].abs().sum()) == 0.0
    rep = ops.seq_representation(t(g['sd.item_embeddings.weight']), t(g['seqs']), None)
    assert_close(rep[:, -1].cpu().numpy(), g['final'], 1e-5, what='final')
    assert_close(rep[:, :-1].permute(0, 2, 1).cpu().numpy(), g['user_rep'], 1e-5, what='user_rep')


@pytest.mark.parametrize('name,loss', [('cnn_pointwise', 'pointwise'), ('cnn_bpr_l2_relu', 'bpr'),
                                       ('cnn_adaptive_k5_nores', 'adaptive_hinge'),
                                       ('cnn_pointwise_d128', 'pointwise')])
def test_cnn_step_golden(name, loss):
    # cnn_pointwise_d128 runs the wgmma conv (D == 128) against the live reference's
    # scores and gradients at the north star's 1e-5; the D = 16 cases run the mma.sync path
    from spotlight_b200 import ops
    g = load_golden(name)
    n_neg = int(g['n_neg']) if loss == 'adaptive_hinge' else 1
    spec = _cnn_spec(g)
    out = ops.seq_train_step(t(g['sd.item_embeddings.weight']), t(g['sd.item_biases.weight']),
                             t(g['seqs']), t(g['negs']), loss, n_neg, spec, want_scores=True)
    assert_close(out['pos'].cpu().numpy(), g['pos'], 1e-5, what='pos')
    assert_close(out['neg'].cpu().numpy().reshape(g['neg'].shape), g['neg'], 1e-5, what='neg')
    assert_close(out['loss'].item(), g['loss'], 1e-5, what='loss')
    assert_close(out['dE'].cpu().numpy(), g['grad.item_embeddings.weight'], 1e-5, what='dE')
    assert_close(out['dbias'].cpu().numpy(), g['grad.item_biases.weight'], 1e-5, what='dbias')
    for i in range(len(spec['weights'])):
        assert_close(out['dconv_w'][i].cpu().numpy(), g['grad.cnn_%d.weight' % i], 1e-5, what='dW%d' % i)
        assert_close(out['dconv_b'][i].cpu().numpy(), g['grad.cnn_%d.bias' % i], 1e-5, what='db%d' % i)
    rep = ops.seq_representation(t(g['sd.item_embeddings.weight']), t(g['seqs']), spec)
    assert_close(rep[:, -1].cpu().numpy(), g['final'], 1e-5, what='final')


@pytest.mark.parametrize('kind', ['pool', 'cnn', 'cnn_relu'])
@pytest.mark.parametrize('D,S,B', [(128, 200, 16), (64, 33, 40), (256, 7, 9)])
def test_seq_step_vs_oracle_sizes(kind, D, S, B):
    nl = 'relu' if kind == 'cnn_relu' else 'tanh'
    kind = kind.split('_')[0]
    from spotlight_b200 import ops
    rs = np.random.RandomState(D + S)
    I = 500
    E = (rs.randn(I, D) * 0.2).astype(np.float32)
    E[0] = 0
    bias = (rs.randn(I, 1) * 0.1).astype(np.float32)
    bias[0] = 0
    seqs = rs.randint(1, I, (B, S)).astype(np.int64)
    for b in range(0, B, 2):
        seqs[b, :rs.randint(0, S)] = 0
    negs = rs.randint(0, I, (B, S)).astype(np.int64)
    spec, convs = None, None
    if kind == 'cnn':
        W = [(rs.randn(D, D, 3, 1) * 0.05).astype(np.float32), (rs.randn(D, D, 2, 1) * 0.05).astype(np.float32)]
        bb = [(rs.randn(D) * 0.05).astype(np.float32) for _ in W]
        convs = list(zip(W, bb))
        spec = dict(kernel_width=[3, 2], dilation=[1, 2], nonlinearity=nl, residual=True,
                    weights=[t(w) for w in W], biases=[t(x) for x in bb])
        ref = oseq.cnn_step(E, bias, convs, seqs, negs, [3, 2], [1, 2], 'bpr', 1, nl, True, np.float64)
    else:
        ref = oseq.pool_step(E, bias, seqs, negs, 'bpr', 1, np.float64)
    out = ops.seq_train_step(t(E), t(bias), t(seqs), t(negs), 'bpr', 1, spec, want_scores=True)
    assert_close(out['pos'].cpu().numpy(), ref['pos'], 2e-5, what='pos')
    assert_close(out['loss'].item(), ref['loss'], 1e-5, what='loss')
    assert_close(out['dE'].cpu().numpy(), ref['dE'], 2e-5, what='dE')
    assert_close(out['dbias'].cpu().numpy(), ref['dbias'], 2e-5, what='dbias')
    if kind == 'cnn':
        for i in range(2):
            assert_close(out['dconv_w'][i].cpu().numpy(), ref['dconvs'][i][0], 2e-5, what='dW')
            assert_close(out['dconv_b'][i].cpu().numpy(), ref['dconvs'][i][1], 2e-5, what='db')
    out2 = ops.seq_train_step(t(E), t(bias), t(seqs), t(negs), 'bpr', 1, spec)
    assert torch.equal(out['dE'], out2['dE']), 'sequence step is not bit-reproducible'


@pytest.mark.parametrize('name,loss', [('pool_bpr', 'bpr'), ('pool_hinge', 'hinge'), ('cnn_pointwise', 'pointwise'),
                                       ('cnn_pointwise_d128', 'pointwise')])
def test_seq_step_fused_sgd_golden(name, loss):
    """The sequence step with the row-wise optimizer fused into the gradient reduction (no dense
    item-table gradient): one SGD step reproduces E - lr * (the live reference's gradient)."""
    from spotlight_b200 import _lib, ops
    g = load_golden(name)
    spec = _cnn_spec(g) if name.startswith('cnn') else None
    gE, gb = g['grad.item_embeddings.weight'], g['grad.item_biases.weight']
    lr = 0.3 / np.abs(gE).max()
    E, b = t(g['sd.item_embeddings.weight'].copy()), t(g['sd.item_biases.weight'].copy())
    out = ops.seq_train_step(E, b, t(g['seqs']), t(g['negs']), loss, 1, spec,
                             fused=dict(kind=_lib.OPT_SGD, lr=lr, weight_decay=0.0, eps=0.0))
    assert out['dE'] is None and out['dbias'] is None
    assert_close(out['loss'].item(), g['loss'], 1e-5, what='loss')
    assert_close(E.cpu().numpy(), g['sd.item_embeddings.weight'].astype(np.float64) - lr * gE, 5e-6, what='E')
    assert_close(b.cpu().numpy(), g['sd.item_biases.weight'].astype(np.float64) - lr * gb, 5e-6, what='bias')
    assert float(E[0].abs().sum()) == 0.0                    # the padding row stays frozen
    if spec is not None:
        for i in range(len(spec['weights'])):
            assert_close(out['dconv_w'][i].cpu().numpy(), g['grad.cnn_%d.weight' % i], 1e-5, what='dW%d' % i)


@pytest.mark.parametrize('name,loss,rep', [('fit_pool_hinge', 'hinge', 'pooling'),
                                           ('fit_cnn_pointwise', 'pointwise', 'cnn')])
def test_sequence_model_fit_golden_fused_optimizer(name, loss, rep, capsys):
    """ImplicitSequenceModel.fit with spotlight_b200.optim.fused_sgd (item table updated inside the
    step, conv parameters by the optimizer's own step()) against the reference trajectory."""
    from spotlight_b200 import optim
    from spotlight_b200.interactions import SequenceInteractions
    from spotlight_b200.sequence.implicit import ImplicitSequenceModel
    g = load_golden(name)
    inter = SequenceInteractions(g['seqs'], num_items=int(g['num_items']))
    model = ImplicitSequenceModel(loss=loss, representation=rep, embedding_dim=int(g['dim']),
                                  batch_size=int(g['batch']), n_iter=int(g['n_iter']),
                                  optimizer_func=optim.fused_sgd(lr=0.5), use_cuda=True,
                                  random_state=np.random.RandomState(int(g['seed'])))
    model._initialize(inter)
    model._net.load_state_dict({k[5:]: torch.from_numpy(v) for k, v in g.items() if k.startswith('init.')})
    model.fit(inter, verbose=True)
    lines = [l for l in capsys.readouterr().out.strip().split('\n') if l.startswith('Epoch')]
    losses = np.array([float(l.split('loss')[1]) for l in lines])
    assert_close(losses, g['epoch_losses'], 1e-5, what='epoch losses')
    for k, v in model._net.state_dict().items():
        assert_close(v.cpu().numpy(), g['final.' + k], 1e-4, atol=1e-7, what=k)
    assert model._net.item_embeddings.weight.grad is None


@pytest.mark.parametrize('name,loss,rep', [('fit_pool_hinge', 'hinge', 'pooling'),
                                           ('fit_cnn_pointwise', 'pointwise', 'cnn')])
def test_sequence_model_fit_golden(name, loss, rep, capsys):
    from spotlight_b200.interactions import SequenceInteractions
    from spotlight_b200.sequence.implicit import ImplicitSequenceModel
    g = load_golden(name)
    inter = SequenceInteractions(g['seqs'], num_items=int(g['num_items']))
    model = ImplicitSequenceModel(loss=loss, representation=rep, embedding_dim=int(g['dim']),
                                  batch_size=int(g['batch']), n_iter=int(g['n_iter']),
                                  optimizer_func=lambda p: torch.optim.SGD(p, lr=0.5), use_cuda=True,
                                  random_state=np.random.RandomState(int(g['seed'])))
    model._initialize(inter)
    model._net.load_state_dict({k[5:]: torch.from_numpy(v) for k, v in g.items() if k.startswith('init.')})
    assert model._route() == 'fused'
    model.fit(inter, verbose=True)
    lines = [l for l in capsys.readouterr().out.strip().split('\n') if l.startswith('Epoch')]
    losses = np.array([float(l.split('loss')[1]) for l in lines])
    assert_close(losses, g['epoch_losses'], 1e-5, what='epoch losses')
    for k, v in model._net.state_dict().items():
        assert_close(v.cpu().numpy(), g['final.' + k], 1e-4, atol=1e-7, what=k)
    st = model._random_state.get_state()
    assert (st[1] == g['rs_key']).all() and st[2] == int(g['rs_pos'])
    assert_close(model.predict(g['seqs'][1]), g['predict'], 1e-4, what='predict')


def test_generic_route_pool_bloom_golden():
    """PoolNet over a BloomEmbedding through the generic autograd route (Bloom gather
    / scatter kernels + loss kernel) vs the reference's grads."""
    from spotlight_b200 import losses
    from spotlight_b200.layers import BloomEmbedding
    from spotlight_b200.sequence.representations import PoolNet
    g = load_golden('pool_pointwise_bloom')
    I, D = int(g['num_items']), int(g['dim'])
    emb = BloomEmbedding(I, D, compression_ratio=float(g['bloom_ratio']),
                         num_hash_functions=int(g['bloom_H']), padding_idx=0)
    net = PoolNet(I, D, item_embedding_layer=emb)
    net.load_state_dict({k[3:]: torch.from_numpy(v) for k, v in g.items() if k.startswith('sd.')})
    net = net.to('cuda:0')
    assert not net.fusable()
    seqs, negs = t(g['seqs']), t(g['negs'])
    rep, final = net.user_representation(seqs)
    pos = net(rep, seqs)
    neg = net(rep, negs)
    loss = losses.pointwise_loss(pos, neg, mask=(seqs != 0))
    loss.backward()
    assert_close(pos.detach().cpu().numpy(), g['pos'], 1e-5, what='pos')
    assert_close(neg.detach().cpu().numpy(), g['neg'], 1e-5, what='neg')
    assert_close(loss.item(), g['loss'], 1e-5, what='loss')
    assert_close(final.detach().cpu().numpy(), g['final'], 1e-5, what='final')
    for k, p in net.named_parameters():
        assert_close(p.grad.cpu().numpy(), g['grad.' + k], 1e-5, atol=1e-7, what=k)


def test_sequence_model_bloom_fit_runs():
    """ImplicitSequenceModel with a Bloom-embedded CNNNet takes the generic route."""
    from spotlight_b200.interactions import SequenceInteractions
    from spotlight_b200.layers import BloomEmbedding
    from spotlight_b200.sequence.implicit import ImplicitSequenceModel
    from spotlight_b200.sequence.representations import CNNNet
    rs = np.random.RandomState(0)
    seqs = rs.randint(1, 200, (64, 8)).astype(np.int32)
    rep = CNNNet(200, 16, item_embedding_layer=BloomEmbedding(200, 16, compression_ratio=0.5,
                                                              num_hash_functions=2, padding_idx=0))
    model = ImplicitSequenceModel(loss='bpr', representation=rep, embedding_dim=16, batch_size=32,
                                  n_iter=2, use_cuda=True, random_state=np.random.RandomState(1))
    model.fit(SequenceInteractions(seqs, num_items=200))
    assert model._route() == 'generic'
    assert model.predict(seqs[0]).shape == (200,)


def test_seq_step_global_norm_count():
    """Multi-GPU hook: with norm_count = c x (this batch's unmasked count) the loss share
    and every gradient are the single-rank ones divided by c."""
    from spotlight_b200 import ops
    g = load_golden('pool_bpr')
    E, b = t(g['sd.item_embeddings.weight']), t(g['sd.item_biases.weight'])
    seqs, negs = t(g['seqs']), t(g['negs'])
    base = ops.seq_train_step(E, b, seqs, negs, 'bpr', 1, None)
    norm = ((seqs != 0).sum() * 4).to(torch.int32).reshape(1)
    out = ops.seq_train_step(E, b, seqs, negs, 'bpr', 1, None, norm_count=norm)
    assert_close(out['loss'].item() * 4, base['loss'].item(), 1e-6, what='loss')
    assert_close(out['dE'].cpu().numpy() * 4, base['dE'].cpu().numpy(), 1e-6, what='dE')
    assert_close(out['dbias'].cpu().numpy() * 4, base['dbias'].cpu().numpy(), 1e-6, what='dbias')
