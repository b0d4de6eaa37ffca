"""MixtureLSTMNet evaluation on the device: slb_mixture_scores against the float64 all-items head
(oracle.mixture_eval.score_items), its bit-determinism, 64-bit offsets and argument checks, and the
sequence scorers on the new path against the live reference (tests/golden/eval_mixture.npz), the
generic forward() path, and the routing that decides between them."""

import ctypes

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import mixture_eval as ome

pytestmark = pytest.mark.gpu


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _scores(reps, M, items, bias):
    """slb_mixture_scores on device tensors; returns the status and the (n, I) block."""
    from spotlight_b200 import _lib, ops
    n, I = reps.shape[0], items.shape[0]
    out = torch.full((n, I), float('nan'), device='cuda')
    rc = _lib.load().slb_mixture_scores(_p(reps), n, M, reps.shape[2], _p(items), _p(bias), I, _p(out),
                                        ops._stream())
    return rc, out


def _inputs(M, D, n, I, seed):
    rs = np.random.RandomState(seed)
    reps = (rs.randn(n, 2 * M, D) * 0.5 / np.sqrt(D) * 4).astype(np.float32)
    items = (rs.randn(I, D) * 0.5).astype(np.float32)
    bias = (rs.randn(I) * 0.1).astype(np.float32)
    return reps, items, bias


def _cuda(*arrays):
    return [torch.from_numpy(a).cuda() for a in arrays]


# (M, D, n_rows, n_items): every M, D, n_rows and n_items of the sweep at least once, full and
# partial D chunks (16 columns), one and several sequence and item tiles, and their tails
CASES = [(1, 4, 1, 1), (2, 16, 5, 6), (3, 36, 64, 1003), (4, 128, 257, 4099), (8, 256, 5, 1003),
         (8, 512, 64, 6), (1, 512, 257, 1003), (4, 4, 64, 4099), (3, 128, 1, 4099), (2, 36, 257, 1),
         (5, 16, 64, 1003), (6, 4, 5, 6), (7, 36, 1, 1003), (1, 16, 65, 4099), (2, 128, 33, 130)]


@pytest.mark.parametrize('M,D,n,I', CASES)
def test_kernel_equals_float64_head(M, D, n, I):
    reps, items, bias = _inputs(M, D, n, I, seed=M * 1000 + D + n + I)
    rc, got = _scores(*_cuda(reps), M, *_cuda(items, bias))
    assert rc == 0
    got = got.cpu().numpy().astype(np.float64)
    want = ome.score_items(reps, items, bias, M)
    tol = 1e-5 * np.abs(want) + 1e-5 * np.abs(want).max(axis=1, keepdims=True)
    err = np.abs(got - want)
    assert (err <= tol).all(), (err.max(), np.unravel_index(np.argmax(err - tol), err.shape))


@pytest.mark.parametrize('M,D', [(4, 36), (1, 128), (3, 20), (8, 16)])
def test_kernel_is_bit_deterministic(M, D):
    n, I = 37, 1003
    reps, items, bias = _inputs(M, D, n, I, seed=7)
    dup = [5, 130, 517, I - 1]                  # other tiles and the tail of the last one
    items[dup] = items[dup[0]]
    bias[dup] = bias[dup[0]]
    r, e, b = _cuda(reps, items, bias)
    rc, block = _scores(r, M, e, b)
    assert rc == 0
    rc, again = _scores(r, M, e, b)
    assert rc == 0 and torch.equal(block.view(torch.int32), again.view(torch.int32))
    for i in range(n):                          # each row alone
        rc, one = _scores(r[i:i + 1].contiguous(), M, e, b)
        assert rc == 0 and torch.equal(one[0].view(torch.int32), block[i].view(torch.int32)), i
    cols = block[:, dup].view(torch.int32)
    assert torch.equal(cols, cols[:, :1].expand_as(cols))
    # the same item in a smaller table (another tile position, another tail) scores the same bits
    rc, few = _scores(r, M, e[dup[0]:dup[0] + 3].contiguous(), b[dup[0]:dup[0] + 3].contiguous())
    assert rc == 0 and torch.equal(few[:, 0].view(torch.int32), block[:, dup[0]].view(torch.int32))


def test_kernel_64bit_offsets():
    free, _ = torch.cuda.mem_get_info()
    if free < 16 << 30:
        pytest.skip('needs 16 GB of free device memory')
    M, D, n, I = 1, 4, 2049, 1048583
    assert n * I > 1 << 31
    reps, items, bias = _inputs(M, D, n, I, seed=11)
    r, e, b = _cuda(reps, items, bias)
    rc, out = _scores(r, M, e, b)
    assert rc == 0
    rs = np.random.RandomState(12)
    flat = np.concatenate([rs.randint(1 << 31, n * I, 2000), [n * I - 1, (1 << 31) - 1, 1 << 31]])
    rows, cols = flat // I, flat % I
    got = out.view(-1)[torch.from_numpy(flat).cuda()].cpu().numpy().astype(np.float64)
    P = reps.astype(np.float64)
    E = items.astype(np.float64)
    c = (P[rows, 0] * E[cols]).sum(1)           # M = 1: the softmax weight is exactly 1
    want = bias[cols] + c
    del out
    assert np.all(np.abs(got - want) <= 1e-5 * np.abs(want) + 1e-6), np.abs(got - want).max()


def test_c_abi_rejects_bad_arguments():
    from spotlight_b200 import _lib, ops
    lib = _lib.load()
    reps, items, bias = _cuda(*_inputs(2, 8, 3, 10, seed=1))
    out = torch.zeros(3, 10, device='cuda')
    reps9 = torch.zeros(3, 18, 8, device='cuda')

    def call(r=reps, n=3, M=2, D=8, e=items, b=bias, I=10, o=out):
        return lib.slb_mixture_scores(_p(r), n, M, D, _p(e), _p(b), I, _p(o), ops._stream())

    assert call() == 0
    assert call(M=0) != 0
    assert call(r=reps9, M=9) != 0
    assert call(D=6) != 0
    assert call(e=None) != 0
    assert call(o=None) != 0
    assert call(n=0) != 0
    assert call(I=0) != 0


# ---- the scorers

def _fixture_model(g, name):
    from spotlight_b200.interactions import SequenceInteractions
    from spotlight_b200.layers import BloomEmbedding
    from spotlight_b200.sequence.implicit import ImplicitSequenceModel
    from spotlight_b200.sequence.representations import MixtureLSTMNet
    I, D, M = int(g['num_items']), int(g['dim']), int(g[name + '.num_mixtures'])
    if name == 'mixture':
        rep = 'mixture'
    elif name + '.bloom' in g:
        ratio, H = g[name + '.bloom']
        rep = MixtureLSTMNet(I, D, num_mixtures=M,
                             item_embedding_layer=BloomEmbedding(I, D, float(ratio), int(H), padding_idx=0))
    else:
        rep = MixtureLSTMNet(I, D, num_mixtures=M)
    inter = SequenceInteractions(g['seqs'], num_items=I)
    model = ImplicitSequenceModel(representation=rep, embedding_dim=D, use_cuda=True)
    model._initialize(inter)
    pre = name + '.sd.'
    model._net.load_state_dict({k[len(pre):]: torch.from_numpy(v) for k, v in g.items() if k.startswith(pre)})
    assert model._net.num_mixtures == M
    return model, inter


def _no_generic(monkeypatch):
    from spotlight_b200 import evaluation

    def fail(*a, **k):
        raise AssertionError('the generic path ran')
    monkeypatch.setattr(evaluation, '_generic_block', fail)


def _all_metrics(model, inter, ex, block):
    from spotlight_b200.evaluation import sequence_mrr_score, sequence_precision_recall_score
    out = {'mrr': sequence_mrr_score(model, inter, exclude_preceding=ex, sequence_block=block)}
    for k in (1, 3):
        out['p%d' % k], out['r%d' % k] = sequence_precision_recall_score(model, inter, k=k, exclude_preceding=ex,
                                                                        sequence_block=block)
    return out


@pytest.mark.parametrize('name', ['mixture', 'm2', 'bloom'])
def test_scorers_match_reference_golden(name, monkeypatch):
    g = load_golden('eval_mixture')
    model, inter = _fixture_model(g, name)
    _no_generic(monkeypatch)
    for ex in (False, True):
        got = _all_metrics(model, inter, ex, block=5)
        np.testing.assert_allclose(got['mrr'], g['%s.mrr.ex%d' % (name, ex)], rtol=1e-6)
        for k in (1, 3):
            np.testing.assert_allclose(got['p%d' % k], g['%s.pr.ex%d.k%d.p' % (name, ex, k)], rtol=1e-6)
            np.testing.assert_allclose(got['r%d' % k], g['%s.pr.ex%d.k%d.r' % (name, ex, k)], rtol=1e-6)


def _trained_model():
    """A fitted 4-taste model with two identical item rows (an exact tie in every score row)."""
    from spotlight_b200.interactions import SequenceInteractions
    from spotlight_b200.sequence.implicit import ImplicitSequenceModel
    rs = np.random.RandomState(3)
    I, N, S = 2000, 300, 12
    seqs = rs.randint(1, I, (N, S)).astype(np.int32)
    seqs[::4, :5] = 0
    seqs[1::7, 3] = seqs[1::7, -1]
    inter = SequenceInteractions(seqs, num_items=I)
    model = ImplicitSequenceModel(representation='mixture', embedding_dim=16, n_iter=1, batch_size=64,
                                  use_cuda=True, random_state=np.random.RandomState(4))
    model.fit(inter)
    with torch.no_grad():
        model._net.item_embeddings.weight[7] = model._net.item_embeddings.weight[3]
        model._net.item_biases.weight[7] = model._net.item_biases.weight[3]
    return model, inter


def _statistically_equal(got, want):
    # the kernel and forward() sum in different fp32 orders: items whose scores differ by ~1e-7
    # relative may swap for a few rows
    err = np.abs(np.asarray(got, np.float64) - want).reshape(len(want), -1).max(1)
    assert np.median(err) < 1e-7 and (err < 1e-6).mean() > 0.9, (np.median(err), err.max())


@pytest.mark.parametrize('ex', [False, True])
def test_scorers_equal_generic_path(ex, monkeypatch):
    from spotlight_b200 import evaluation
    g = load_golden('eval_mixture')
    models = [_fixture_model(g, name) for name in ('mixture', 'm2', 'bloom')] + [_trained_model()]
    for model, inter in models:
        fused = _all_metrics(model, inter, ex, block=64)
        with monkeypatch.context() as mp:
            mp.setattr(evaluation, '_mixture_head', lambda net, final: False)
            generic = _all_metrics(model, inter, ex, block=64)
        for key in fused:
            _statistically_equal(fused[key], generic[key])
    model, inter = models[-1]
    with torch.no_grad():                        # the tied items score the same bits
        blk = evaluation._score_sequences(model, torch.from_numpy(inter.sequences[:64, :-1].astype(np.int64)).cuda())
    assert torch.equal(blk[:, 3].view(torch.int32), blk[:, 7].view(torch.int32))
    # the block size changes nothing
    a = _all_metrics(model, inter, ex, block=64)
    b = _all_metrics(model, inter, ex, block=7)
    for key in a:
        assert np.array_equal(a[key], b[key]), key


def test_routing_takes_the_kernel_without_forward(monkeypatch):
    from spotlight_b200.sequence.representations import MixtureLSTMNet
    g = load_golden('eval_mixture')
    model, inter = _fixture_model(g, 'm2')
    want = _all_metrics(model, inter, True, block=5)

    def fail(self, *a):
        raise AssertionError('forward() ran')
    monkeypatch.setattr(MixtureLSTMNet, 'forward', fail)
    got = _all_metrics(model, inter, True, block=5)
    for key in want:
        assert np.array_equal(got[key], want[key]), key


def _small_net(cls, D, M):
    from spotlight_b200.interactions import SequenceInteractions
    from spotlight_b200.sequence.implicit import ImplicitSequenceModel
    rs = np.random.RandomState(5)
    I = 50
    seqs = rs.randint(1, I, (20, 7)).astype(np.int32)
    inter = SequenceInteractions(seqs, num_items=I)
    torch.manual_seed(5)
    model = ImplicitSequenceModel(representation=cls(I, D, num_mixtures=M), embedding_dim=D, use_cuda=True)
    model._initialize(inter)
    return model, inter


@pytest.mark.parametrize('kind', ['subclass', 'nine_mixtures', 'd6'])
def test_routing_keeps_other_nets_on_forward(kind, monkeypatch):
    from spotlight_b200 import evaluation
    from spotlight_b200.sequence.representations import MixtureLSTMNet
    calls = []

    class Overriding(MixtureLSTMNet):
        def forward(self, user_representations, targets):
            calls.append(1)
            return super(Overriding, self).forward(user_representations, targets)

    if kind == 'subclass':
        model, inter = _small_net(Overriding, 8, 2)
    else:
        model, inter = _small_net(MixtureLSTMNet, 8 if kind == 'nine_mixtures' else 6,
                                  9 if kind == 'nine_mixtures' else 2)
        real = MixtureLSTMNet.forward

        def counting(self, *a):
            calls.append(1)
            return real(self, *a)
        monkeypatch.setattr(MixtureLSTMNet, 'forward', counting)

    def no_kernel(*a, **k):
        raise AssertionError('slb_mixture_scores ran')
    got = {}
    with monkeypatch.context() as mp:
        mp.setattr(evaluation, '_mixture_block', no_kernel)
        got = _all_metrics(model, inter, True, block=8)
    assert calls
    # the previous route: the net's forward over item chunks
    with monkeypatch.context() as mp:
        mp.setattr(evaluation, '_mixture_head', lambda net, final: False)
        want = _all_metrics(model, inter, True, block=8)
    for key in want:
        assert np.array_equal(got[key], want[key]), key
